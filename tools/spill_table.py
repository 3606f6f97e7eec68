"""Static register / spill table of the lighting kernels (no GPU needed).

    ZR_PTXAS_V=1 python zetaray_b200/build.py --force 2> ptxas.log
    python tools/spill_table.py ptxas.log [zetaray_b200/libzetaray_b200.so]

For every k_pathtrace, k_di_temporal, k_di_spatial and k_shift<CASE, REPLAY, TEMPORAL> entry point, in its plain (no clear coat,
no transmission) and its full material-feature build, it prints what ptxas
reported (registers, stack frame, static spill store / load bytes, static shared memory; k_pathtrace's dynamic shared
memory is not in the log) and, from `cuobjdump -sass` of the library,
the number of SASS instructions and of local-memory loads (LDL) and stores (STL) in the kernel's code. The library
defaults to the one the log's build wrote (ZR_VARIANT selects libzetaray_b200_<variant>.so)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_BIN = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")
KERNELS = ("k_pathtrace", "k_di_temporal", "k_di_spatial", "k_shift")


def variant(mf):
    """The material-feature template argument (BSDF::ShadingDataT): 0 = the plain build, otherwise the full one."""
    return "plain" if int(mf) == 0 else "full"


def short_name(mangled):
    """_ZN2zr..._GLOBAL__N__..._6_rdi_cu_...13k_di_temporalILj0EEvNS_... -> k_di_temporal [plain]; k_shift keeps its template
    arguments and the pass it belongs to (spatial / temporal). Every kernel is listed once per material-feature build."""
    for k in KERNELS:
        if not re.search(r"\d+%sI" % k, mangled):
            continue
        if k != "k_shift":
            return "%s [%s]" % (k, variant(re.search(r"\d+%sILj(\d+)E" % k, mangled).group(1)))
        case, replay, temporal, mf = re.search(r"ILi(\d)ELb(\d)ELb(\d)ELj(\d+)E", mangled).groups()
        return "k_shift<%s,%s,%s> [%s]" % (case, "replay" if replay == "1" else "-", "temporal" if temporal == "1" else "spatial",
                                           variant(mf))
    return None


def parse_ptxas(text):
    rows, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = short_name(m.group(1))
            if cur:
                rows[cur] = {"mangled": m.group(1)}
            continue
        if not cur:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            rows[cur].update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            rows[cur]["regs"] = int(m.group(1))
            s = re.search(r"(\d+) bytes smem", line)
            rows[cur]["smem"] = int(s.group(1)) if s else 0
            cur = None
    return rows


def sass_counts(lib):
    out = subprocess.run([os.path.join(CUDA_BIN, "cuobjdump"), "-sass", lib], capture_output=True, text=True, check=True).stdout
    counts, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = {"insts": 0, "ldl": 0, "stl": 0}
            continue
        if cur is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if m:
            op = m.group(2).split(".")[0]
            counts[cur]["insts"] += 1
            counts[cur]["ldl"] += op == "LDL"
            counts[cur]["stl"] += op == "STL"
    return counts


def main():
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    rows = parse_ptxas(open(sys.argv[1]).read())
    variant = os.environ.get("ZR_VARIANT", "")
    lib = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "zetaray_b200", "libzetaray_b200%s.so" % ("_" + variant if variant else ""))
    sass = sass_counts(lib)
    print("| kernel | regs | stack B | spill st / ld B | smem B | SASS insts | LDL | STL |")
    print("|---|---|---|---|---|---|---|---|")
    for name in sorted(rows):
        r = rows[name]
        s = sass.get(r["mangled"], {"insts": "-", "ldl": "-", "stl": "-"})
        print("| `%s` | %s | %s | %s / %s | %s | %s | %s | %s |" % (name, r.get("regs"), r.get("stack"), r.get("spill_st"), r.get("spill_ld"),
                                                               r.get("smem"), s["insts"], s["ldl"], s["stl"]))


if __name__ == "__main__":
    main()
