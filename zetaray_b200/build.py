"""In-tree build of libzetaray_b200.so for sm_90a (H100) (nvcc cross-compiles without a GPU).

    python zetaray_b200/build.py [--force]

Every .cu under zetaray_b200/csrc is compiled to an object (in parallel) and linked into
zetaray_b200/libzetaray_b200.so next to this file, so the binary travels with the repo snapshot."""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# ZR_VARIANT=<name> ZR_EXTRA_FLAGS="-D..." builds an experimental libzetaray_b200_<name>.so beside the default one
# (selected at run time with ZETARAY_B200_LIB); used for A/B measurements.
VARIANT = os.environ.get("ZR_VARIANT", "")
OBJ = os.path.join(HERE, "build" + ("_" + VARIANT if VARIANT else ""))
SO = os.path.join(HERE, "libzetaray_b200%s.so" % ("_" + VARIANT if VARIANT else ""))
NVCC = os.environ.get("NVCC", os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc"))
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]

# -fmad=false / -ffp-contract=off: the numeric contract (DESIGN.md) -- fused multiply-adds appear only
# where the code says fmaf(), exactly like the CPU oracle, so results are bit-comparable.
NVCC_FLAGS = [
    *GENCODE, "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=hidden,-O2",
    "-I" + os.path.join(os.path.dirname(HERE), "include"),
]


def _deps():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    inc = os.path.join(os.path.dirname(HERE), "include")
    hdrs += [os.path.join(inc, f) for f in os.listdir(inc)]
    return hdrs


def _compile(src, force):
    obj = os.path.join(OBJ, os.path.basename(src) + ".o")
    deps = [src] + _deps() + [__file__]
    if not force and os.path.exists(obj) and all(os.path.getmtime(d) <= os.path.getmtime(obj) for d in deps):
        return obj, False
    cmd = [NVCC] + NVCC_FLAGS + os.environ.get("ZR_EXTRA_FLAGS", "").split() + ["-c", src, "-o", obj]
    if os.environ.get("ZR_PTXAS_V"):
        cmd += ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    if os.environ.get("ZR_PTXAS_V"):
        sys.stderr.write(r.stderr)
    return obj, True


def build(force=False, verbose=True):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, force), srcs))
    objs = [o for o, _ in res]
    changed = any(c for _, c in res)
    if changed or not os.path.exists(SO):
        cmd = [NVCC, "-shared", *GENCODE, "-o", SO] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
        if verbose:
            print("built", SO)
    return SO


if __name__ == "__main__":
    build(force="--force" in sys.argv)
