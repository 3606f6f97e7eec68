"""ctypes loader for the CPU oracle (oracle/liborc.so) and the compiled reference (oracle/_ref).

Only tests/, __graft_entry__.smoke(), bench.py's cpu_baseline / --impl reference legs and tools/make_reference_golden.py may use
this; the compiled reference is for the tool alone (the tests read its stored outputs in tests/golden/)."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
_lib = None
_ref = None


def build(force=False):
    so = os.path.join(ORACLE_DIR, "liborc.so")
    srcs = [os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.startswith("orc_")]
    srcs += [os.path.join(ROOT, "include", f) for f in os.listdir(os.path.join(ROOT, "include"))]
    stale = force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if stale:
        subprocess.check_call(["make", "-C", ORACLE_DIR, "liborc.so"], stdout=subprocess.DEVNULL)
    return so


def load():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_kahan_sum.restype = C.c_float
        _lib.orc_halton.restype = C.c_float
        _lib.orc_pcg.restype = C.c_uint32
    return _lib


def load_ref():
    global _ref
    if _ref is None:
        so = os.path.join(ORACLE_DIR, "_ref", "libref_alias.so")
        if not os.path.exists(so):
            return None
        _ref = C.CDLL(so)
        _ref.ref_kahan_sum.restype = C.c_float
        _ref.ref_halton.restype = C.c_float
    return _ref


def ptr(a, t=C.c_void_p):
    return a.ctypes.data_as(t)
