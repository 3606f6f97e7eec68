"""ctypes loader for the CPU oracle (oracle/liborc.so) and the compiled reference (oracle/_ref).

Only tests/, __graft_entry__.smoke(), bench.py's cpu_baseline / --impl reference legs and tools/make_reference_golden.py may use
this; the compiled reference is for the tool alone (the tests read its stored outputs in tests/golden/).

Every function a library exports gets its argtypes and restype from its prototype in the library's header (oracle/orc_api.h,
oracle/ref_*/ref_*_api.h) when the library is opened, so a wrongly typed call raises in Python instead of reaching C."""
import ctypes as C
import os
import subprocess

from zetaray_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
HEADER = os.path.join(ORACLE_DIR, "orc_api.h")
REF_HEADERS = {"libref_alias.so": os.path.join(ORACLE_DIR, "ref_alias", "ref_alias_api.h"),
               "libref_scene.so": os.path.join(ORACLE_DIR, "ref_scene", "ref_scene_api.h")}
_lib_orc = None
_refs = {}


def prototypes(header=HEADER, macro="ORC_API", prefix="orc_"):
    with open(header) as f:
        return _lib.prototypes(f.read(), macro, prefix)


class SurfaceDesc(C.Structure):
    """orc_surface_desc: a BSDF probe surface (the oracle's and tests/hostsim's BSDF probes take it)."""
    _fields_ = [("normal", C.c_float * 3), ("wo", C.c_float * 3), ("metallic", C.c_uint32), ("roughness", C.c_float),
                ("baseColor", C.c_float * 3), ("eta_curr", C.c_float), ("eta_next", C.c_float), ("specTr", C.c_uint32),
                ("trDepth", C.c_float), ("subsurface", C.c_float), ("coat_weight", C.c_float), ("coat_color", C.c_float * 3),
                ("coat_roughness", C.c_float), ("coat_ior", C.c_float)]


class RptBuffers(C.Structure):
    """orc_rpt_buffers: the planes ReSTIR PT keeps across frames."""
    _fields_ = [("res", C.c_void_p * 2), ("target", C.c_void_p), ("finalImg", C.c_void_p), ("neighbor", C.c_void_p),
                ("threadMapCtN", C.c_void_p), ("threadMapNtC", C.c_void_p)]


def build(force=False):
    so = os.path.join(ORACLE_DIR, "liborc.so")
    srcs = [os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.startswith("orc_")]
    srcs += [os.path.join(ROOT, "include", f) for f in os.listdir(os.path.join(ROOT, "include"))]
    stale = force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if stale:
        subprocess.check_call(["make", "-C", ORACLE_DIR, "liborc.so"], stdout=subprocess.DEVNULL)
    return so


def load():
    global _lib_orc
    if _lib_orc is None:
        _lib_orc = _lib.declare(C.CDLL(build()), prototypes())
    return _lib_orc


def _load_ref(name):
    """oracle/_ref/<name> with the prototypes of its wrapper's header, or None when the reference was not built here."""
    if name not in _refs:
        so = os.path.join(ORACLE_DIR, "_ref", name)
        _refs[name] = _lib.declare(C.CDLL(so), prototypes(REF_HEADERS[name], "REF_API", "ref_")) if os.path.exists(so) else None
    return _refs[name]


def load_ref():
    return _load_ref("libref_alias.so")


def load_ref_scene():
    return _load_ref("libref_scene.so")


def ptr(a, t=C.c_void_p):
    return a.ctypes.data_as(t)
