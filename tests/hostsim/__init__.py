"""TEST INFRASTRUCTURE: the product's device headers compiled for the host (g++) -- hostsim.cpp (traversal, BSDF, ray queries, ReSTIR PT
shift, ReSTIR GI reuse, probes mirrored by the oracle) and hostsim_di.cpp (ReSTIR DI; a translation unit of its own)."""
import ctypes as C
import os
import subprocess

from zetaray_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libhostsim.so")
SO_DI = os.path.join(HERE, "libhostsim_di.so")
SO_IO = os.path.join(HERE, "libhostsim_io.so")
_CSRC = os.path.join(os.path.dirname(os.path.dirname(HERE)), "zetaray_b200", "csrc")
_INC = os.path.join(os.path.dirname(os.path.dirname(HERE)), "include")
HEADER = os.path.join(HERE, "hostsim_api.h")
ORC_HEADER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "orc_api.h")


def prototypes():
    """{name: (restype, [argtypes])} of every function of hostsim_api.h, across the three libraries."""
    with open(HEADER) as f:
        return _lib.prototypes(f.read(), "HOSTSIM_API", "hostsim_")


class Scene(C.Structure):
    """hostsim_scene: a scene resident in host memory, in the device's layouts."""
    _fields_ = [("vertices", C.c_void_p), ("indices", C.c_void_p), ("instances", C.c_void_p), ("materials", C.c_void_p),
                ("emissives", C.c_void_p), ("aliasTable", C.c_void_p), ("nodes", C.c_void_p), ("leafTris", C.c_void_p),
                ("triMesh", C.c_void_p), ("meshFirstTri", C.c_void_p), ("rho", C.c_void_p),
                ("numInstances", C.c_uint32), ("numEmissives", C.c_uint32), ("numTris", C.c_uint32),
                ("sampleSets", C.c_void_p), ("numSampleSets", C.c_uint32), ("sampleSetSize", C.c_uint32),
                ("lvg", C.c_void_p), ("lvgDim", C.c_uint32 * 3), ("lvgExtents", C.c_float * 3), ("lvgOffsetY", C.c_float)]


def _deps(src):
    hdrs = [os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h"))]
    hdrs += [os.path.join(_INC, f) for f in os.listdir(_INC)]
    return [src, os.path.join(HERE, "prelude.h"), HEADER, ORC_HEADER] + hdrs


def _build(src, so, force, defines=()):
    if not force and os.path.exists(so) and all(os.path.getmtime(d) <= os.path.getmtime(so) for d in _deps(src)):
        return so
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I" + cuda_inc,
           "-D__forceinline__=inline __attribute__((always_inline))"] + ["-D" + d for d in defines] + [src, "-o", so, "-lpthread"]
    subprocess.check_call(cmd)
    return so


def build(force=False):
    _build(os.path.join(HERE, "hostsim_di.cpp"), SO_DI, force)
    _build(os.path.join(HERE, "hostsim_io.cpp"), SO_IO, force)
    return _build(os.path.join(HERE, "hostsim.cpp"), SO, force)


def _open(so):
    """The library with the prototypes of the functions of hostsim_api.h it defines (the header declares all three libraries')."""
    lib = C.CDLL(so)
    return _lib.declare(lib, {name: p for name, p in prototypes().items() if hasattr(lib, name)})


def load():
    return _open(build())


def load_di():
    build()
    return _open(SO_DI)


def load_io():
    build()
    return _open(SO_IO)
