"""ctypes binding of include/zr_abi.h. No compute happens here.

Every ZR_API function gets its argtypes and restype from its prototype in the header (prototypes()), so a call with a
wrongly typed or missing argument raises in Python instead of reaching the library."""
import ctypes as C
import os
import re

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(HERE), "include", "zr_abi.h")
SO_PATH = os.environ.get("ZETARAY_B200_LIB") or os.path.join(HERE, "libzetaray_b200.so")


class ZRError(RuntimeError):
    pass


def _load():
    if not os.path.exists(SO_PATH):
        raise ZRError(
            "libzetaray_b200.so is missing -- run `python -m zetaray_b200.build` (there is no CPU fallback)")
    try:
        import torch  # noqa: F401  (makes the process share torch's libcudart.so.12)
    except Exception:
        pass
    return C.CDLL(SO_PATH)


class _NoLibrary:
    """ZETARAY_B200_STRUCTS_ONLY=1 (bench.py's CPU reference arm): only the ctypes mirrors of the ABI structs are needed, the
    shared library is NOT mapped into the process; any call through `lib` fails loudly."""

    def __getattr__(self, name):
        raise ZRError("zetaray_b200 was imported with ZETARAY_B200_STRUCTS_ONLY=1: %s is not available in this process" % name)


u32, u64, f32, vp, i32 = C.c_uint32, C.c_uint64, C.c_float, C.c_void_p, C.c_int32

# Parameter and return types of the ZR_API prototypes. Besides these, every pointer parameter (T*, T**, T[N]) and every
# function-pointer typedef is a c_void_p, which takes byref(), pointer(), arrays, None, ints and CFUNCTYPE instances;
# every enum typedef is a c_int.
ARG_TYPES = {"uint32_t": u32, "uint64_t": u64, "size_t": C.c_size_t, "float": f32, "int": C.c_int}
RET_TYPES = {"zr_status": i32, "void": None, "uint32_t": u32, "uint64_t": u64, "const char*": C.c_char_p}


def prototypes(text=None):
    """{name: (restype, [argtypes])} for every ZR_API function of include/zr_abi.h (or of the header text `text`).
    A declaration that does not parse or uses a type outside the maps above raises ZRError naming it."""
    if text is None:
        with open(HEADER) as f:
            text = f.read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)          # the ZR_API definition itself
    args = dict(ARG_TYPES)
    args.update((e, C.c_int) for e in re.findall(r"typedef\s+enum\b[^{;]*\{[^}]*\}\s*(\w+)\s*;", text))
    args.update((fn, vp) for fn in re.findall(r"typedef\s+[\w\s*]+\(\s*\*\s*(\w+)\s*\)", text))
    out = {}
    for decl in re.findall(r"\bZR_API\b([^;]*);", text):
        decl = " ".join(decl.split())
        m = re.fullmatch(r"(.+?) ?\b(zr_\w+) ?\((.*)\)", decl)
        if m is None:
            raise ZRError("zr_abi.h: cannot parse the declaration %r" % decl)
        ret, name, params = m.groups()
        ret = ret.replace(" *", "*")
        if ret not in RET_TYPES:
            raise ZRError("zr_abi.h: %s returns %r, which has no ctypes type" % (decl, ret))
        argtypes = []
        for p in ([] if params == "void" else params.split(",")):
            p = p.strip()
            t = vp if "*" in p or "[" in p else args.get(p.rsplit(" ", 1)[0])
            if t is None:
                raise ZRError("zr_abi.h: %s takes %r, which has no ctypes type" % (decl, p))
            argtypes.append(t)
        out[name] = (RET_TYPES[ret], argtypes)
    return out


def declared_symbols():
    """All ZR_API functions declared in include/zr_abi.h."""
    return sorted(prototypes())


def _declare(dll):
    for name, (restype, argtypes) in prototypes().items():
        f = getattr(dll, name)
        f.restype, f.argtypes = restype, argtypes
    return dll


lib = _NoLibrary() if os.environ.get("ZETARAY_B200_STRUCTS_ONLY") == "1" else _declare(_load())


class FrameConstants(C.Structure):
    _fields_ = [
        ("CurrView", f32 * 12), ("PrevView", f32 * 12), ("CurrViewInv", f32 * 12), ("PrevViewInv", f32 * 12),
        ("CurrViewProj", f32 * 16), ("PrevViewProj", f32 * 16),
        ("CameraPos", f32 * 3), ("CameraNear", f32),
        ("AspectRatio", f32), ("PixelSpreadAngle", f32), ("TanHalfFOV", f32), ("dt", f32),
        ("FrameNum", u32), ("CurrGBufferDescHeapOffset", u32), ("PrevGBufferDescHeapOffset", u32),
        ("BaseColorMapsDescHeapOffset", u32),
        ("NormalMapsDescHeapOffset", u32), ("MetallicRoughnessMapsDescHeapOffset", u32),
        ("EmissiveMapsDescHeapOffset", u32), ("EnvMapDescHeapOffset", u32),
        ("RenderWidth", u32), ("RenderHeight", u32), ("DisplayWidth", u32), ("DisplayHeight", u32),
        ("CurrCameraJitter", f32 * 2), ("PrevCameraJitter", f32 * 2),
        ("PlanetRadius", f32), ("SunCosAngularRadius", f32), ("SunSinAngularRadius", f32), ("pad", f32),
        ("SunDir", f32 * 3), ("SunIlluminance", f32),
        ("RayleighSigmaSColor", f32 * 3), ("RayleighSigmaSScale", f32),
        ("OzoneSigmaAColor", f32 * 3), ("OzoneSigmaAScale", f32),
        ("MieSigmaS", f32), ("MieSigmaA", f32), ("AtmosphereAltitude", f32), ("g", f32),
        ("NumFramesCameraStatic", u32), ("CameraStatic", u32), ("Accumulate", u32), ("SunMoved", u32),
        ("CameraRayUVGradsScale", f32), ("MipBias", f32), ("OneDivNumEmissiveTriangles", f32),
        ("NumEmissiveTriangles", u32),
        ("FocusDepth", f32), ("LensRadius", f32), ("DoF", u32), ("pad2", u32),
    ]


class GBuffer(C.Structure):
    _fields_ = [("d_core", vp), ("d_depth", vp), ("d_motion_emissive", vp), ("d_coat", vp), ("d_tridiff", vp)]


class FrameInputs(C.Structure):
    _fields_ = [("frame", FrameConstants), ("curr", GBuffer), ("prev", GBuffer), ("scene", vp)]


class Image2D(C.Structure):
    _fields_ = [("d_ptr", vp), ("width", u32), ("height", u32), ("pitch_bytes", u32), ("texel_bytes", u32)]


class SceneDesc(C.Structure):
    _fields_ = [
        ("h_vertices", vp), ("num_vertices", u32),
        ("h_indices", vp), ("num_indices", u32),
        ("h_instances", vp), ("num_instances", u32),
        ("h_instance_num_tris", vp),
        ("h_materials", vp), ("num_materials", u32),
        ("h_emissives", vp), ("num_emissives", u32),
    ]


class DirectParams(C.Structure):
    _fields_ = [("temporal_resample", u32), ("spatial_resample", u32), ("stochastic_spatial", u32),
                ("extra_disocclusion_sampling", u32), ("M_max", u32), ("alpha_min", f32)]


class SvgfParams(C.Structure):
    _fields_ = [("sigma_z", f32), ("k_n", f32), ("sigma_l", f32), ("radius", u32), ("num_passes", u32)]


class IndirectParams(C.Structure):
    _fields_ = [("max_non_tr_bounces", u32), ("max_glossy_tr_bounces", u32), ("russian_roulette", u32),
                ("temporal_resample", u32), ("num_spatial_passes", u32), ("M_max_temporal", u32),
                ("M_max_spatial", u32), ("boiling_suppression", u32), ("sort_temporal", u32),
                ("sort_spatial", u32), ("alpha_min", f32)]


class CompositingParams(C.Structure):
    _fields_ = [("emissive_di", u32), ("indirect", u32), ("firefly_filter", u32)]


class AutoExposureParams(C.Structure):
    _fields_ = [("min_lum", f32), ("max_lum", f32), ("lum_map_exp", f32), ("adaptation_rate", f32)]


class DisplayParams(C.Structure):
    _fields_ = [("tonemapper", u32), ("auto_exposure", u32), ("saturation", f32), ("agx_exp", f32)]


class GIParams(C.Structure):
    _fields_ = [("max_non_tr_bounces", u32), ("max_glossy_tr_bounces", u32), ("russian_roulette", u32), ("stochastic_multi_bounce", u32),
                ("boiling_suppression", u32), ("M_max", u32), ("temporal_resample", u32)]


class RendererDesc(C.Structure):
    _fields_ = [("width", u32), ("height", u32), ("with_tridiff", C.c_int), ("two_streams", C.c_int)]


# zr_halo_exchange_fn (include/zr_abi.h "Strip-sharded frames")
HALO_EXCHANGE_FN = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(Image2D), C.c_int, C.c_void_p)
# zr_reduce_u32_fn (include/zr_abi.h "AutoExposure")
REDUCE_U32_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p)


class CommTransport(C.Structure):
    """zr_comm_transport (include/zr_abi.h "Strip-sharded frames"): every callback returns a zr_status."""
    _fields_ = [("exchange_halos", C.CFUNCTYPE(i32, vp, C.c_int, C.POINTER(u32), u32, C.POINTER(Image2D), C.c_int, vp)),
                ("gather_rows", C.CFUNCTYPE(i32, vp, C.POINTER(u32), C.POINTER(Image2D), C.c_int, vp)),
                ("allreduce_u32", C.CFUNCTYPE(i32, vp, C.c_int, vp, u32, vp))]


# zr_alias_entry (RT::EmissiveLumenAliasTableEntry) as a numpy record
ALIAS_ENTRY = np.dtype([("CachedP_Orig", "<f4"), ("CachedP_Alias", "<f4"), ("P_Curr", "<f4"), ("Alias", "<u4")])


def check(status):
    if status != 0:
        raise ZRError("zr_status %d: %s" % (status, lib.zr_last_error().decode()))
