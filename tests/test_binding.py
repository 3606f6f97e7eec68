"""The ctypes binding against include/zr_abi.h (no GPU): every entry point's types come from its prototype, and every struct
mirror has the header's layout as the system C compiler lays it out."""
import ctypes as C
import os
import subprocess
import sys

import pytest

from zetaray_b200 import _lib, ZRError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MIRRORS = {
    "zr_frame_constants": _lib.FrameConstants, "zr_gbuffer": _lib.GBuffer, "zr_frame_inputs": _lib.FrameInputs,
    "zr_image2d": _lib.Image2D, "zr_scene_desc": _lib.SceneDesc, "zr_renderer_desc": _lib.RendererDesc,
    "zr_direct_params": _lib.DirectParams, "zr_indirect_params": _lib.IndirectParams, "zr_gi_params": _lib.GIParams,
    "zr_compositing_params": _lib.CompositingParams, "zr_svgf_params": _lib.SvgfParams,
    "zr_auto_exposure_params": _lib.AutoExposureParams, "zr_display_params": _lib.DisplayParams,
    "zr_comm_transport": _lib.CommTransport,
}


def test_every_entry_point_is_declared_from_its_prototype():
    protos = _lib.prototypes()
    assert sorted(protos) == _lib.declared_symbols() and len(protos) > 100
    for name, (restype, argtypes) in protos.items():
        f = getattr(_lib.lib, name)
        assert f.restype is restype and list(f.argtypes) == argtypes, name
    vp, u32 = C.c_void_p, C.c_uint32
    spot = {
        "zr_last_error": (C.c_char_p, []),
        "zr_abi_version": (u32, []),
        "zr_kernel_launch_count": (C.c_uint64, []),
        "zr_scene_destroy": (None, [vp]),
        "zr_memcpy_d2h": (C.c_int32, [vp, vp, C.c_size_t, vp]),
        "zr_bvh_build_host": (C.c_int32, [vp, u32, vp, u32, vp, vp]),
        "zr_scene_set_light_voxel_grid": (C.c_int32, [vp, vp, vp, C.c_float]),
        "zr_gi_pass_set_method": (C.c_int32, [vp, C.c_int]),
        "zr_direct_pass_get_output": (C.c_int32, [vp, C.c_int, vp]),
        "zr_auto_exposure_pass_set_reduce": (C.c_int32, [vp, vp, vp]),
        "zr_renderer_set_display": (C.c_int32, [vp, C.c_int, vp, vp]),
    }
    for name, want in spot.items():
        assert protos[name] == want, name


def test_declared_types_refuse_wrong_arguments_before_the_call():
    lib = _lib.lib
    with pytest.raises(C.ArgumentError):
        lib.zr_gi_pass_set_method(None, C.c_uint32(1))          # int parameter, uint32_t value
    with pytest.raises(C.ArgumentError):
        lib.zr_scene_set_presampling(None, 1.5, 2)               # float for a uint32_t
    with pytest.raises(TypeError):
        lib.zr_memcpy_d2h(None, None)                            # too few arguments


def test_a_type_outside_the_map_fails_the_declaration():
    hdr = "typedef enum zr_mode { ZR_MODE_A = 0 } zr_mode;\ntypedef void (*zr_fn)(void* user);\n"
    ok = _lib.prototypes(hdr + "ZR_API zr_status zr_fake_set(zr_fake* p, zr_mode m, zr_fn fn,\n    const float v[3], size_t n);")
    assert ok == {"zr_fake_set": (C.c_int32, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t])}
    for decl, what in (("ZR_API zr_status zr_fake_scale(zr_fake* p, double s);", "double s"),
                       ("ZR_API int16_t zr_fake_count(void);", "int16_t"),
                       ("ZR_API zr_status zr_fake_set(zr_fake* p, zr_other_mode m);", "zr_other_mode m")):
        with pytest.raises(ZRError, match=what) as e:
            _lib.prototypes(hdr + decl)
        assert "zr_fake_" in str(e.value)


def test_struct_mirrors_match_the_c_layout(tmp_path):
    """sizeof and every field's offset and size, from a C program built against the header, against each ctypes mirror and
    against the alias-entry record dtype."""
    mirrored = {v for v in vars(_lib).values() if isinstance(v, type) and issubclass(v, C.Structure)}
    assert mirrored == set(MIRRORS.values())
    lines = ['printf("%s sizeof %%zu 0\\n", sizeof(%s));' % (t, t) for t in list(MIRRORS) + ["zr_alias_entry"]]
    fields = [(t, f) for t, cls in MIRRORS.items() for f, *_ in cls._fields_] + [("zr_alias_entry", f) for f in _lib.ALIAS_ENTRY.names]
    lines += ['printf("%s %s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s*)0)->%s));' % (t, f, t, f, t, f) for t, f in fields]
    src = tmp_path / "layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"zr_abi.h\"\nint main(void)\n{\n%s\n    return 0;\n}\n"
                   % "\n".join("    " + s for s in lines))
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    c = {(t, f): (int(off), int(size)) for t, f, off, size in (line.split() for line in out.splitlines())}
    for t, cls in MIRRORS.items():
        assert C.sizeof(cls) == c[t, "sizeof"][0], t
        for f, *_ in cls._fields_:
            assert (getattr(cls, f).offset, getattr(cls, f).size) == c[t, f], (t, f)
    assert _lib.ALIAS_ENTRY.itemsize == c["zr_alias_entry", "sizeof"][0]
    for f in _lib.ALIAS_ENTRY.names:
        dt, off = _lib.ALIAS_ENTRY.fields[f][:2]
        assert (off, dt.itemsize) == c["zr_alias_entry", f], f


def test_comm_transport_refuses_missing_callbacks_and_bad_rank():
    """zr_comm_create_transport checks its arguments on the host: all three callbacks, 0 <= rank < world. A comm it makes
    needs neither NCCL nor a GPU, and at world 1 every exchange returns before reaching the transport."""
    from zetaray_b200.passes import Comm
    lib = _lib.lib
    called = []
    fns = [lambda *a: called.append(a) or 0 for _ in range(3)]
    fields = [ftype(fn) for (_, ftype), fn in zip(_lib.CommTransport._fields_, fns)]
    h = C.c_void_p()
    for i in range(3):
        t = _lib.CommTransport(*fields)
        setattr(t, _lib.CommTransport._fields_[i][0], _lib.CommTransport._fields_[i][1]())      # a NULL callback
        assert lib.zr_comm_create_transport(C.byref(t), None, 0, 2, C.byref(h)) == 1
        assert b"zr_comm_create_transport" in lib.zr_last_error()
    t = _lib.CommTransport(*fields)
    for rank, world in ((-1, 2), (2, 2), (3, 2), (0, 0)):
        assert lib.zr_comm_create_transport(C.byref(t), None, rank, world, C.byref(h)) == 1, (rank, world)
    assert lib.zr_comm_create_transport(None, None, 0, 1, C.byref(h)) == 1
    assert lib.zr_comm_create_transport(C.byref(t), None, 0, 1, None) == 1
    comm = Comm.from_transport(*fns, 0, 1)
    bounds = (C.c_uint32 * 2)(0, 64)
    img = _lib.Image2D(None, 8, 64, 32, 4)
    assert lib.zr_comm_exchange_halos(comm.handle, 0, bounds, 32, C.byref(img), 1, None) == 0
    assert lib.zr_comm_gather_rows(comm.handle, bounds, C.byref(img), 0, None) == 0
    assert lib.zr_comm_allreduce_u32(comm.handle, 0, C.byref(C.c_uint32()), 1, None) == 0
    assert lib.zr_comm_exchange_halos(comm.handle, 2, bounds, 32, C.byref(img), 1, None) == 1      # which_comm out of range
    assert comm.stats() == (0, 0) and not called
    comm.close()


def test_structs_only_import_does_not_map_the_library(tmp_path):
    """ZETARAY_B200_STRUCTS_ONLY=1 imports the binding without the shared library (here: one that does not exist); a call
    through `lib` then raises ZRError."""
    code = ("import zetaray_b200.passes\n"
            "from zetaray_b200 import lib, ZRError\n"
            "try:\n"
            "    lib.zr_abi_version()\n"
            "except ZRError as e:\n"
            "    print('ZRError:', e)\n")
    env = dict(os.environ, ZETARAY_B200_STRUCTS_ONLY="1", ZETARAY_B200_LIB=str(tmp_path / "missing.so"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stdout.startswith("ZRError:") and "zr_abi_version" in r.stdout, r.stdout
