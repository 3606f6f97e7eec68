"""The ctypes bindings of the test libraries (no GPU): the oracle (oracle/liborc.so), the host builds of the device source
(tests/hostsim) and, where they were built, the reference wrappers (oracle/_ref). Every exported function is declared in the
library's header and gets its types from that prototype; every struct mirror has the header's layout as the system C compiler
lays it out."""
import ctypes as C
import os
import re
import subprocess

import pytest

from tests import hostsim, orc

vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float

MIRRORS = {"orc_surface_desc": orc.SurfaceDesc, "orc_rpt_buffers": orc.RptBuffers, "hostsim_scene": hostsim.Scene}
HEADERS = (orc.HEADER, hostsim.HEADER, *orc.REF_HEADERS.values())


def exported(so, prefix):
    out = subprocess.run(["nm", "-D", "--defined-only", so], check=True, capture_output=True, text=True).stdout
    return {line.split()[-1] for line in out.splitlines() if line.split()[-1].startswith(prefix)}


def assert_declared(dll, protos):
    for name, (restype, argtypes) in protos.items():
        f = getattr(dll, name)
        assert f.restype is restype and list(f.argtypes) == argtypes, name


def test_oracle_declares_every_export_from_its_prototype():
    protos = orc.prototypes()
    assert set(protos) == exported(orc.build(), "orc_") and len(protos) >= 70
    assert_declared(orc.load(), protos)
    spot = {
        "orc_scene_create": (vp, [vp, vp, vp, u32, vp, vp, vp, u32, vp]),
        "orc_alias_sample": (None, [vp, C.c_int64, C.c_uint64, C.c_int, vp, vp]),
        "orc_alias_build_emissive": (None, [vp, C.c_int64, C.c_int, vp]),
        "orc_kahan_sum": (f32, [vp, C.c_int64, C.c_int]),
        "orc_pcg": (u32, [u32]),
        "orc_display_view": (None, [vp, vp, vp, u32, u32, u32, u32, f32, f32, vp]),
        "orc_rgi_render": (None, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int]),
    }
    for name, want in spot.items():
        assert protos[name] == want, name


def test_hostsim_libraries_declare_every_export_from_its_prototype():
    protos = hostsim.prototypes()
    hostsim.build()
    libs = {hostsim.SO: hostsim.load(), hostsim.SO_DI: hostsim.load_di(), hostsim.SO_IO: hostsim.load_io()}
    names = set()
    for so, dll in libs.items():
        mine = exported(so, "hostsim_")
        assert mine <= set(protos), (so, mine - set(protos))
        assert_declared(dll, {n: protos[n] for n in mine})
        names |= mine
    assert names == set(protos)
    spot = {
        "hostsim_pack_half2": (u32, [f32, f32]),
        "hostsim_validate": (C.c_uint64, [vp, u32, vp, u32, vp]),
        "hostsim_bsdf_sampler_pdf": (f32, [vp, vp, u32]),
        "hostsim_oct32_round_trip": (C.c_uint64, [C.c_int, vp]),
        "hostsim_trace": (C.c_int, [vp, vp, vp, vp, vp, u32, vp, vp, vp, C.c_int]),
    }
    for name, want in spot.items():
        assert protos[name] == want, name


@pytest.mark.parametrize("name", sorted(orc.REF_HEADERS))
def test_reference_wrappers_declare_every_export_from_its_prototype(name):
    so = os.path.join(orc.ORACLE_DIR, "_ref", name)
    if not os.path.exists(so):
        pytest.skip("oracle/_ref/%s is built only where the reference tree is present" % name)
    protos = orc.prototypes(orc.REF_HEADERS[name], "REF_API", "ref_")
    assert set(protos) == exported(so, "ref_")
    assert_declared(orc.load_ref() if name == "libref_alias.so" else orc.load_ref_scene(), protos)
    spot = {"ref_kahan_sum": (f32, [vp, C.c_int64]), "ref_alias_sample": (None, [vp, C.c_int64, C.c_uint64, C.c_int, vp, vp]),
            "ref_half": (C.c_uint16, [f32]), "ref_frame_constants_offset": (C.c_int, [vp])}
    for f, want in spot.items():
        if f in protos:
            assert protos[f] == want, f


def test_declared_types_refuse_wrong_arguments_before_the_call():
    o = orc.load()
    with pytest.raises(C.ArgumentError):
        o.orc_pcg(1.5)                                           # float for a uint32_t
    one = C.c_uint32(1)
    with pytest.raises(C.ArgumentError):
        o.orc_halton(one, 2)                                     # c_uint32 for an int
    with pytest.raises(C.ArgumentError):
        o.orc_pack_snorm16x2(0.5, "0.5")                         # str for a float
    with pytest.raises(TypeError):
        o.orc_alias_sample(None, 4, 1)                           # too few arguments
    hs = hostsim.load()
    with pytest.raises(C.ArgumentError):
        hs.hostsim_pack_half2(1.0, None)                         # None for a float
    with pytest.raises(C.ArgumentError):
        hs.hostsim_set_rho_lut(1.5)                              # float for a pointer


def test_struct_mirrors_match_the_c_layout(tmp_path):
    """sizeof and every field's offset and size, from a C program built against the headers, against each ctypes mirror; and the
    mirrors are exactly the structs the headers define."""
    defined = set()
    for h in HEADERS:
        with open(h) as f:
            defined |= set(re.findall(r"typedef\s+struct\s+\w+\s*\{[^}]*\}\s*(\w+)\s*;", f.read()))
    assert defined == set(MIRRORS)
    lines = ['printf("%s sizeof %%zu 0\\n", sizeof(%s));' % (t, t) for t in MIRRORS]
    fields = [(t, f) for t, cls in MIRRORS.items() for f, *_ in cls._fields_]
    lines += ['printf("%s %s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s*)0)->%s));' % (t, f, t, f, t, f) for t, f in fields]
    src = tmp_path / "layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"hostsim_api.h\"\nint main(void)\n{\n%s\n    return 0;\n}\n"
                   % "\n".join("    " + s for s in lines))
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.dirname(hostsim.HEADER), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    c = {(t, f): (int(off), int(size)) for t, f, off, size in (line.split() for line in out.splitlines())}
    for t, cls in MIRRORS.items():
        assert C.sizeof(cls) == c[t, "sizeof"][0], t
        for f, *_ in cls._fields_:
            assert (getattr(cls, f).offset, getattr(cls, f).size) == c[t, f], (t, f)
