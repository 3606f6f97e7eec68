"""Material-feature builds of the lighting kernels: the scene's feature mask (clear coat, transmission, thin-walled over its material
table) and the build the passes pick from it. The Cornell box uses none of the features, so the other tests that render it run the
plain build; here one material of it at a time gets one feature, which must select the full build -- the plain one has no code for
that lobe, so the frames would differ from the oracle."""
import ctypes as C
import pytest

from tests.parity import WHOLE_FRAME, frame_parity

COAT, TRANSMISSION, THIN_WALLED = 0x1, 0x2, 0x4     # ZR_MATERIAL_* (include/zr_abi.h)


def _cornell_with(index, **material):
    def make():
        from tests import scene_util
        from zetaray_b200 import scene as zscene
        s = scene_util.cornell()
        m = s.materials.copy()
        m[index] = zscene.make_material(**material)
        s.materials = m
        return s
    return make


# index 3: back wall, 7: short box
CHANGED = {
    "cornell_coated": (COAT, _cornell_with(3, base_color=(0.2, 0.3, 0.7, 1), roughness=0.6, coat_weight=1.0, coat_roughness=0.1,
                                           coat_color=(0.9, 0.9, 0.9), double_sided=True)),
    "cornell_transmissive": (TRANSMISSION, _cornell_with(7, base_color=(0.6, 0.85, 0.7, 1), roughness=0.3, ior=1.33, transmission=1.0,
                                                         transmission_depth=0.5, double_sided=True)),
    "cornell_thin_walled": (THIN_WALLED, _cornell_with(3, base_color=(0.8, 0.7, 0.5, 1), roughness=0.5, thin_walled=True, subsurface=0.6,
                                                       double_sided=True)),
}
# fields of those features that leave the material plain: a coat roughness without coat weight, a thin-walled flag without
# subsurface weight
PLAIN = {
    "cornell": None,
    "cornell_coat_roughness_only": _cornell_with(3, base_color=(0.2, 0.3, 0.7, 1), roughness=0.6, coat_roughness=0.4, double_sided=True),
    "cornell_thin_walled_no_subsurface": _cornell_with(3, base_color=(0.8, 0.7, 0.5, 1), roughness=0.5, thin_walled=True, double_sided=True),
}


def _features(flat):
    from zetaray_b200 import lib, check
    from zetaray_b200.passes import Scene
    sc = Scene(flat)
    out = C.c_uint32(0xffffffff)
    check(lib.zr_scene_material_features(sc.handle, C.byref(out)))
    return out.value


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PLAIN))
def test_plain_scenes_have_no_features(name):
    from tests import scene_util
    flat = (PLAIN[name] or scene_util.cornell)()
    assert _features(flat) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CHANGED))
def test_one_material_sets_its_feature(name):
    bit, make = CHANGED[name]
    assert _features(make()) == bit


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CHANGED))
def test_one_material_frames_match_the_oracle(name):
    # ReSTIR DI, ReSTIR PT (path generation, temporal and spatial reuse), compositing and TAA, bit-exact, 3 frames
    problems, _ = frame_parity(CHANGED[name][1](), 256, 144, 3, WHOLE_FRAME)
    assert not problems, "\n".join(problems)
