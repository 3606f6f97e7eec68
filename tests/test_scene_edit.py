"""Material edits between frames on the host (zetaray_b200.scene.update_materials, the FlatScene form of zr_scene_update_materials):
an edited scene holds the bytes SceneBuilder emits when it is built with the edited materials from the start, and the edits the
library refuses are the ones after which SceneBuilder would emit a different set of emissive triangles."""
import numpy as np
import pytest

from tests import scene_util
from zetaray_b200 import scene as zscene


def rebuild(flat, materials):
    """(materials, emissive triangles, BaseEmissiveTriOffset per instance) that SceneBuilder emits for flat's geometry and
    instances with `materials` (SceneBuilder._emit_emissives per instance, in instance order, as add_mesh / add_instance_of call it)."""
    b = zscene.SceneBuilder()
    for m in materials:
        b.add_material(m)
    offsets = []
    for k, (inst, nt) in enumerate(zip(flat.instances, flat.instance_num_tris)):
        inst = inst.copy()
        bi = int(inst["BaseIdxOffset"]); bv = int(inst["BaseVtxOffset"])
        idx = flat.indices[bi:bi + 3 * int(nt)]
        verts = flat.vertices[bv:bv + int(idx.max()) + 1]
        b._emit_emissives(inst, int(inst["MatIdx"]), verts["pos"], verts["uv"], idx, k)
        offsets.append(int(inst["BaseEmissiveTriOffset"]))
    em = np.concatenate(b.em) if b.em else np.zeros(0, dtype=zscene.EMISSIVE_TRI)
    return np.array(b.mats, dtype=zscene.MATERIAL), em, np.array(offsets, dtype=np.uint32)


_CACHE = {}


def _scene(name):
    if name not in _CACHE:
        _CACHE[name] = scene_util.cornell() if name == "cornell" else scene_util.atrium_small()
    return _CACHE[name]


def _lights(flat):
    return sorted({int(i["MatIdx"]) for i in flat.instances if int(i["BaseEmissiveTriOffset"]) != 0xffffffff})


def _random_material(rng, emissive):
    """A random material; an emissive one keeps a non-zero factor (a factor of zero takes a light out of what SceneBuilder emits,
    while the library keeps its triangles with zero power)."""
    ef = (0, 0, 0)
    if emissive:
        ef = tuple(rng.random(3))
        ef = (max(ef[0], 0.05),) + ef[1:]
    return zscene.make_material(base_color=tuple(rng.random(3)) + (1.0,), metallic=float(rng.random() > 0.7),
                                roughness=float(rng.random()), ior=1.0 + 1.5 * float(rng.random()),
                                transmission=float(rng.random() > 0.8), emissive_factor=ef,
                                emissive_strength=float(rng.choice([0.0, 0.5, 1.0, 7.25, 40.0, 1000.0])) if emissive else 1.0,
                                coat_weight=float(rng.random() > 0.6) * float(rng.random()), double_sided=bool(rng.random() > 0.5),
                                thin_walled=bool(rng.random() > 0.8), subsurface=float(rng.random()))


@pytest.mark.parametrize("name", ["cornell", "atrium"])
@pytest.mark.parametrize("seed", range(6))
def test_edit_equals_scene_built_with_edited_materials(name, seed):
    """A random edit of a random material range: the edited FlatScene's materials and emissive triangles are byte-identical to
    SceneBuilder's output for the edited material table, and so is the unedited scene's rebuild (the rebuild is SceneBuilder's)."""
    flat = _scene(name)
    rng = np.random.default_rng(seed * 7 + len(name))
    lights = set(_lights(flat))
    n = len(flat.materials)
    first = int(rng.integers(0, n))
    count = int(rng.integers(1, n - first + 1))
    edit = [_random_material(rng, emissive=(first + k) in lights) for k in range(count)]
    if seed == 0:       # the light alone: colour, strength and double-sided flag
        first, count = min(lights), 1
        edit = [_random_material(rng, emissive=True)]
    try:
        got = zscene.update_materials(flat, first, edit)
    except ValueError as e:
        # the only refusal random edits of lights can meet: every light off at once
        assert "zero emissive factor or strength" in str(e)
        assert all(int(m["EmissiveStrength_IOR"]) & 0x7fff == 0 for k, m in enumerate(edit) if first + k in lights)
        return
    m0, e0, _ = rebuild(flat, flat.materials)
    assert e0.tobytes() == flat.emissives.tobytes(), "the rebuild does not reproduce the scene's own emissive triangles"
    mats = flat.materials.copy()
    mats[first:first + count] = edit
    want_m, want_e, want_off = rebuild(flat, mats)
    assert got.materials.tobytes() == want_m.tobytes()
    assert np.array_equal(want_off, flat.instances["BaseEmissiveTriOffset"])
    assert got.emissives.tobytes() == want_e.tobytes()
    assert got.instances is flat.instances and got.vertices is flat.vertices and got.indices is flat.indices


@pytest.mark.parametrize("name", ["cornell", "atrium"])
def test_refused_lights_are_the_ones_scene_builder_would_add(name):
    """Giving a material an emissive factor is refused exactly when SceneBuilder, built with the edit, emits emissive triangles for
    an instance that has none; a material no instance uses may become emissive."""
    base = _scene(name)
    flat = zscene.FlatScene()
    flat.vertices, flat.indices, flat.instances, flat.instance_num_tris, flat.emissives = (
        base.vertices, base.indices, base.instances, base.instance_num_tris, base.emissives)
    flat.materials = np.concatenate([base.materials, zscene.make_material()[None]])       # one unused material
    lights = set(_lights(flat))
    for k in range(len(flat.materials)):
        if k in lights:
            continue
        lit = zscene.make_material(emissive_factor=(0.3, 0.2, 0.1), emissive_strength=5.0)
        mats = flat.materials.copy()
        mats[k] = lit
        _, want_e, want_off = rebuild(flat, mats)
        changes_set = not np.array_equal(want_off, flat.instances["BaseEmissiveTriOffset"])
        try:
            got = zscene.update_materials(flat, k, [lit])
            refused = False
        except ValueError as e:
            assert "has no emissive triangles" in str(e)
            refused = True
        assert refused == changes_set, k
        if not refused:
            assert got.emissives.tobytes() == want_e.tobytes()


def test_refusals():
    """The other refusals: an empty or out-of-range edit, and switching every light off (zero strength, or zero factor)."""
    flat = scene_util.cornell()
    light = _lights(flat)[0]
    for first, mats in ((0, []), (len(flat.materials), [flat.materials[0]]), (len(flat.materials) - 1, flat.materials[:2])):
        with pytest.raises(ValueError):
            zscene.update_materials(flat, first, mats)
    for off in (zscene.make_material(emissive_factor=(0.5, 0.5, 0.5), emissive_strength=0.0),
                zscene.make_material(emissive_factor=(0.5, 0.5, 0.5), emissive_strength=-0.0),
                zscene.make_material(emissive_factor=(0, 0, 0), emissive_strength=3.0)):
        with pytest.raises(ValueError, match="zero emissive factor or strength"):
            zscene.update_materials(flat, light, [off])
    # a factor of zero on a light is not a refusal while another light keeps power; its triangles stay, with factor 0
    atrium = _scene("atrium")
    lights = _lights(atrium)
    got = zscene.update_materials(atrium, lights[0], [zscene.make_material()])
    assert len(got.emissives) == len(atrium.emissives)
    inst = atrium.instances[atrium.instances["MatIdx"] == lights[0]][0]
    assert int(got.emissives[int(inst["BaseEmissiveTriOffset"])]["PackedA"]) & 0xffffff == 0
