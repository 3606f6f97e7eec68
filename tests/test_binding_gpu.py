"""Pass wrappers on the device: SetParams reaches the native pass, a refused value leaves `params` as it was, and a pass the
renderer keeps across SetMethod / SetDenoiser / SetDisplay keeps one wrapper and the params set through it."""
import pytest

from zetaray_b200 import ZRError

pytestmark = pytest.mark.gpu
W, H = 64, 64


@pytest.fixture
def renderer():
    from zetaray_b200.passes import Scene, Renderer
    from tests import scene_util
    sc = Scene(scene_util.cornell())
    R = Renderer(sc, W, H)
    yield R
    R.close()
    sc.close()


def _refused(p, **bad):
    before = bytes(p.params)
    with pytest.raises(ZRError):
        p.SetParams(**bad)
    assert bytes(p.params) == before, "%s.params changed by refused values %s" % (type(p).__name__, bad)


def test_renderer_gi_params_reach_the_pass(renderer):
    R = renderer
    R.SetMethod(R.RESTIR_GI)
    R.gi.SetParams(M_max=7)
    assert R.gi.params.M_max == 7
    _refused(R.gi, M_max=0)                     # 1..2047
    _refused(R.gi, max_non_tr_bounces=9)        # 1..8
    assert R.gi.params.M_max == 7


def test_refused_params_leave_params_unchanged(renderer):
    from zetaray_b200.passes import DirectLighting, SVGF
    R = renderer
    R.SetDenoiser(True)
    for p, good, bad in ((DirectLighting(W, H), dict(M_max=12), dict(M_max=0)), (R.direct, dict(M_max=12), dict(M_max=0)),
                         (SVGF(W, H), dict(num_passes=3), dict(radius=3)), (R.svgf, dict(num_passes=3), dict(radius=3))):
        p.SetParams(**good)
        _refused(p, **bad)
        assert all(getattr(p.params, k) == v for k, v in good.items()), type(p).__name__


def test_renderer_keeps_one_wrapper_per_pass(renderer):
    from zetaray_b200.passes import Display
    R = renderer
    R.SetMethod(R.RESTIR_GI)
    gi = R.gi
    gi.SetParams(M_max=5)
    R.SetMethod(R.RESTIR_GI)
    R.SetMethod(R.PATH_TRACING)                 # the same native pass runs both integrators
    assert R.gi is gi and gi.params.M_max == 5

    R.SetDenoiser(True)
    svgf = R.svgf
    svgf.SetParams(num_passes=3)
    R.SetDenoiser(True)
    assert R.svgf is svgf and svgf.params.num_passes == 3

    R.SetDisplay(True)
    ae, disp = R.auto_exposure, R.display
    ae.SetParams(max_lum=2.0)
    disp.SetParams(tonemapper=Display.AGX_PUNCHY)
    R.SetDisplay(True)
    assert R.auto_exposure is ae and R.display is disp
    assert ae.params.max_lum == 2.0 and disp.params.tonemapper == Display.AGX_PUNCHY

    # a pass the renderer removes and creates again starts from its defaults, and so does its wrapper
    R.SetDenoiser(False)
    assert R.svgf is None
    R.SetDenoiser(True)
    assert R.svgf is not svgf and R.svgf.params.num_passes == 5
