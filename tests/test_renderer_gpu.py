"""zr_renderer (the native frame driver) produces byte-identical frames to the passes driven one by one -- which the
other GPU tests compare with the oracle -- including the frame-1 pre-lighting protocol, presampling and the second stream."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("which,presample,two_streams", [("glossy", None, True), ("glass", (16, 64), True), ("cornell", None, False)])
def test_renderer_matches_manual_sequence(which, presample, two_streams):
    from zetaray_b200 import lib, check
    from zetaray_b200.passes import Scene, Renderer
    from tests import scene_util, rpt_util
    from tests.parity import WHOLE_FRAME, DeviceFrame, pt_reservoirs, uint32x2
    w, h = 320, 180
    flat = scene_util.SCENES[which]()
    manual = DeviceFrame(flat, w, h, WHOLE_FRAME, rpt_params=dict(M_max_temporal=9), presample=presample)
    # renderer on its own scene object (it runs pre-lighting itself in its first frame)
    sc2 = Scene(flat)
    if presample:
        sc2.set_presampling(*presample)
    R = Renderer(sc2, w, h, two_streams=two_streams)
    R.indirect.SetParams(M_max_temporal=9)
    seq = rpt_util.FrameSequence(w, h, cam_path=lambda f: (0.02 * f, 1.2, -4.043))
    for fr in range(4):
        fc = seq.next()
        manual.render(fc)
        R.Render(fc)
        check(lib.zr_stream_synchronize(None))
        assert uint32x2(manual.taa.GetOutput()).tobytes() == uint32x2(R.GetOutput()).tobytes(), \
            "frame %d: renderer output differs from the manual pass sequence" % fr
        assert pt_reservoirs(manual.rpt.GetOutput(1)).tobytes() == pt_reservoirs(R.indirect.GetOutput(1)).tobytes()
    assert lib.zr_renderer_render(R.handle, None, None) != 0
    manual.close()
