"""The device's ReSTIR DI (GBufferRT -> PresampleEmissives -> DirectLighting, the real passes) against the independent float64
radiometric truth (oracle/indep_radiometry.py). Same statistics as tests/test_radiometry_oracle.py, with hundreds of frames per
replica. Every tile is compared in every RGB channel at a Student-t threshold that holds the file's family-wise false-alarm
rate to 1 %; the tiles that can detect a 1 % luminance bias must cover at least 60 % of the lit tiles, and together they must
resolve 0.25 % in each channel."""
import numpy as np
import pytest

from tests import radiometry_util as ru

W, H = 128, 72
REPLICAS, FRAMES, WARMUP = 48, 324, 4
TILE_BOUND, REGION_BOUND = 0.01, 0.0025
# every tile x channel and every region channel of the 12 DI cases is one comparison; a correct device fails one with
# probability <= ru.ALPHA
THRESHOLD = ru.threshold(REPLICAS, 12 * 3 * (ru.num_tiles(W, H) + 1))
DI_MODES = {"no_reuse": dict(temporal_resample=0, spatial_resample=0), "temporal": dict(temporal_resample=1, spatial_resample=0),
            "temporal_spatial": {}}


def _device_replicas(T, di_params, presample):
    from zetaray_b200.camera import FrameSequence
    from zetaray_b200.passes import download_image
    from tests.parity import DeviceFrame
    dev = DeviceFrame(T.flat, T.w, T.h, ("rdi",), di_params=di_params, presample=presample)
    out = []
    try:
        for r in range(REPLICAS):
            dev.di.ResetTemporal()
            seq = FrameSequence(T.w, T.h, jitter=False, first_frame=1 + 1000 * r)
            acc = np.zeros((T.w * T.h, 3))
            for f in range(FRAMES):
                dev.render(seq.next())
                if f >= WARMUP:
                    acc += download_image(dev.di.GetOutput(0), np.float32, 4)[:, :3]
            out.append(acc / (FRAMES - WARMUP))
    finally:
        dev.close()
    return np.array(out)


@pytest.mark.gpu
@pytest.mark.parametrize("sampling", ["alias", "presampled"])
@pytest.mark.parametrize("mode", list(DI_MODES))
@pytest.mark.parametrize("name", ["truth_a", "truth_b"])
def test_device_restir_di_matches_radiometric_truth(name, mode, sampling):
    T = ru.truth(name, W, H)
    reps = _device_replicas(T, DI_MODES[mode], (16, 64) if sampling == "presampled" else None)
    em = T.prim.emissive
    rel = (T.le[em] - reps[0][em]) / T.le[em]
    assert em.sum() >= 20 and (rel >= 0).all() and (rel[:, :2] <= 2.0 ** -6).all() and (rel[:, 2] <= 2.0 ** -5).all()
    s = ru.tile_stats(reps, T, THRESHOLD)
    region = ru.asserted_region(s, TILE_BOUND)
    ru.check(s, region, ru.region_stats(s, region, THRESHOLD), THRESHOLD, REGION_BOUND, "%s %s %s" % (name, mode, sampling))
