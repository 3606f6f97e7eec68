"""Parity at the resolutions the numbers are quoted on (VERDICT r1, item 1c): the whole Cornell frame -- G-buffer, ReSTIR DI,
ReSTIR PT (temporal + spatial), compositing + firefly, TAA -- at 1920x1080 (BENCH configuration), and a ReSTIR GI sequence at
2560x1440 (the C4 frame size), device vs oracle, every buffer byte for byte. The oracle runs on all host cores here."""
import pytest

from tests.parity import WHOLE_FRAME, frame_parity

pytestmark = pytest.mark.gpu


def test_full_frame_pipeline_1080p():
    problems, R = frame_parity("cornell", 1920, 1080, 3, WHOLE_FRAME)
    assert not problems, "\n".join(problems)
    assert ((R.curr_reservoirs()["meta"] >> 4) & 0xf).max() >= 8        # spatial reuse ran (M reaches M_max_spatial)


def test_restir_pt_glossy_1080p():
    # k > 2 replay, case 3, metals and coat at the bench resolution (two frames: path generation, temporal + spatial reuse)
    problems, R = frame_parity("glossy", 1920, 1080, 2, ("rpt",))
    assert not problems, "\n".join(problems)


def test_restir_gi_1440p():
    problems, R = frame_parity("cornell", 2560, 1440, 3, ("rgi",))
    assert not problems, "\n".join(problems)
