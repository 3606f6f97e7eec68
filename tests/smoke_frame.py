"""smoke(): three small frames of the whole hot path on cuda:0, checked bit-exactly against the CPU oracle."""


def run():
    from tests.parity import WHOLE_FRAME, frame_parity
    problems, _ = frame_parity("glossy", 160, 90, 3, WHOLE_FRAME)
    assert not problems, "\n".join(problems)
    print("smoke frames ok (G-buffer -> ReSTIR DI -> ReSTIR PT -> compositing/firefly -> TAA, 160x90 x 3 frames, bit-exact vs oracle)")
