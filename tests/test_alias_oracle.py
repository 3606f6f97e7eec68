"""C1 -- alias-table correctness on the host (reference: Tests/TestAliasTable.cpp:14-121).

Pins oracle/orc_alias.cpp against (a) the golden vector of SURVEY 8c, (b) the outputs of the reference's own code
(oracle/_ref/libref_alias.so) stored in tests/golden/reference_alias.npz by tools/make_reference_golden.py (bit-exact,
including the pointer-alignment dependence of KahanSum), and re-states the reference's three doctest cases with fixed seeds."""
import hashlib
import os
import numpy as np
import pytest
from tests.orc import ptr
from zetaray_b200._lib import ALIAS_ENTRY

GOLDEN_REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_alias.npz")
REF_SIZES = [1, 2, 6, 17, 50, 999, 13107, 100000]
REF_PROLOGUES = [0, 3]
REF_FULL_TABLE_MAX_N = 999      # larger tables are stored as their SHA-256
RNG_STREAMS = (0xda3e39cb94b95bdb, 1, 12345)

ENTRY = np.dtype([("P_Curr", "<f4"), ("P_Orig", "<f4"), ("Alias", "<u4")])
GOLDEN_W = np.array([1, 22, 4, 8, 3.5, 10], dtype=np.float32)
GOLDEN = [
    (0.12371134, 0.0206185579, 1), (1.0, 0.453608245, 1), (0.494845361, 0.0824742317, 1),
    (0.989690721, 0.164948463, 1), (0.432989687, 0.0721649528, 5), (0.670103073, 0.206185564, 1)]


def aligned(n, dtype=np.float32, offset_elems=0):
    raw = np.zeros(n * np.dtype(dtype).itemsize + 64 + 4 * 8, dtype=np.uint8)
    # offset_elems = number of leading elements before the next 32-byte boundary ("prologue")
    off = (-raw.ctypes.data) % 32 + 4 * ((8 - offset_elems) % 8)
    return raw[off:off + n * np.dtype(dtype).itemsize].view(dtype)


def orc_build(o, w, prologue=0):
    w = w.astype(np.float32).copy()
    t = np.zeros(len(w), dtype=ENTRY)
    o.orc_alias_build(ptr(w), len(w), prologue, ptr(t))
    return t, w


def ref_build(r, w, prologue=0):
    buf = aligned(len(w), np.float32, prologue)
    buf[:] = w
    t = np.zeros(len(w), dtype=ENTRY)
    r.ref_alias_build(ptr(buf), len(w), ptr(t))
    return t, buf.copy()


def test_golden_vector(oracle):
    t, _ = orc_build(oracle, GOLDEN_W)
    for i, (pc, po, al) in enumerate(GOLDEN):
        assert t["Alias"][i] == al
        assert abs(t["P_Curr"][i] - pc) < 1e-7
        assert abs(t["P_Orig"][i] - po) < 1e-8
    idx = np.zeros(5, dtype=np.uint32)
    pdf = np.zeros(5, dtype=np.float32)
    oracle.orc_alias_sample(ptr(t), 6, 12345, 5, ptr(idx), ptr(pdf))
    assert idx.tolist() == [1, 1, 5, 5, 5]


def test_normalize(oracle):
    # TestAliasTable.cpp:14-28
    w = GOLDEN_W.copy()
    oracle.orc_alias_normalize(ptr(w), 6, 0)
    s = np.float32(0)
    for e in w:
        s = np.float32(s + e)
    assert abs(float(s) - 6.0) < 1e-7 * 6 + 1e-6


@pytest.mark.parametrize("seed", [1, 12345, 0xda3e39cb94b95bdb])
def test_returned_pdf_matches_original(oracle, seed):
    # TestAliasTable.cpp:30-67 with fixed seeds
    n_buf = np.zeros(1, dtype=np.uint32)
    oracle.orc_rng64_stream(seed, 2, 999, 1, ptr(n_buf), None)
    n = 1 + int(n_buf[0])
    f = np.zeros(n + 1, dtype=np.float32)
    oracle.orc_rng64_stream(seed + 7, 1, 0, n, None, ptr(f))
    vals = (f[:n] * np.float32(100.0)).astype(np.float32)
    s = oracle.orc_kahan_sum(ptr(vals), n, 0)
    normalized = vals / np.float32(s)
    t, _ = orc_build(oracle, vals)
    idx = np.zeros(100, dtype=np.uint32)
    pdf = np.zeros(100, dtype=np.float32)
    oracle.orc_alias_sample(ptr(t), n, seed, 100, ptr(idx), ptr(pdf))
    assert (idx < n).all()
    assert np.abs(pdf - normalized[idx]).max() < 1e-7


@pytest.mark.parametrize("seed", [3, 99, 2024])
def test_density_chi_squared(oracle, seed):
    # TestAliasTable.cpp:69-121
    n = 50
    u = np.zeros(n, dtype=np.uint32)
    oracle.orc_rng64_stream(seed, 2, 1000, n, ptr(u), None)
    vals = u.astype(np.float32)
    s = oracle.orc_kahan_sum(ptr(vals), n, 0)
    normalized = vals / np.float32(s)
    t, _ = orc_build(oracle, vals)
    idx = np.zeros(100, dtype=np.uint32)
    pdf = np.zeros(100, dtype=np.float32)
    oracle.orc_alias_sample(ptr(t), n, seed * 31 + 1, 100, ptr(idx), ptr(pdf))
    count = np.bincount(idx, minlength=n).astype(np.float64)
    expected = normalized.astype(np.float64) * 100
    chi = np.where(expected == 0, 0, (count - expected) ** 2 / np.where(expected == 0, 1, expected)).sum()
    assert chi <= 124.34211340400407


def ref_case_weights(n, prologue):
    rng = np.random.default_rng(n * 7 + prologue)
    w = (rng.random(n, dtype=np.float32) * np.float32(100.0)).astype(np.float32)
    if n > 10:
        w[rng.integers(0, n, size=n // 10)] = 0.0      # dead emitters
    return w


def reference_alias_outputs(reflib):
    """What the reference's own code returns for the cases below; tools/make_reference_golden.py stores it."""
    out = {}
    for n in REF_SIZES:
        for prologue in REF_PROLOGUES:
            if prologue and n < prologue + 16:
                continue
            w = ref_case_weights(n, prologue)
            buf = aligned(n, np.float32, prologue)
            buf[:] = w
            key = "n%d_p%d" % (n, prologue)
            out[key + "_kahan"] = np.float32(reflib.ref_kahan_sum(ptr(buf), n))
            t, _ = ref_build(reflib, w, prologue)
            out[key + "_table"] = t if n <= REF_FULL_TABLE_MAX_N else np.array(hashlib.sha256(t.tobytes()).hexdigest())
            idx = np.zeros(200, dtype=np.uint32); pdf = np.zeros(200, dtype=np.float32)
            reflib.ref_alias_sample(ptr(t), n, 12345, 200, ptr(idx), ptr(pdf))
            out[key + "_idx"], out[key + "_pdf"] = idx, pdf
    for sid in RNG_STREAMS:
        a = np.zeros(64, dtype=np.uint32)
        reflib.ref_rng_stream(sid, 0, 0, 64, ptr(a), None)
        out["rng_%x" % sid] = a
    out["halton"] = np.array([[reflib.ref_halton(i, base) for base in (2, 3)] for i in range(1, 70)], dtype=np.float32)
    return out


@pytest.fixture(scope="module")
def golden_ref():
    with np.load(GOLDEN_REF) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("n", REF_SIZES)
@pytest.mark.parametrize("prologue", REF_PROLOGUES)
def test_bit_exact_vs_reference(oracle, golden_ref, n, prologue):
    if n < prologue + 16:
        # the reference's alignment prologue does not bound-check N (Common.cpp:82-90): with an
        # unaligned pointer and a short span it reads past the data -- undefined, nothing to pin
        if prologue:
            pytest.skip("reference reads out of bounds for short unaligned spans")
    w = ref_case_weights(n, prologue)
    key = "n%d_p%d" % (n, prologue)
    ks_orc = oracle.orc_kahan_sum(ptr(w.copy()), n, prologue)
    assert golden_ref[key + "_kahan"].tobytes() == np.float32(ks_orc).tobytes()
    t_orc, w_orc = orc_build(oracle, w, prologue)
    t_ref = golden_ref[key + "_table"]
    if t_ref.dtype.kind == "U":
        assert hashlib.sha256(t_orc.tobytes()).hexdigest() == str(t_ref)
    else:
        assert (t_ref["Alias"] == t_orc["Alias"]).all()
        assert t_ref["P_Curr"].tobytes() == t_orc["P_Curr"].tobytes()
        assert t_ref["P_Orig"].tobytes() == t_orc["P_Orig"].tobytes()
    idx_o = np.zeros(200, dtype=np.uint32); pdf_o = np.zeros(200, dtype=np.float32)
    oracle.orc_alias_sample(ptr(t_orc), n, 12345, 200, ptr(idx_o), ptr(pdf_o))
    assert (golden_ref[key + "_idx"] == idx_o).all() and golden_ref[key + "_pdf"].tobytes() == pdf_o.tobytes()


def test_rng_and_halton_vs_reference(oracle, golden_ref):
    for sid in RNG_STREAMS:
        b = np.zeros(64, dtype=np.uint32)
        oracle.orc_rng64_stream(sid, 0, 0, 64, ptr(b), None)
        assert (golden_ref["rng_%x" % sid] == b).all()
    for i in range(1, 70):
        for j, base in enumerate((2, 3)):
            assert golden_ref["halton"][i - 1, j].tobytes() == np.float32(oracle.orc_halton(i, base)).tobytes()


def test_emissive_table_consistent_with_twin(oracle):
    n = 777
    rng = np.random.default_rng(5)
    w = (rng.random(n, dtype=np.float32) * 50).astype(np.float32)
    t, _ = orc_build(oracle, w)
    e = np.zeros(n, dtype=ALIAS_ENTRY)
    ww = w.copy()
    oracle.orc_alias_build_emissive(ptr(ww), n, 0, ptr(e))
    assert (e["Alias"] == t["Alias"]).all()
    assert e["P_Curr"].tobytes() == t["P_Curr"].tobytes()
    assert e["CachedP_Orig"].tobytes() == t["P_Orig"].tobytes()
    assert (e["CachedP_Alias"] == t["P_Orig"][t["Alias"]]).all()
