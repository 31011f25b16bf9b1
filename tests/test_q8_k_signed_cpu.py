"""CPU: the NumPy statement of the reference's Q3_K / Q4_K / Q5_K x Q8_K arithmetic (tests/kq_signed_ref.py) against the compiled
reference's own from_float and vec_dot, and synth's plain Q3_K writer against the reference's dequantize_row_q3_K."""
import numpy as np
import pytest

import kq_signed_ref as kq
from wbtest import load_ref, ref_dequantize, ref_quantize
from e2e_util import synth

WTS = [kq.Q3_K]
DOT_WTS = [kq.Q3_K, kq.Q4_K, kq.Q5_K]


@pytest.fixture(scope="module")
def cpu():
    return kq.RefCpuK(load_ref())


def _matrix(rng, rows, k):
    w = (rng.standard_normal((rows, k)) * 0.05).astype(np.float32)
    w[0, :256] = 0.0                                            # an all-zero super-block
    if rows > 2:
        w[1] *= np.float32(1e3)                                 # an outlier row
    return w


def _extreme_scales(wt, raw, rows):
    """set the integer scales of row 2 (Q4_K / Q5_K: and row 3) to the extremes of the format: Q3_K -32 and 31; Q4_K / Q5_K 6-bit scales
    and minimums at 63 / 0 (row 2) and 0 / 63 (row 3)"""
    blk = np.frombuffer(raw, np.uint8).reshape(rows, -1, kq.BLOCK[wt]).copy()
    if wt == kq.Q3_K:
        blk[2, :, 96:108] = np.array([0x00, 0xFF] * 6, np.uint8)   # stored 0 / 63 patterns: sc - 32 = -32 and 31 mixed
    else:                                                          # get_scale_min_k4 of scales[12] = bytes 4 .. 15
        blk[2, :, 4:16] = np.array([0xFF] * 4 + [0x00] * 4 + [0x0F] * 4, np.uint8)
        blk[3, :, 4:16] = np.array([0x00] * 4 + [0xFF] * 4 + [0xF0] * 4, np.uint8)
    return blk.tobytes()


@pytest.mark.parametrize("wt", WTS)
def test_q8_k_rows_match_reference_bytes(cpu, wt):
    rng = np.random.default_rng(4)
    x = (rng.standard_normal(256 * 6) * 0.3).astype(np.float32)
    x[:256] = 0.0
    x[300] = 40.0; x[700] = -40.0
    assert kq.q8_k_bytes(x) == cpu.quantize_act(wt, x)


@pytest.mark.parametrize("wt", DOT_WTS)
@pytest.mark.parametrize("k", [256, 512, 1280, 5120])
def test_vec_dot_matches_reference(cpu, wt, k):
    """one dot per row against type_traits_cpu[wt].vec_dot: equal up to the f32 summation order (the integer sums are exact), both the
    exact statement dot_q8_k and mul_mat_q; the activation rows hold a zero super-block"""
    ref = cpu.ref
    rng = np.random.default_rng(k + wt)
    rows = 6
    raw = _extreme_scales(wt, ref_quantize(ref, wt, _matrix(rng, rows, k)), rows)
    x = rng.standard_normal((2, k)).astype(np.float32)
    x[1, :256] = 0.0
    got = kq.mul_mat_q(wt, raw, rows, k, x)
    row = kq.BLOCK[wt] * (k // 256)
    for t in range(2):
        xb = cpu.quantize_act(wt, x[t])
        xq, xd = kq.quantize_q8_k(x[t])
        if wt == kq.Q3_K:
            assert np.abs(kq.sumi32(wt, raw, rows, k, xq)).max() < 2 ** 24     # the two-k16 combine is exact in f32
        exact, mag = (v[0] for v in kq.dot_q8_k(wt, raw, rows, k, xq, xd))
        for n in range(rows):
            want = cpu.vec_dot(wt, k, raw[n * row:(n + 1) * row], xb)
            assert abs(exact[n] - want) <= 1e-6 * mag[n] + 1e-30, (t, n, exact[n], want)
            assert abs(got[t, n] - want) <= 1e-6 * mag[n] + 1e-30, (t, n, got[t, n], want)


@pytest.mark.parametrize("wt", WTS)
def test_numpy_dequantize_matches_reference(wt):
    ref = load_ref()
    rng = np.random.default_rng(wt)
    w = _matrix(rng, 8, 1280)
    raw = _extreme_scales(wt, ref_quantize(ref, wt, w), 8)
    assert np.array_equal(kq.dequantize(wt, raw, 8, 1280).view(np.uint32), ref_dequantize(ref, wt, raw, 8, 1280).view(np.uint32))


@pytest.mark.parametrize("wt", WTS)
def test_simple_writers_dequantise_close_to_input(wt):
    """synth's plain writers produce valid super-blocks: the reference's dequantize_row_* gives back the input within the format's step"""
    ref = load_ref()
    rng = np.random.default_rng(7)
    w = (rng.standard_normal((16, 1024)) * 0.05).astype(np.float32)
    w[3, :256] = 0.0
    raw = synth.quantize(wt, w)
    assert len(raw) == 16 * 4 * kq.BLOCK[wt]
    back = ref_dequantize(ref, wt, raw, 16, 1024)
    assert np.array_equal(back, kq.dequantize(wt, raw, 16, 1024))
    rel = np.sqrt(((back - w) ** 2).mean() / (w ** 2).mean())
    assert rel < 0.3, rel
    assert not back[3, :256].any()
