"""Reference arithmetic of ggml's CPU backend for K-quant weights against activation rows quantised to Q8_K (quantize_row_q8_K,
ggml-quants.c):
  Q3_K: an exact integer sumi = sum_j sc_j * sum_16 q_w q_x per super-block and (d_w d_x) * sumi accumulated in f32
        (ggml_vec_dot_q3_K_q8_K, ggml-cpu/quants.c:617).  The sums are formed per 32-value sub-block, as the device kernels do
        (two 16-value products combined with their scales).
  Q4_K / Q5_K: per 32-value sub-block j the exact integer sumi_j = sum q_w q_x (q_w unsigned) and the activation sum bsum_j; a super-block
        adds d_x (d sc_j sumi_j - dmin m_j bsum_j) (ggml_vec_dot_q4_K_q8_K / _q5_K_q8_K, ggml-cpu/quants.c); d sc_j and dmin m_j are exact
        in f32 (11-bit by 6-bit products).
Only the f32 summation order differs from the reference.

NumPy restatement plus ctypes taps into the compiled reference's CPU type traits (tests/test_q8_k_signed_cpu.py pins one to the other).
Test infrastructure only.
"""
import ctypes as C

import numpy as np

from q1_ref import _FROM_FLOAT, _VEC_DOT, RefCpu

Q3_K, Q4_K, Q5_K, Q8_K = 11, 12, 13, 15
BLOCK = {Q3_K: 110, Q4_K: 144, Q5_K: 176, Q8_K: 292}

_E = np.arange(256)
_N, _R, _L = _E >> 7, (_E >> 5) & 3, _E & 31


def _f16(b):
    return np.frombuffer(np.ascontiguousarray(b).tobytes(), dtype=np.float16).astype(np.float32)


def block_ints(wtype, raw):
    """Q3_K file super-blocks -> (signed q int64 [nb][256], integer scales int64 [nb][16], d [nb])"""
    blk = np.frombuffer(raw, dtype=np.uint8).reshape(-1, BLOCK[wtype]).astype(np.int64)
    lo = (blk[:, 32 + 32 * _N + _L] >> (2 * _R)) & 3
    h = (blk[:, _L] >> (4 * _N + _R)) & 1
    q = lo - np.where(h != 0, 0, 4)
    k, i = np.arange(16) >> 2, np.arange(16) & 3
    # the 12 scale bytes start at 96: low nibbles in bytes 96 .. 103, high bit pairs in 104 .. 107
    sc = (((blk[:, 96 + (k & 1) * 4 + i] >> (4 * (k >> 1))) & 0xF) | (((blk[:, 104 + i] >> (2 * k)) & 3) << 4)) - 32
    return q, sc, _f16(blk[:, 108:110].astype(np.uint8))


def block_ints_k4(wtype, raw):
    """Q4_K / Q5_K file super-blocks -> (unsigned q int64 [nb][256], sc int64 [nb][8], m int64 [nb][8], d [nb], dmin [nb]) (get_scale_min_k4)"""
    blk = np.frombuffer(raw, dtype=np.uint8).reshape(-1, BLOCK[wtype]).astype(np.int64)
    j = np.arange(8)
    lo = j < 4
    sc = np.where(lo, blk[:, 4 + (j & 3)] & 63, (blk[:, 8 + j] & 0xF) | ((blk[:, 4 + (j & 3)] >> 6) << 4))
    m = np.where(lo, blk[:, 4 + (j & 3) + 4] & 63, (blk[:, 8 + j] >> 4) | ((blk[:, 4 + (j & 3) + 4] >> 6) << 4))
    sj, sl = _E >> 5, _E & 31
    qoff = 16 + (32 if wtype == Q5_K else 0)
    q = (blk[:, qoff + 32 * (sj >> 1) + sl] >> (4 * (sj & 1))) & 0xF
    if wtype == Q5_K:
        q |= ((blk[:, 16 + sl] >> sj) & 1) << 4
    return q, sc, m, _f16(blk[:, 0:2].astype(np.uint8)), _f16(blk[:, 2:4].astype(np.uint8))


def dot_q8_k(wtype, raw, rows, k, xq, xd):
    """activation rows given as Q8_K ints xq [t][k] and scales xd [t][k / 256] against every weight row: (y float64 [t][rows] -- the
    reference's sum in exact arithmetic --, the sum of the terms' magnitudes [t][rows]).  Integer sums as f32 matrix products (exact)."""
    xq = np.asarray(xq, np.float32).reshape(-1, k)
    n_t = xq.shape[0]
    xs = np.repeat(np.asarray(xd, np.float64).reshape(n_t, k // 256), 8, axis=1)[:, None, :]         # [t][1][k / 32]
    if wtype == Q3_K:
        q, sc, wd = block_ints(wtype, raw)
        s16 = np.matmul(q.astype(np.float32).reshape(rows, k // 16, 16).transpose(1, 0, 2), xq.reshape(n_t, k // 16, 16).transpose(1, 2, 0))
        s = (s16.transpose(2, 1, 0).astype(np.float64) * sc.reshape(1, rows, k // 16)).reshape(n_t, rows, k // 32, 2).sum(axis=3)
        dd = (np.repeat(wd.reshape(rows, k // 256), 8, axis=1)[None] * np.asarray(xd, np.float32).reshape(n_t, 1, k // 256).repeat(8, axis=2)).astype(np.float32)
        t = dd.astype(np.float64) * s
        return t.sum(axis=2), np.abs(t).sum(axis=2)
    q, sc, m, d, dmin = block_ints_k4(wtype, raw)
    sumi = np.matmul(q.astype(np.float32).reshape(rows, k // 32, 32).transpose(1, 0, 2), xq.reshape(n_t, k // 32, 32).transpose(1, 2, 0))
    sumi = sumi.transpose(2, 1, 0).astype(np.float64)                                                   # [t][rows][k / 32]
    dl = (d[:, None] * sc).astype(np.float64).reshape(1, rows, k // 32)
    ml = (dmin[:, None] * m).astype(np.float64).reshape(1, rows, k // 32)
    bsum = xq.reshape(n_t, 1, k // 32, 32).sum(axis=3, dtype=np.float64)
    a, b = xs * dl * sumi, xs * ml * bsum
    return (a - b).sum(axis=2), (np.abs(a) + np.abs(b)).sum(axis=2)


def dequantize(wtype, raw, rows, k):
    """dequantize_row_q3_K: (d * sc) * q, each product rounded in f32"""
    q, sc, d = block_ints(wtype, raw)
    dl = (d[:, None] * np.repeat(sc, 16, axis=1).astype(np.float32)).astype(np.float32)
    return (dl * q.astype(np.float32)).astype(np.float32).reshape(rows, k)


def quantize_q8_k(x):
    """x: float32 [256 * nb] -> (q int64 [nb][256], d f32 [nb]) (quantize_row_q8_K: iscale = -127 / signed max, q = min(127, rint))"""
    x = np.asarray(x, np.float32).reshape(-1, 256)
    idx = np.abs(x).argmax(axis=1)
    mx = x[np.arange(x.shape[0]), idx]
    nz = mx != 0
    iscale = np.where(nz, np.float32(-127.0) / np.where(nz, mx, 1), 0).astype(np.float32)
    q = np.minimum(127, np.rint((iscale[:, None] * x).astype(np.float32))).astype(np.int64)
    d = np.where(nz, np.float32(1.0) / np.where(nz, iscale, 1), 0).astype(np.float32)
    return np.where(nz[:, None], q, 0), d


def q8_k_bytes(x):
    """block_q8_K records (f32 d, int8 qs[256], int16 bsums[16]) of quantize_q8_k(x)"""
    q, d = quantize_q8_k(x)
    out = np.empty((q.shape[0], 292), np.uint8)
    out[:, 0:4] = d.view(np.uint8).reshape(-1, 4)
    out[:, 4:260] = q.astype(np.int8).view(np.uint8)
    out[:, 260:] = q.reshape(-1, 16, 16).sum(axis=2).astype(np.int16).view(np.uint8).reshape(-1, 32)
    return out.tobytes()


def sumi32(wtype, raw, rows, k, xq):
    """exact integer sum_16 sc * q_w . q_x per 32-value sub-block: int64 [rows][k / 32] (the two-k16 combine of the kernels)"""
    q, sc, _ = block_ints(wtype, raw)
    p = (q.reshape(rows, k // 16, 16) * xq.reshape(1, k // 16, 16)).sum(axis=2) * sc.reshape(rows, k // 16)
    return p.reshape(rows, k // 32, 2).sum(axis=2)


def mul_mat_q(wtype, raw, rows, k, x):
    """y[t][n] as ggml's CPU mul_mat computes it for K-quant weights, up to the f32 summation order"""
    x = np.asarray(x, np.float32).reshape(-1, k)
    if wtype != Q3_K:
        return np.stack([dot_q8_k(wtype, raw, rows, k, *quantize_q8_k(x[t]))[0][0] for t in range(x.shape[0])]).astype(np.float32)
    _, _, wd = block_ints(wtype, raw)
    wd = wd.reshape(rows, k // 256)
    out = np.empty((x.shape[0], rows), np.float32)
    for t in range(x.shape[0]):
        xq, xd = quantize_q8_k(x[t])
        s = sumi32(wtype, raw, rows, k, xq).astype(np.float32)
        dd = np.repeat((wd * xd[None, :]).astype(np.float32), 8, axis=1)
        out[t] = (dd * s).astype(np.float32).sum(axis=1, dtype=np.float32)
    return out


class RefCpuK(RefCpu):
    """RefCpu for the 256-value activation type"""

    def quantize_act(self, wtype, x):
        x = np.ascontiguousarray(x, np.float32)
        vt = self._traits(wtype).vec_dot_type
        assert vt == Q8_K
        out = np.zeros(x.size // 256 * BLOCK[Q8_K], np.uint8)
        _FROM_FLOAT(self._traits(vt).from_float)(x.ctypes.data, out.ctypes.data, x.size)
        return out.tobytes()
