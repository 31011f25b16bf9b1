"""Reference arithmetic of ggml's CPU backend for Q4_1 / Q5_1 weights: activation rows quantised to Q8_1, an integer dot per 32-value
block and the block minimum against the activation block's sum (ggml-cpu/ggml-cpu.c:249-270; quantize_row_q8_1 AVX2 form
ggml-cpu/arch/x86/quants.c:400-496; ggml_vec_dot_q4_1_q8_1 / _q5_1_q8_1 :859-912, :1222-1264).

NumPy restatement plus ctypes taps into the compiled reference's own CPU type traits (ggml_get_type_traits_cpu of oracle/_ref), which
tests/test_q8_1_cpu.py pins it against.  Test infrastructure only.
"""
import ctypes as C

import numpy as np

Q4_1, Q5_1, Q8_0, Q8_1 = 3, 7, 8, 9
BLOCK = {Q4_1: 20, Q5_1: 24, Q8_0: 34, Q8_1: 36}


def _f16(b):
    return np.frombuffer(np.ascontiguousarray(b).tobytes(), dtype=np.float16).astype(np.float32)


def quantize_q8_1(x):
    """x: float32 [..., 32 * nb] -> (q int32 [nb][32], d [nb], s [nb]); d and s are the f16 values of the block, as f32"""
    x = np.asarray(x, np.float32).reshape(-1, 32)
    amax = np.abs(x).max(axis=1)
    d = (amax / np.float32(127.0)).astype(np.float32)
    idv = np.where(amax != 0, np.float32(127.0) / np.where(amax != 0, amax, 1), 0).astype(np.float32)
    q = np.rint((x * idv[:, None]).astype(np.float32)).astype(np.int32)            # _MM_ROUND_NEAREST: ties to even
    s = (d * q.sum(axis=1).astype(np.float32)).astype(np.float32)                   # with the unrounded d
    return q, d.astype(np.float16).astype(np.float32), s.astype(np.float16).astype(np.float32)


def q8_1_bytes(x):
    """block_q8_1 records (ggml-common.h: f16 d, f16 s, int8 qs[32]) of quantize_q8_1(x)"""
    q, d, s = quantize_q8_1(x)
    out = np.empty((q.shape[0], 36), np.uint8)
    out[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(-1, 2)
    out[:, 2:4] = s.astype(np.float16).view(np.uint8).reshape(-1, 2)
    out[:, 4:] = q.astype(np.int8).view(np.uint8)
    return out.tobytes()


def block_ints(wtype, raw):
    """file blocks -> (unsigned q int32 [nb][32], d [nb], m [nb])"""
    blk = np.frombuffer(raw, dtype=np.uint8).reshape(-1, BLOCK[wtype])
    d, m = _f16(blk[:, 0:2]), _f16(blk[:, 2:4])
    if wtype == Q4_1:
        qs = blk[:, 4:20]
        return np.concatenate([(qs & 0xF).astype(np.int32), (qs >> 4).astype(np.int32)], axis=1), d, m
    qh = blk[:, 4:8].copy().view(np.uint32).reshape(-1, 1)
    bits = ((qh >> np.arange(32, dtype=np.uint32)[None, :]) & 1).astype(np.int32)
    qs = blk[:, 8:24]
    return np.concatenate([(qs & 0xF).astype(np.int32) | (bits[:, :16] << 4), (qs >> 4).astype(np.int32) | (bits[:, 16:] << 4)], axis=1), d, m


def dequantize(wtype, raw, rows, k):
    """dequantize_row_q4_1 / _q5_1 without contraction: q * d (rounded) + m (rounded), f32"""
    q, d, m = block_ints(wtype, raw)
    return ((q.astype(np.float32) * d[:, None]).astype(np.float32) + m[:, None]).astype(np.float32).reshape(rows, k)


def mul_mat_q(wtype, raw, rows, k, x):
    """y[t][n] as ggml's CPU mul_mat computes it for Q4_1 / Q5_1 weights: sum_b (d_w d_x) sumi_b + sum_b m_w s_x (f32 sums)"""
    x = np.asarray(x, np.float32).reshape(-1, k)
    wi, wd, wm = block_ints(wtype, raw)
    nb = k // 32
    wi = wi.reshape(rows, nb, 32); wd = wd.reshape(rows, nb); wm = wm.reshape(rows, nb)
    out = np.empty((x.shape[0], rows), np.float32)
    for t in range(x.shape[0]):
        xq, xd, xs = quantize_q8_1(x[t])
        sumi = np.einsum("nbk,bk->nb", wi, xq).astype(np.float32)
        acc = (sumi * (wd * xd[None, :]).astype(np.float32)).astype(np.float32).sum(axis=1, dtype=np.float32)
        out[t] = acc + (wm * xs[None, :]).astype(np.float32).sum(axis=1, dtype=np.float32)
    return out


class _Traits(C.Structure):
    _fields_ = [("from_float", C.c_void_p), ("vec_dot", C.c_void_p), ("vec_dot_type", C.c_int), ("nrows", C.c_int64)]


_FROM_FLOAT = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int64)
_VEC_DOT = C.CFUNCTYPE(None, C.c_int, C.POINTER(C.c_float), C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int)


class RefCpu:
    """the reference CPU backend's per-row arithmetic: from_float of a type's vec_dot_type, and its vec_dot"""

    def __init__(self, ref):
        ref.ggml_cpu_init()
        ref.ggml_get_type_traits_cpu.restype = C.POINTER(_Traits)
        ref.ggml_get_type_traits_cpu.argtypes = [C.c_int]
        self.ref = ref

    def _traits(self, t):
        return self.ref.ggml_get_type_traits_cpu(t).contents

    def quantize_act(self, wtype, x):
        """bytes the CPU backend writes for the activation row x in front of a matrix of type wtype"""
        x = np.ascontiguousarray(x, np.float32)
        vt = self._traits(wtype).vec_dot_type
        out = np.zeros(x.size // 32 * BLOCK[vt], np.uint8)
        _FROM_FLOAT(self._traits(vt).from_float)(x.ctypes.data, out.ctypes.data, x.size)
        return out.tobytes()

    def vec_dot(self, wtype, n, w_row, x_row):
        """type_traits_cpu[wtype].vec_dot of one weight row (file bytes) with the quantised activation row x_row"""
        s = C.c_float(0.0)
        w = np.frombuffer(w_row, np.uint8); xb = np.frombuffer(x_row, np.uint8)
        _VEC_DOT(self._traits(wtype).vec_dot)(n, C.byref(s), 0, w.ctypes.data, 0, xb.ctypes.data, 0, 1)
        return s.value
