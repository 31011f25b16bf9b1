"""wgmma GEMM (whisper.cpp_b200/csrc/wb_gemm.cu) against a float64 contraction of the reference-dequantised
weights (ggml-quants.c dequantize_row_*) and the f16-rounded activations the kernel consumes.

Tolerance: the kernel multiplies f16 operands exactly and accumulates in f32 on the tensor core, so the only
differences are (a) the f16 rounding of each dequantised weight (<= 2^-11 relative, absent for F16 weights) and
(b) f32 accumulation order.  Bound used: 2e-3 * sqrt(K) * rms(w) * rms(x) for quantised, 1e-4 scale for F16.
"""
import ctypes as C
import numpy as np
import pytest

from wbtest import F16, Q4_0, Q5_0, Q8_0, Q4_K, Q5_K, ref_quantize, ref_dequantize, gelu_ref_f16

pytestmark = pytest.mark.gpu


def run_gemm(lib, wtype, raw, x, bias, M, N, K, BN, flags, res=None):
    out = np.empty((M, N) if (flags & 2) else (N, M), dtype=np.float32)
    if flags & 32:
        out[:] = res
    rawb = np.frombuffer(raw, dtype=np.uint8)
    rc = lib.wb200_dbg_gemm(C.c_int(wtype), M, N, K, rawb.ctypes.data_as(C.c_void_p), x.ctypes.data_as(C.c_void_p),
                            bias.ctypes.data_as(C.c_void_p) if bias is not None else None,
                            out.ctypes.data_as(C.c_void_p), BN, flags)
    assert rc == 0, (rc, lib.wb200_last_error())
    return out


CASES = [
    # wtype, M,   N,    K,    BN, flags
    (F16,   128,  64,   64,   64,  0),
    (F16,   256,  200,  192,  128, 0),
    (F16,   384,  1500, 384,  256, 0),
    (F16,   200,  77,   80,   64,  1),     # ragged M/N/K (K tail zero-filled by TMA), gelu
    (F16,   128,  300,  128,  128, 2),     # m-major output
    (Q5_0,  128,  64,   64,   64,  0),
    (Q5_0,  384,  1500, 384,  256, 0),
    (Q5_0,  1280, 700,  1280, 256, 1),
    (Q4_0,  256,  333,  512,  128, 0),
    (Q8_0,  256,  333,  512,  128, 2),
    (Q4_K,  256,  300,  512,  128, 0),
    (Q5_K,  384,  1500, 1280, 256, 0),
    (Q5_0,  200,  50,   1280, 64,  0),     # ragged M with quantised rows
]


CASES_V2 = [(w, M, N, K, BN, f | 4) for (w, M, N, K, BN, f) in CASES] + [
    (Q5_0, 1280, 6000, 1280, 256, 4),      # 10 x 24 = 240 tiles on 132 persistent CTAs: several tiles per CTA
    (Q5_0, 2560, 3000, 1280, 256, 5),
    (F16,  640,  4500, 320,  128, 4),
]


CASES_CL2 = [(w, M, N, K, BN, f | 8) for (w, M, N, K, BN, f) in CASES_V2 if BN >= 128]     # CTA pairs + TMA multicast

# the two specialised epilogues of the encoder: FC1 (GELU, f16 rows out: flags 1 | 16) and attention-O / FC2 (x += W a on the f32 residual
# stream, in place: flag 32); second-generation kernel, with and without CTA pairs; ragged N so that partial tiles are covered
CASES_EPI = [(Q5_0, 1280, 2900, 1280, 256, 4 | 1 | 16), (F16, 384, 1500, 384, 128, 4 | 1 | 16), (Q5_0, 1280, 2900, 1280, 256, 4 | 8 | 1 | 16),
             (Q5_0, 1280, 2900, 1280, 256, 4 | 32), (F16, 384, 1500, 1536, 128, 4 | 32), (Q5_0, 1280, 2900, 1280, 256, 4 | 8 | 32), (Q8_0, 200, 77, 256, 64, 4 | 32)]


@pytest.mark.parametrize("wtype,M,N,K,BN,flags", CASES + CASES_V2 + CASES_CL2 + CASES_EPI)
def test_gemm_matches_dequantised_reference(lib, ref, wtype, M, N, K, BN, flags):
    rng = np.random.default_rng(1234 + M + 7 * N + 13 * K + wtype)
    w = (rng.standard_normal((M, K)) * 0.05).astype(np.float32)
    x = rng.standard_normal((N, K)).astype(np.float32)
    bias = rng.standard_normal(M).astype(np.float32)
    raw = ref_quantize(ref, wtype, w)
    wd = ref_dequantize(ref, wtype, raw, M, K).astype(np.float64)
    xh = x.astype(np.float16).astype(np.float64)
    want = xh @ wd.T + bias[None, :]
    if flags & 1:
        want = gelu_ref_f16(want.astype(np.float32)).astype(np.float64)
    res = None
    if flags & 32:
        res = rng.standard_normal((N, M)).astype(np.float32)
        want = want + res.astype(np.float64)
    got = run_gemm(lib, wtype, raw, x, bias, M, N, K, BN, flags, res)
    if flags & 16:
        want = want.astype(np.float32).astype(np.float16).astype(np.float64)
    if flags & 2:
        got = got.T
    scale = np.sqrt(K) * np.sqrt((wd ** 2).mean()) * np.sqrt((xh ** 2).mean())
    tol = (1e-4 if wtype == F16 else 2e-3) * scale + 1e-5
    if flags & 1:
        tol += 2e-3 * np.abs(want).max()   # one f16 ulp of the table-GELU output where rounding straddles
    if flags & 16:
        tol += 1e-3 * np.abs(want).max()   # f16 rounding of the output
    err = np.abs(got - want).max()
    assert np.isfinite(got).all()
    assert err <= tol, f"max err {err:.3e} > tol {tol:.3e} (scale {scale:.3e})"
