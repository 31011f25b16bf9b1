"""Every epilogue kind of the wgmma GEMM (whisper.cpp_b200/csrc/wb_gemm.cu) on ragged shapes, through the test hook wb200_dbg_gemm:
f16 token-major (QK), f16 GELU (FC1), f32 residual in place (attention-O / FC2), f16 m-major (V^T), f16 head-major (cross K/V) and the
general path (f32 out).  Same float64 reference and tolerances as test_gemm_gpu.py; N >= 6000 gives several tiles per persistent CTA.
"""
import numpy as np
import pytest

from test_gemm_gpu import run_gemm
from wbtest import F16, Q5_0, Q8_0, ref_quantize, ref_dequantize, gelu_ref_f16

pytestmark = pytest.mark.gpu

V2 = 4
GELU, MMAJOR, F16OUT, RES, HEADMAJOR = 1, 2, 16, 32, 64

CASES = [
    # wtype, M,    N,    K,    BN,  flags
    (Q5_0, 1280, 6007, 1280, 256, V2 | F16OUT),                  # QK kind
    (F16,  200,  77,   80,   64,  V2 | F16OUT),
    (Q5_0, 1280, 6007, 1280, 256, V2 | GELU | F16OUT),           # FC1 kind
    (F16,  330,  1001, 200,  128, V2 | GELU | F16OUT),
    (Q5_0, 1280, 6007, 1280, 256, V2 | RES),                     # attention-O / FC2 kind
    (F16,  330,  1001, 1000, 128, V2 | RES),
    (F16,  203,  333,  64,   64,  V2 | RES),
    (Q5_0, 1280, 6000, 1280, 256, V2 | MMAJOR | F16OUT),         # V^T kind
    (F16,  200,  1501, 200,  128, V2 | MMAJOR | F16OUT),
    (F16,  130,  77,   96,   64,  V2 | MMAJOR | F16OUT),
    (Q5_0, 1280, 6007, 1280, 256, V2 | F16OUT | HEADMAJOR),      # cross K/V head-major kind
    (F16,  320,  1501, 200,  128, V2 | F16OUT | HEADMAJOR),
    (Q8_0, 192,  77,   256,  64,  V2 | F16OUT | HEADMAJOR),
    (Q5_0, 1280, 6007, 1280, 256, V2),                           # general path (f32 token-major)
    (F16,  200,  1001, 200,  128, V2 | MMAJOR),                  # general path (f32 m-major)
    (Q5_0, 640,  1001, 640,  128, MMAJOR | F16OUT),              # first-generation launch, quantised weights: general path
    (Q5_0, 640,  1001, 640,  128, F16OUT | HEADMAJOR),
]


@pytest.mark.parametrize("wtype,M,N,K,BN,flags", CASES)
def test_gemm_epilogue_kinds(lib, ref, wtype, M, N, K, BN, flags):
    rng = np.random.default_rng(4321 + M + 7 * N + 13 * K + wtype + flags)
    w = (rng.standard_normal((M, K)) * 0.05).astype(np.float32)
    x = rng.standard_normal((N, K)).astype(np.float32)
    bias = rng.standard_normal(M).astype(np.float32)
    raw = ref_quantize(ref, wtype, w)
    wd = ref_dequantize(ref, wtype, raw, M, K).astype(np.float64)
    xh = x.astype(np.float16).astype(np.float64)
    want = xh @ wd.T + bias[None, :]
    if flags & GELU:
        want = gelu_ref_f16(want.astype(np.float32)).astype(np.float64)
    res = None
    if flags & RES:
        res = rng.standard_normal((N, M)).astype(np.float32)
        want = want + res.astype(np.float64)
    got = run_gemm(lib, wtype, raw, x, bias, M, N, K, BN, flags, res)
    if flags & F16OUT:
        want = want.astype(np.float32).astype(np.float16).astype(np.float64)
    if flags & MMAJOR:
        got = got.T
    scale = np.sqrt(K) * np.sqrt((wd ** 2).mean()) * np.sqrt((xh ** 2).mean())
    tol = (1e-4 if wtype == F16 else 2e-3) * scale + 1e-5
    if flags & GELU:
        tol += 2e-3 * np.abs(want).max()
    if flags & F16OUT:
        tol += 1e-3 * np.abs(want).max()
    err = np.abs(got - want).max()
    assert np.isfinite(got).all()
    assert err <= tol, f"max err {err:.3e} > tol {tol:.3e} (scale {scale:.3e})"
