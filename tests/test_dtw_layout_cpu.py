"""CPU: the alignment-weight kernel (k_dtw_qk) reads the cross K in either layout.  The persistent decode kernel keeps cross K head-major
([layer][d/64][Tp][64]), the kernel chain token-major ([layer][Tp][d]); walked on the host (wb200_dbg_dtw_qk_layout), both layouts of the
same K must give bit-identical weights, and the token-major walk must equal wb200_dbg_dtw_qk."""
import ctypes as C

import numpy as np
import pytest

vp = C.c_void_p


def _head_major(k, d):
    """[L][Tp][d] -> [L][d/64][Tp][64]"""
    L, Tp, _ = k.shape
    return np.ascontiguousarray(k.reshape(L, Tp, d // 64, 64).transpose(0, 2, 1, 3))


@pytest.mark.parametrize("d,Tp,n_ctx,n_tok,heads", [
    (384, 1536, 1500, 7, [(0, 1, 4), (0, 1, 0), (1, 2, 5)]),               # heads of several layers, the full audio context
    (384, 1536, 768, 5, [(1, 2, 3), (0, 0, 5), (1, 2, 0)]),                # a reduced n_audio_ctx (whisper_full_params.audio_ctx)
    (1280, 1536, 1500, 3, [(0, 2, 19), (1, 3, 0), (1, 3, 7), (0, 2, 11)]),  # large-v3 width
])
def test_head_major_k_gives_identical_weights(lib, d, Tp, n_ctx, n_tok, heads):
    rng = np.random.default_rng(11)
    n_layers = 1 + max(h[1] for h in heads)
    n_sel = 1 + max(h[0] for h in heads)
    q = (rng.standard_normal((n_sel, n_tok, d)) * 3).astype(np.float32)
    k = (rng.standard_normal((n_layers, Tp, d)) * 0.5).astype(np.float16)
    kh = _head_major(k, d)
    tri = np.asarray(heads, np.int32)
    scale = C.c_float(float(np.float32(64.0) ** np.float32(-0.25)))
    lib.wb200_dbg_dtw_qk.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_float, vp]
    lib.wb200_dbg_dtw_qk_layout.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, vp]
    outs = [np.full((len(heads), n_ctx, n_tok), np.nan, np.float32) for _ in range(3)]
    assert lib.wb200_dbg_dtw_qk(q.ctypes.data, k.ctypes.data, Tp, d, tri.ctypes.data, len(heads), n_tok, n_ctx, scale, outs[0].ctypes.data) == 0
    assert lib.wb200_dbg_dtw_qk_layout(q.ctypes.data, k.ctypes.data, Tp, d, tri.ctypes.data, len(heads), n_tok, n_ctx, scale, 0, outs[1].ctypes.data) == 0
    assert lib.wb200_dbg_dtw_qk_layout(q.ctypes.data, kh.ctypes.data, Tp, d, tri.ctypes.data, len(heads), n_tok, n_ctx, scale, 1, outs[2].ctypes.data) == 0
    assert np.isfinite(outs[0]).all()
    assert outs[0].tobytes() == outs[1].tobytes()
    assert outs[0].tobytes() == outs[2].tobytes()
    assert np.allclose(outs[2].sum(axis=1), 1.0, atol=1e-5)
    # the keys beyond n_ctx are never read: changing them changes nothing
    kh2 = kh.copy(); kh2[:, :, n_ctx:, :] = np.float16(7.0)
    out3 = np.empty_like(outs[2])
    assert lib.wb200_dbg_dtw_qk_layout(q.ctypes.data, kh2.ctypes.data, Tp, d, tri.ctypes.data, len(heads), n_tok, n_ctx, scale, 1, out3.ctypes.data) == 0
    assert out3.tobytes() == outs[2].tobytes()
