"""CPU: the warping path of DTW token timestamps as the device computes it (k_dtw_norm, k_dtw_cost, k_dtw_sweep in wb_dtw_kernel.cu),
walked on the host phase by phase (wb200_dbg_dtw_path, device_walk = 1), must be exactly dtw_path's path (device_walk = 0): every token
index and every time index.  Inputs: the alignment weights the reference itself computed (oracle tap wref_dtw_qks) and generated weights
chosen to hit equalities (quantised levels: ties in the medians, the costs and the DTW comparisons), constant token columns (variance 0),
the smallest non-empty and the empty cases, the largest shapes (448 tokens, 1500 positions), a reduced audio context and 1 / 12 / 40 heads."""
import ctypes as C
import os

import numpy as np
import pytest

from wbtest import DATA_DIR, F16, bind_whisper_api, read_wav_f32
from e2e_util import synth
from test_full_scripted_cpu import Script, LOG_CB, _quiet

vp = C.c_void_p


class Ahead(C.Structure):
    _fields_ = [("n_text_layer", C.c_int), ("n_head", C.c_int)]


def paths(lib, qk, n_tok, n_ctx, n_heads, M, sot):
    """(dtw_path's path, the host walk's path) as (tok_idx, time_idx) arrays"""
    lib.wb200_dbg_dtw_path.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int]
    qk = np.ascontiguousarray(qk, np.float32)
    assert qk.size >= n_heads * n_ctx * n_tok
    cap = n_tok + M + 1
    out = []
    for walk in (0, 1):
        tok = np.full(cap, -9, np.int32); tim = np.full(cap, -9, np.int32)
        n = lib.wb200_dbg_dtw_path(qk.ctypes.data, n_tok, n_ctx, n_heads, M, sot, walk, tok.ctypes.data, tim.ctypes.data, cap)
        assert n >= 0, lib.wb200_last_error()
        out.append((tok[:n].copy(), tim[:n].copy()))
    return out


def assert_same_path(lib, qk, n_tok, n_ctx, n_heads, M, sot):
    (t0, j0), (t1, j1) = paths(lib, qk, n_tok, n_ctx, n_heads, M, sot)
    assert len(t0) == len(t1)
    assert np.array_equal(t0, t1) and np.array_equal(j0, j1), np.flatnonzero((t0 != t1) | (j0 != j1))[:8]
    return len(t0)


def weights(rng, n_heads, n_ctx, n_tok, kind="softmax", levels=4):
    """[n_heads][n_ctx][n_tok]: softmax over the audio positions of a band along the diagonal plus noise, or quantised levels"""
    if kind == "levels":
        return (rng.integers(0, levels, (n_heads, n_ctx, n_tok)) / float(levels)).astype(np.float32)
    pos = np.arange(n_ctx)[None, :, None]; tok = np.arange(n_tok)[None, None, :]
    logits = -((pos - tok * (n_ctx / max(n_tok, 1))) ** 2) / (2.0 * 40.0 ** 2) + rng.standard_normal((n_heads, n_ctx, n_tok)) * 2.0
    p = np.exp(logits - logits.max(axis=1, keepdims=True))
    return (p / p.sum(axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("preset", ["n_top_2", "n_top_1", "custom"])
def test_device_path_matches_host_on_reference_weights(lib, ref, tmp_path, preset):
    if not hasattr(ref, "wref_dtw_qks"):
        pytest.skip("oracle/_ref predates wref_dtw_qks (rebuild with make -C oracle)")
    R = bind_whisper_api(ref)
    R.whisper_log_set.argtypes = [LOG_CB, vp]; R.whisper_log_set(_quiet, None)
    path = str(tmp_path / "m.bin")
    synth.write_model(path, (51864, 1500, 384, 6, 1, 448, 384, 6, 3, 80), F16, seed=9, vocab_from=os.path.join(DATA_DIR, "for-tests-ggml-tiny.en.bin"))
    cp = R.whisper_context_default_params(); cp.use_gpu = False; cp.flash_attn = False; cp.dtw_token_timestamps = True
    keep = None
    if preset == "custom":
        keep = (Ahead * 5)(Ahead(2, 3), Ahead(0, 1), Ahead(1, 5), Ahead(2, 0), Ahead(1, 2))
        cp.dtw_aheads_preset = 2; cp.dtw_aheads.n_heads = 5; cp.dtw_aheads.heads = C.cast(keep, vp)
    else:
        cp.dtw_aheads_preset = 1; cp.dtw_n_top = int(preset[-1])
    ctx = R.whisper_init_from_file_with_params(path.encode(), cp)
    assert ctx
    try:
        pcm = np.ascontiguousarray(read_wav_f32(os.path.join(DATA_DIR, "jfk.wav")), np.float32)
        fp = R.whisper_full_default_params(0)
        fp.print_progress = False; fp.n_threads = 4; fp.no_speech_thold = 2.0; fp.greedy.best_of = 1; fp.temperature_inc = 0.0
        script = Script(R, ctx, 77, "peaked")
        fp.logits_filter_callback = C.cast(script.cb, vp)
        assert R.whisper_full(ctx, fp, pcm.ctypes.data_as(vp), len(pcm)) == 0
        R.wref_ctx_state.restype = vp; R.wref_ctx_state.argtypes = [vp]
        R.wref_dtw_qks.restype = C.c_int64; R.wref_dtw_qks.argtypes = [vp, vp, C.c_int64, vp, vp, vp]
        st = R.wref_ctx_state(ctx)
        nt, na, nh = C.c_int(), C.c_int(), C.c_int()
        n = R.wref_dtw_qks(st, None, 0, C.byref(nt), C.byref(na), C.byref(nh))
        qk = np.empty(n, np.float32)
        assert R.wref_dtw_qks(st, qk.ctypes.data, n, C.byref(nt), C.byref(na), C.byref(nh)) == n > 0
        R.whisper_n_len.argtypes = [vp]
        n_frames = min(3000, R.whisper_n_len(ctx))
    finally:
        R.whisper_free(ctx)
    assert assert_same_path(lib, qk, nt.value, na.value, nh.value, n_frames // 2, 1) > n_frames // 2


# (n_tokens, n_audio_ctx, n_heads, M, sot_len, kind)
CASES = [
    (40, 1500, 12, 700, 1, "softmax"),
    (40, 1500, 12, 700, 2, "levels"),                 # ties everywhere: medians, costs, DTW comparisons
    (33, 1500, 1, 300, 1, "levels2"),                 # two levels, one head: many equal costs
    (25, 1500, 12, 500, 2, "const"),                  # constant token columns: variance 0
    (3, 1500, 12, 8, 1, "softmax"),                   # N = 1, M = 8: the smallest non-empty path
    (4, 1500, 12, 7, 2, "softmax"),                   # M = 7: empty path
    (2, 1500, 12, 100, 1, "softmax"),                 # N = 0: empty path
    (448, 1536, 1, 1500, 1, "softmax"),               # the largest path: 446 rows x 1500 positions, M < n_audio_ctx
    (448, 1500, 12, 1499, 2, "levels"),
    (120, 768, 12, 384, 1, "softmax"),                # audio_ctx = 768
    (100, 768, 40, 768, 2, "levels"),                 # 40 heads (large-v3 width, 2 + 2 layers), M = n_audio_ctx
    (224, 1500, 40, 1500, 2, "softmax"),
    (9, 1500, 40, 1500, 1, "const"),                  # short text, long audio
]


@pytest.mark.parametrize("n_tok,n_ctx,n_heads,M,sot,kind", CASES)
def test_device_path_matches_host_on_generated_weights(lib, n_tok, n_ctx, n_heads, M, sot, kind):
    rng = np.random.default_rng(n_tok * 7919 + M * 31 + n_heads)
    if kind == "levels2":
        qk = weights(rng, n_heads, n_ctx, n_tok, "levels", levels=2)
    elif kind == "const":
        qk = weights(rng, n_heads, n_ctx, n_tok)
        cols = rng.random((n_heads, n_ctx)) < 0.3
        qk[cols] = np.float32(1.0 / n_ctx)
        qk[:, : min(M, 12), :] = np.float32(0.25)       # a run of constant columns longer than the median window
    else:
        qk = weights(rng, n_heads, n_ctx, n_tok, kind)
    n = assert_same_path(lib, qk, n_tok, n_ctx, n_heads, M, sot)
    N = n_tok - sot - 1
    if N <= 0 or M <= 7:
        assert n == 0
    else:
        assert max(N, M) <= n <= N + M


def test_device_path_rejects_what_it_cannot_hold(lib):
    """more audio positions than the weights have, or a trace that does not fit the sweep's shared memory, is an error, not a wrong path"""
    lib.wb200_dbg_dtw_path.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int]
    qk = np.zeros(12 * 768 * 20, np.float32)
    tok = np.empty(4096, np.int32); tim = np.empty(4096, np.int32)
    assert lib.wb200_dbg_dtw_path(qk.ctypes.data, 20, 768, 12, 769, 1, 1, tok.ctypes.data, tim.ctypes.data, 4096) == -1
    big = np.zeros(1 * 4000 * 700, np.float32)
    assert lib.wb200_dbg_dtw_path(big.ctypes.data, 700, 4000, 1, 3000, 1, 1, tok.ctypes.data, tim.ctypes.data, 4096) == -1
    assert b"too large" in lib.wb200_last_error()
