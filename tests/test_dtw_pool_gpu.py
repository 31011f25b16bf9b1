"""GPU: DTW token timestamps on the context's device pool and the persistent decode kernel.

A DTW context is an ordinary pool context: its states share encoder passes and decode launches with every other state of the context, and
the extra DTW pass of a window is one more decode request whose rows leave the alignment-head queries in a capture buffer (wb_dtw_kernel.cuh).
The transcript is scripted through logits_filter_callback (tests/test_full_scripted_cpu.py), so it is fixed whatever the random weights
compute; no_speech_thold = 2.0 keeps the no-speech rule out of it.  Asserted:
  * batch invariance: tokens, every t_dtw and the alignment weights of the last window are bit-identical whether a clip runs alone, next to
    seven others through concurrent whisper_full_with_state callers, whisper_full_parallel or wb200_full_batch -- with windows of more than
    64 text tokens, whose DTW pass spans two persistent-kernel passes;
  * the persistent kernel's weights against the kernel chain (WB200_MEGAKERNEL=0) and the reference at large-v3 width, F16 / Q5_0 / Q4_K;
  * DTW changes nothing else: tokens and segment times with DTW on equal those with DTW off, on the device sampler too.
"""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from wbtest import DATA_DIR, F16, Q4_K, Q5_0, FullParams, TokenData, bind_whisper_api, ref_quantize
from e2e_util import synth
from test_full_scripted_cpu import Script, LOG_CB, _quiet

pytestmark = pytest.mark.gpu
vp = C.c_void_p
SMALL = (51864, 1500, 384, 6, 1, 448, 384, 6, 3, 80)                   # 3 text layers, 6 heads; DTW heads: the last 2 layers (12 heads)
WIDE = (51865, 1500, 1280, 20, 2, 448, 1280, 20, 2, 80)               # large-v3 width: d = 1280, 20 heads; 2 + 2 layers (40 heads)


def _bind(L):
    bind_whisper_api(L)
    L.whisper_log_set.argtypes = [LOG_CB, vp]; L.whisper_log_set(_quiet, None)
    if hasattr(L, "wb200_last_error"):
        L.wb200_last_error.restype = C.c_char_p
        L.wb200_ctx_state.restype = vp; L.wb200_ctx_state.argtypes = [vp]
        L.wb200_dbg_last_dtw_qks.restype = C.c_int64; L.wb200_dbg_last_dtw_qks.argtypes = [vp, vp, C.c_int64, vp]
        L.wb200_full_batch.argtypes = [vp, FullParams, C.POINTER(vp), C.POINTER(C.c_int), C.c_int, C.POINTER(vp)]
    L.whisper_full_get_token_data_from_state.restype = TokenData; L.whisper_full_get_token_data_from_state.argtypes = [vp, C.c_int, C.c_int]
    return L


def _context(L, path, dtw=True, use_gpu=True):
    cp = L.whisper_context_default_params()
    cp.use_gpu = use_gpu
    if dtw:
        cp.flash_attn = False; cp.dtw_token_timestamps = True; cp.dtw_aheads_preset = 1; cp.dtw_n_top = 2
    ctx = L.whisper_init_from_file_with_params(path.encode(), cp)
    assert ctx, L.wb200_last_error() if use_gpu else "reference init failed"
    return ctx


def _params(L, script, language=b"en"):
    fp = L.whisper_full_default_params(0)
    fp.print_progress = False; fp.n_threads = 4; fp.no_speech_thold = 2.0; fp.greedy.best_of = 1; fp.temperature_inc = 0.0
    fp.language = language
    if script is not None:
        fp.logits_filter_callback = C.cast(script.cb, vp)
    return fp


def _result(L, st):
    """per segment: (t0, t1, [(id, t_dtw)])"""
    out = []
    for i in range(L.whisper_full_n_segments_from_state(st)):
        toks = [L.whisper_full_get_token_data_from_state(st, i, j) for j in range(L.whisper_full_n_tokens_from_state(st, i))]
        out.append((L.whisper_full_get_segment_t0_from_state(st, i), L.whisper_full_get_segment_t1_from_state(st, i), [(t.id, t.t_dtw) for t in toks]))
    return out


def _tokens(res):
    return [s[2] for s in res]


def _qks(L, st):
    shape = (C.c_int * 3)()
    n = L.wb200_dbg_last_dtw_qks(st, None, 0, shape)
    a = np.empty(n, np.float32)
    assert L.wb200_dbg_last_dtw_qks(st, a.ctypes.data, n, shape) == n
    return a, tuple(shape)


def _model(tmp_path, cfg, wt, seed, ref=None):
    stub = os.path.join(DATA_DIR, "for-tests-ggml-tiny.en.bin" if cfg[0] == 51864 else "for-tests-ggml-tiny.bin")
    path = str(tmp_path / f"m-{cfg[2]}-{wt}-{seed}.bin")
    synth.write_model(path, cfg, wt, seed=seed, vocab_from=stub, quantizer=(lambda t, w: ref_quantize(ref, t, w)) if ref is not None else None)
    return path


def test_dtw_pool_batch_invariance(lib, tmp_path):
    L = _bind(lib)
    path = _model(tmp_path, SMALL, Q5_0, 9)
    ctx = _context(L, path)
    try:
        secs = (30.0, 11.0, 47.0, 3.0, 21.5, 8.0, 30.0, 40.0)
        clips = [synth.synth_audio(seed=60 + i, seconds=s) for i, s in enumerate(secs)]
        script = Script(L, ctx, 77, "peaked")
        fp = _params(L, script)
        st0 = L.wb200_ctx_state(ctx)
        alone, alone_qk = [], []
        for c in clips:
            assert L.whisper_full(ctx, fp, c.ctypes.data_as(vp), len(c)) == 0, L.wb200_last_error()
            alone.append(_result(L, st0)); alone_qk.append(_qks(L, st0))
        eot = L.whisper_token_eot(ctx)
        text = [t for r in alone for s in r for t in s[2] if t[0] < eot]
        assert len(text) > 200 and all(t[1] >= 0 for t in text)                # every text token stamped
        assert max(q[1][0] for q in alone_qk) > 64                            # a DTW pass of more than one 64-row persistent pass
        # concurrent whisper_full_with_state callers
        states = [L.whisper_init_state(ctx) for _ in clips]
        assert all(states), L.wb200_last_error()
        rcs = [None] * len(clips)

        def work(i):
            rcs[i] = L.whisper_full_with_state(ctx, states[i], fp, clips[i].ctypes.data_as(vp), len(clips[i]))
        th = [threading.Thread(target=work, args=(i,)) for i in range(len(clips))]
        for t in th: t.start()
        for t in th: t.join()
        assert rcs == [0] * len(clips), L.wb200_last_error()
        assert [_result(L, s) for s in states] == alone
        for s, (a, shp) in zip(states, alone_qk):
            b, shb = _qks(L, s)
            assert shb == shp and b.tobytes() == a.tobytes()
        for s in states: L.whisper_free_state(s)
        # wb200_full_batch: result-only states carry t_dtw like the other token data
        n = len(clips)
        ptrs = (vp * n)(*[c.ctypes.data for c in clips]); lens = (C.c_int * n)(*[len(c) for c in clips]); outs = (vp * n)()
        assert L.wb200_full_batch(ctx, fp, ptrs, lens, n, outs) == 0, L.wb200_last_error()
        batched = [_result(L, outs[i]) for i in range(n)]
        for i in range(n): L.whisper_free_state(outs[i])
        assert [_tokens(r) for r in batched] == [_tokens(r) for r in alone]
        # whisper_full_parallel(8): every piece equals the same samples run alone (tokens and t_dtw; segment times are shifted by the split)
        pcm = synth.synth_audio(seed=91, seconds=8 * 33.0)
        per = len(pcm) // 8
        pieces = [pcm[i * per:(i + 1) * per] if i < 7 else pcm[7 * per:] for i in range(8)]
        want = []
        for p in pieces:
            p = np.ascontiguousarray(p)
            assert L.whisper_full(ctx, fp, p.ctypes.data_as(vp), len(p)) == 0
            want += _tokens(_result(L, st0))
        assert L.whisper_full_parallel(ctx, fp, pcm.ctypes.data_as(vp), len(pcm), 8) == 0, L.wb200_last_error()
        assert _tokens(_result(L, st0)) == want
    finally:
        L.whisper_free(ctx)


def _wide_run(L, path, script_seed, pcm, dtw=True):
    ctx = _context(L, path, dtw=dtw, use_gpu=hasattr(L, "wb200_last_error"))
    script = Script(L, ctx, script_seed, "peaked")
    fp = _params(L, script)
    assert L.whisper_full(ctx, fp, pcm.ctypes.data_as(vp), len(pcm)) == 0
    return ctx, script


@pytest.mark.parametrize("wt,tol_ref", [(F16, 2e-2), (Q5_0, 8e-2), (Q4_K, 8e-2)])
def test_dtw_persistent_kernel_against_chain_and_reference(lib, ref, tmp_path, wt, tol_ref):
    """large-v3 width: alignment weights of the persistent kernel vs the kernel chain (the decoder layout is chosen when the context is
    created: WB200_MEGAKERNEL=0 selects the chain) and vs the reference's aheads_cross_QKs; t_dtw is what the host DTW makes of them"""
    L = _bind(lib)
    path = _model(tmp_path, WIDE, wt, 13, ref)
    pcm = synth.synth_audio(seed=5, seconds=14.0)
    runs = {}
    for mode in ("1", "0"):
        os.environ["WB200_MEGAKERNEL"] = mode
        try:
            ctx, _ = _wide_run(L, path, 77, pcm)
        finally:
            os.environ.pop("WB200_MEGAKERNEL")
        st = L.wb200_ctx_state(ctx)
        runs[mode] = (_result(L, st), *_qks(L, st), L.whisper_n_len(ctx))
        L.whisper_free(ctx)
    (res_mk, a, shape, n_len), (res_ch, b, shape_ch, _) = runs["1"], runs["0"]
    assert [[t[0] for t in s] for s in _tokens(res_mk)] == [[t[0] for t in s] for s in _tokens(res_ch)]
    assert shape == shape_ch and shape[2] == 40
    err = float(np.sqrt(((a - b) ** 2).mean()) / np.sqrt((b ** 2).mean()))
    print("wt %d: alignment weights %s, persistent kernel vs chain relative rms %.2e" % (wt, shape, err))
    assert err < tol_ref / 2
    assert np.allclose(a.reshape(shape[2], shape[1], shape[0]).sum(axis=1), 1.0, atol=1e-4)
    # t_dtw of the persistent-kernel run is exactly what the host DTW makes of its weights (one window)
    lctx = _context(L, path)
    try:
        flat = [t for s in _tokens(res_mk) for t in s]
        ids = np.asarray([t[0] for t in flat], np.int32); sizes = np.asarray([len(s) for s in _tokens(res_mk)], np.int32)
        got = (C.c_int64 * len(ids))()
        L.wb200_dbg_dtw.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, vp]
        eot = L.whisper_token_eot(lctx)
        assert L.wb200_dbg_dtw(a.ctypes.data, shape[0], shape[1], shape[2], min(3000, n_len), 2, 0, eot, ids.ctypes.data, sizes.ctypes.data, len(sizes), got) > 0
        assert list(got) == [t[1] for t in flat]
    finally:
        L.whisper_free(lctx)
    # the reference, same model, transcript and alignment heads
    R = _bind(ref)
    rctx, _ = _wide_run(R, path, 77, pcm)
    try:
        assert [[t[0] for t in s] for s in _ref_tokens(R, rctx)] == [[t[0] for t in s] for s in _tokens(res_mk)]
        R.wref_ctx_state.restype = vp; R.wref_ctx_state.argtypes = [vp]
        R.wref_dtw_qks.restype = C.c_int64; R.wref_dtw_qks.argtypes = [vp, vp, C.c_int64, vp, vp, vp]
        nt, na, nh = C.c_int(), C.c_int(), C.c_int()
        m = R.wref_dtw_qks(R.wref_ctx_state(rctx), None, 0, C.byref(nt), C.byref(na), C.byref(nh))
        w = np.empty(m, np.float32)
        assert R.wref_dtw_qks(R.wref_ctx_state(rctx), w.ctypes.data, m, C.byref(nt), C.byref(na), C.byref(nh)) == m
        assert (nt.value, na.value, nh.value) == shape
        err_ref = float(np.sqrt(((a - w) ** 2).mean()) / np.sqrt((w ** 2).mean()))
        mine = np.asarray([t[1] for s in _tokens(res_mk) for t in s if t[0] < eot])
        theirs = np.asarray([t[1] for s in _ref_tokens(R, rctx) for t in s if t[0] < eot])
        d = np.abs(mine - theirs)
        print("wt %d: vs reference relative rms %.2e; t_dtw median |d| = %.0f cs, identical %d / %d" % (wt, err_ref, np.median(d), int((d == 0).sum()), len(d)))
        assert err_ref < tol_ref
    finally:
        R.whisper_free(rctx)


def _ref_tokens(R, ctx):
    return [[(t.id, t.t_dtw) for t in (R.whisper_full_get_token_data(ctx, i, j) for j in range(R.whisper_full_n_tokens(ctx, i)))]
            for i in range(R.whisper_full_n_segments(ctx))]


def test_dtw_changes_nothing_else(lib, tmp_path):
    """tokens and segment times with DTW on equal those with DTW off: scripted (host logits) and greedy on the device sampler, where a
    DTW pass rides on the other members' sampler configuration"""
    L = _bind(lib)
    path = _model(tmp_path, SMALL, Q5_0, 9)
    clips = [synth.synth_audio(seed=80 + i, seconds=s) for i, s in enumerate((30.0, 12.0, 45.0, 6.0, 30.0, 19.0, 33.0, 9.0))]
    n = len(clips)
    out = {}
    for dtw in (False, True):
        ctx = _context(L, path, dtw=dtw)
        try:
            script = Script(L, ctx, 78, "peaked")
            for mode, fp in (("scripted", _params(L, script)), ("device", _params(L, None))):
                ptrs = (vp * n)(*[c.ctypes.data for c in clips]); lens = (C.c_int * n)(*[len(c) for c in clips]); outs = (vp * n)()
                assert L.wb200_full_batch(ctx, fp, ptrs, lens, n, outs) == 0, L.wb200_last_error()
                res = [_result(L, outs[i]) for i in range(n)]
                for i in range(n): L.whisper_free_state(outs[i])
                out[(dtw, mode)] = [[(s[0], s[1], [t[0] for t in s[2]]) for s in r] for r in res]
                if dtw:
                    eot = L.whisper_token_eot(ctx)
                    assert all(t[1] >= 0 for r in res for s in r for t in s[2] if t[0] < eot)
        finally:
            L.whisper_free(ctx)
    for mode in ("scripted", "device"):
        assert sum(len(s[2]) for r in out[(False, mode)] for s in r) > 100
        assert out[(True, mode)] == out[(False, mode)], mode
