"""GPU: the warping path of DTW token timestamps computed on the device (k_dtw_norm, k_dtw_cost, k_dtw_sweep; wb_dtw_kernel.cuh).

  * one launch of mixed requests (token counts, audio positions M, n_audio_ctx, head counts, empty paths): every path equals dtw_path's
    bit for bit, and equals the same request launched alone;
  * end to end, scripted transcripts (tests/test_full_scripted_cpu.py, no_speech_thold = 2.0): every DTW window's t_dtw equals what the host
    DTW (wb200_dbg_dtw: dtw_path + dtw_assign) makes of that window's alignment weights (wb200_dbg_last_dtw_qks), through whisper_full,
    8 concurrent whisper_full_with_state callers, whisper_full_parallel and wb200_full_batch, windows of more than 64 text tokens,
    audio_ctx = 768, the persistent kernel and the kernel chain, at the SMALL and WIDE shapes of test_dtw_pool_gpu.py.  A window's weights
    are read from inside the logits callback of the next window's first step, when the state's last DTW pass is that window's;
  * a DTW run adds GPU time to the device DTW counter (wb200_counters[11]).
"""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from wbtest import Q5_0
from e2e_util import synth
from test_full_scripted_cpu import Script
from test_dtw_pool_gpu import SMALL, WIDE, _bind, _context, _params, _result, _tokens, _qks, _model
from test_dtw_device_cpu import weights

pytestmark = pytest.mark.gpu
vp = C.c_void_p


def _device_paths(L, reqs):
    """reqs: [(qk, n_tok, n_ctx, n_heads, M, sot)] -> [(tok_idx, time_idx)] from one launch of each kernel"""
    L.wb200_dbg_dtw_path_device.argtypes = [C.c_int, vp, C.c_int64, vp, vp, C.c_int, vp, vp, vp, vp]
    w = np.ascontiguousarray(np.concatenate([np.asarray(r[0], np.float32).ravel() for r in reqs]))
    w_off = np.cumsum([0] + [r[0].size for r in reqs[:-1]]).astype(np.int64)
    req = np.asarray([r[1:] for r in reqs], np.int32).ravel()
    caps = [r[1] + r[4] for r in reqs]
    out_off = np.cumsum([0] + caps[:-1]).astype(np.int64)
    tok = np.full(sum(caps) + 1, -9, np.int32); tim = np.full(sum(caps) + 1, -9, np.int32); ln = np.full(len(reqs), -1, np.int32)
    assert L.wb200_dbg_dtw_path_device(0, w.ctypes.data, w.size, w_off.ctypes.data, req.ctypes.data, len(reqs), tok.ctypes.data, tim.ctypes.data,
                                       out_off.ctypes.data, ln.ctypes.data) == 0, L.wb200_last_error()
    return [(tok[o:o + n].copy(), tim[o:o + n].copy()) for o, n in zip(out_off, ln)]


def _host_path(L, qk, n_tok, n_ctx, n_heads, M, sot):
    L.wb200_dbg_dtw_path.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int]
    cap = n_tok + M + 1
    tok = np.empty(cap, np.int32); tim = np.empty(cap, np.int32)
    n = L.wb200_dbg_dtw_path(np.ascontiguousarray(qk, np.float32).ctypes.data, n_tok, n_ctx, n_heads, M, sot, 0, tok.ctypes.data, tim.ctypes.data, cap)
    assert n >= 0, L.wb200_last_error()
    return tok[:n].copy(), tim[:n].copy()


def test_device_paths_mixed_batch_one_launch(lib):
    L = _bind(lib)
    rng = np.random.default_rng(17)
    shapes = [(60, 1500, 12, 700, 1, "softmax"), (448, 1536, 1, 1500, 1, "softmax"), (120, 768, 40, 384, 2, "levels"), (4, 1500, 12, 7, 2, "softmax"),
              (3, 1500, 12, 8, 1, "softmax"), (224, 1500, 40, 1500, 2, "softmax"), (25, 768, 12, 768, 2, "levels"), (447, 1500, 10, 1500, 2, "softmax")]
    reqs = [(weights(rng, h, c, t, kind), t, c, h, m, s) for t, c, h, m, s, kind in shapes]
    together = _device_paths(L, reqs)
    for r, (tok, tim) in zip(reqs, together):
        want_t, want_j = _host_path(L, *r)
        assert np.array_equal(tok, want_t) and np.array_equal(tim, want_j), r[1:]
        alone_t, alone_j = _device_paths(L, [r])[0]
        assert np.array_equal(tok, alone_t) and np.array_equal(tim, alone_j), r[1:]
    assert [len(p[0]) for p in together][3] == 0 and min(len(p[0]) for i, p in enumerate(together) if i != 3) > 0


class Tap(Script):
    """a Script that, at each logits callback, records the state's last DTW window once: its weights, its parameters and the (id, t_dtw)
    of its text tokens as the state holds them"""

    def __init__(self, L, ctx, seed, style):
        super().__init__(L, ctx, seed, style)
        self.L, self.windows, self._seen = L, [], {}
        L.wb200_dbg_last_dtw_window.argtypes = [vp, vp]

    def _cb(self, ctx, st, toks, n, logits, ud):
        self.snap(st)
        return super()._cb(ctx, st, toks, n, logits, ud)

    def snap(self, st):
        win = (C.c_int * 4)()
        assert self.L.wb200_dbg_last_dtw_window(st, win) == 0
        if win[3] == 0 or self._seen.get(st) == win[3]:
            return
        self._seen[st] = win[3]
        qk, shape = _qks(self.L, st)
        text = [t for s in _tokens(_result(self.L, st)) for t in s if t[0] < self.eot]
        n_text = shape[0] - win[1] - 2
        if len(text) < n_text:                  # a new transcript started on this state: the window's tokens are gone
            return
        self.windows.append((qk, shape, tuple(win[:3]), text[len(text) - n_text:] if n_text > 0 else []))


def _check_windows(L, tap, eot):
    """every recorded window: t_dtw of its text tokens == host dtw_path + dtw_assign of its weights; returns (windows, tokens) checked"""
    L.wb200_dbg_dtw.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, vp]
    n_tok = 0
    for qk, shape, (n_frames, sot, seek), text in tap.windows:
        if not text:
            continue
        ids = np.asarray([t[0] for t in text], np.int32); sizes = np.asarray([len(ids)], np.int32)
        got = (C.c_int64 * len(ids))()
        assert L.wb200_dbg_dtw(qk.ctypes.data, shape[0], shape[1], shape[2], n_frames, sot, seek, eot, ids.ctypes.data, sizes.ctypes.data, 1, got) > 0
        assert list(got) == [t[1] for t in text], (shape, n_frames, seek)
        n_tok += len(ids)
    return len(tap.windows), n_tok


def _counters(L):
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    a = (C.c_double * 16)(); L.wb200_counters(a, 16)
    return list(a)


def test_device_dtw_end_to_end_pool(lib, tmp_path):
    """SMALL shape, persistent kernel: whisper_full, 8 concurrent callers, wb200_full_batch, whisper_full_parallel"""
    L = _bind(lib)
    path = _model(tmp_path, SMALL, Q5_0, 9)
    ctx = _context(L, path)
    try:
        eot = L.whisper_token_eot(ctx)
        secs = (30.0, 11.0, 47.0, 3.0, 21.5, 8.0, 30.0, 40.0)
        clips = [synth.synth_audio(seed=60 + i, seconds=s) for i, s in enumerate(secs)]
        tap = Tap(L, ctx, 77, "peaked")
        fp = _params(L, tap)
        st0 = L.wb200_ctx_state(ctx)
        c0 = _counters(L)
        alone = []
        for c in clips:
            assert L.whisper_full(ctx, fp, c.ctypes.data_as(vp), len(c)) == 0, L.wb200_last_error()
            tap.snap(st0)
            alone.append(_result(L, st0))
        c1 = _counters(L)
        assert c1[9] > c0[9] and c1[11] > c0[11]                           # DTW passes, device DTW GPU ms
        n_win, n_tok = _check_windows(L, tap, eot)
        text = [t for r in alone for s in r for t in s[2] if t[0] < eot]
        assert n_tok == len(text) > 200 and all(t[1] >= 0 for t in text)  # every text token of every window checked
        assert max(w[1][0] for w in tap.windows) > 64                      # a window of more than 64 text tokens
        # 8 concurrent whisper_full_with_state callers
        tap.windows.clear()
        states = [L.whisper_init_state(ctx) for _ in clips]
        assert all(states), L.wb200_last_error()
        rcs = [None] * len(clips)

        def work(i):
            rcs[i] = L.whisper_full_with_state(ctx, states[i], fp, clips[i].ctypes.data_as(vp), len(clips[i]))
        th = [threading.Thread(target=work, args=(i,)) for i in range(len(clips))]
        for t in th: t.start()
        for t in th: t.join()
        assert rcs == [0] * len(clips), L.wb200_last_error()
        for s in states: tap.snap(s)
        assert _check_windows(L, tap, eot)[1] == len(text)
        assert [_result(L, s) for s in states] == alone
        for s in states: L.whisper_free_state(s)
        # wb200_full_batch: windows followed by another are checked from the callback; all tokens equal the runs alone
        tap.windows.clear()
        n = len(clips)
        ptrs = (vp * n)(*[c.ctypes.data for c in clips]); lens = (C.c_int * n)(*[len(c) for c in clips]); outs = (vp * n)()
        assert L.wb200_full_batch(ctx, fp, ptrs, lens, n, outs) == 0, L.wb200_last_error()
        batched = [_result(L, outs[i]) for i in range(n)]
        for i in range(n): L.whisper_free_state(outs[i])
        assert _check_windows(L, tap, eot)[0] > 0
        assert [_tokens(r) for r in batched] == [_tokens(r) for r in alone]
        # whisper_full_parallel(8): the same, against each piece run alone
        pcm = synth.synth_audio(seed=91, seconds=8 * 33.0)
        per = len(pcm) // 8
        pieces = [np.ascontiguousarray(pcm[i * per:(i + 1) * per] if i < 7 else pcm[7 * per:]) for i in range(8)]
        want = []
        for p in pieces:
            assert L.whisper_full(ctx, fp, p.ctypes.data_as(vp), len(p)) == 0
            want += _tokens(_result(L, st0))
        tap.windows.clear()
        assert L.whisper_full_parallel(ctx, fp, pcm.ctypes.data_as(vp), len(pcm), 8) == 0, L.wb200_last_error()
        assert _check_windows(L, tap, eot)[0] > 0
        assert _tokens(_result(L, st0)) == want
    finally:
        L.whisper_free(ctx)


@pytest.mark.parametrize("shape,megakernel,audio_ctx", [("SMALL", "0", 0), ("SMALL", "1", 768), ("SMALL", "0", 768), ("WIDE", "1", 0), ("WIDE", "0", 0)])
def test_device_dtw_end_to_end_paths(lib, tmp_path, shape, megakernel, audio_ctx):
    """whisper_full, every window checked, on the persistent kernel or the chain (WB200_MEGAKERNEL=0), at a full or reduced audio_ctx"""
    L = _bind(lib)
    path = _model(tmp_path, SMALL if shape == "SMALL" else WIDE, Q5_0, 13)
    os.environ["WB200_MEGAKERNEL"] = megakernel
    try:
        ctx = _context(L, path)
    finally:
        os.environ.pop("WB200_MEGAKERNEL")
    try:
        eot = L.whisper_token_eot(ctx)
        tap = Tap(L, ctx, 77, "peaked")
        fp = _params(L, tap)
        if audio_ctx:
            fp.audio_ctx = audio_ctx
        st0 = L.wb200_ctx_state(ctx)
        n_text = 0
        secs = (9.0, 14.0) if audio_ctx else (14.0, 37.0)                 # a window covers at most 2 * audio_ctx frames
        for i, s in enumerate(secs):
            pcm = synth.synth_audio(seed=5 + i, seconds=s)
            assert L.whisper_full(ctx, fp, pcm.ctypes.data_as(vp), len(pcm)) == 0, L.wb200_last_error()
            tap.snap(st0)
            n_text += sum(1 for sg in _tokens(_result(L, st0)) for t in sg if t[0] < eot)
        n_win, n_tok = _check_windows(L, tap, eot)
        assert n_tok == n_text and n_text > 10, (n_win, n_tok, n_text)
        assert all(w[1][1] == (audio_ctx or 1500) for w in tap.windows)
        assert tap.windows[0][1][2] == (12 if shape == "SMALL" else 40) and tap.windows[0][2][1] == (1 if shape == "SMALL" else 2)
    finally:
        L.whisper_free(ctx)
