"""GPU: run-ahead decode passes of the context pool (Group::run, wb_api.cpp).

After a pass of greedy rows sampled on the device, the pool enqueues the next single-token step of every sequence that may continue,
with the token read on the device from the pass's sampler output; the next batch takes the results of the rows whose real request
equals the prediction.  The per-row arithmetic of the persistent decode kernel does not depend on the batch, so taking a run-ahead
row changes no output.  Each case runs the same work with run-ahead on and off (wb200_dbg_run_ahead) in one process and asserts that
token ids, probabilities, segment times and no-speech probabilities are bit-identical, and what wb200_counters [12] (run-ahead rows
launched) and [13] (rows taken) say about the path that ran:
  * 64 chunks, greedy, no timestamps, through wb200_full_batch_ex: every single-token step is a run-ahead row that was taken, except
    the one after a sequence's end-of-text token;
  * the same chunks with timestamps on: sampled timestamps make rows mismatch, windows restart; some rows are rejected and recomputed;
  * staggered concurrent whisper_full_with_state callers, one of which creates its state mid-transcription and grows the pool;
  * states at audio_ctx 768 and 1500 in one pool;
  * DTW token timestamps and beam search never run ahead; a temperature fallback gives the same transcript either way.
"""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

from wbtest import DATA_DIR, Q5_0, FullParams, TokenData, bind_whisper_api
from e2e_util import synth
from test_full_scripted_cpu import LOG_CB, _quiet

pytestmark = pytest.mark.gpu
vp = C.c_void_p


def _bind(L):
    bind_whisper_api(L)
    L.whisper_log_set.argtypes = [LOG_CB, vp]; L.whisper_log_set(_quiet, None)
    L.wb200_last_error.restype = C.c_char_p
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    L.wb200_dbg_run_ahead.argtypes = [vp, C.c_int]
    L.wb200_full_batch_ex.argtypes = [vp, FullParams, C.POINTER(vp), C.POINTER(C.c_int), C.c_int, C.POINTER(vp), C.c_int]
    L.whisper_full_get_token_data_from_state.restype = TokenData; L.whisper_full_get_token_data_from_state.argtypes = [vp, C.c_int, C.c_int]
    L.whisper_full_get_segment_no_speech_prob_from_state.restype = C.c_float
    L.whisper_full_get_segment_no_speech_prob_from_state.argtypes = [vp, C.c_int]
    return L


def _model(tmp_path, seed=3):
    path = str(tmp_path / f"test-3l.en-q5_0-{seed}.bin")       # 3 text layers: timestamps stay on when asked for
    synth.write_model(path, "test-3l.en", Q5_0, seed=seed, vocab_from=os.path.join(DATA_DIR, "for-tests-ggml-tiny.en.bin"))
    return path


def _context(L, path, dtw=False):
    cp = L.whisper_context_default_params()
    if dtw:
        cp.flash_attn = False; cp.dtw_token_timestamps = True; cp.dtw_aheads_preset = 1; cp.dtw_n_top = 2
    ctx = L.whisper_init_from_file_with_params(path.encode(), cp)
    assert ctx, L.wb200_last_error()
    return ctx


def _params(L, no_timestamps=True, **kw):
    fp = L.whisper_full_default_params(0)
    fp.print_progress = False; fp.n_threads = 4; fp.greedy.best_of = 1; fp.temperature_inc = 0.0; fp.no_timestamps = no_timestamps
    for k, v in kw.items():
        obj, _, name = k.rpartition("__")
        setattr(getattr(fp, obj) if obj else fp, name, v)
    return fp


def _counters(L):
    a = (C.c_double * 14)(); L.wb200_counters(a, 14)
    return np.array([a[i] for i in range(14)])


def _result(L, st):
    """per segment: t0, t1, no-speech probability (bits), [(id, p bits)]"""
    out = []
    for i in range(L.whisper_full_n_segments_from_state(st)):
        toks = [L.whisper_full_get_token_data_from_state(st, i, j) for j in range(L.whisper_full_n_tokens_from_state(st, i))]
        nsp = np.float32(L.whisper_full_get_segment_no_speech_prob_from_state(st, i)).view(np.uint32).item()
        out.append((L.whisper_full_get_segment_t0_from_state(st, i), L.whisper_full_get_segment_t1_from_state(st, i), nsp,
                    [(t.id, np.float32(t.p).view(np.uint32).item()) for t in toks]))
    return out


def _batch(L, ctx, fp, clips):
    """wb200_full_batch_ex on host PCM: per chunk its result, and the counters it moved"""
    n = len(clips)
    ptrs = (vp * n)(*[c.ctypes.data for c in clips]); lens = (C.c_int * n)(*[len(c) for c in clips]); outs = (vp * n)()
    c0 = _counters(L)
    assert L.wb200_full_batch_ex(ctx, fp, ptrs, lens, n, outs, 0) == 0, L.wb200_last_error()
    d = _counters(L) - c0
    res = [_result(L, outs[i]) for i in range(n)]
    for i in range(n):
        L.whisper_free_state(outs[i])
    return res, d


def _on_off(L, ctx, run):
    """run() with run-ahead on, then off: (result on, counters on, result off, counters off)"""
    out = []
    for on in (1, 0):
        assert L.wb200_dbg_run_ahead(ctx, on) == 0
        out.extend(run())
    assert L.wb200_dbg_run_ahead(ctx, 1) == 0
    return out


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return _model(tmp_path_factory.mktemp("run_ahead"))


def test_greedy_text_only_batch_takes_every_step(lib, model):
    L = _bind(lib)
    ctx = _context(L, model)
    try:
        clips = [synth.synth_audio(seed=300 + i, seconds=30.0) for i in range(64)]
        fp = _params(L, no_timestamps=True)
        _batch(L, ctx, fp, clips[:2])                               # sizes the pool
        on, c_on, off, c_off = _on_off(L, ctx, lambda: _batch(L, ctx, fp, clips))
        assert on == off
        eot = L.whisper_token_eot(ctx)
        n_tok = sum(len(s[3]) for r in on for s in r)
        ended_by_eot = sum(1 for r in on if r and r[-1][3] and r[-1][3][-1][0] == eot)
        launched, taken = c_on[12], c_on[13]
        print(f"64 chunks: {n_tok} tokens, {c_on[0]:.0f} passes (off: {c_off[0]:.0f}), run-ahead rows {launched:.0f} launched, {taken:.0f} taken, "
              f"{ended_by_eot} sequences ended by end-of-text")
        assert c_off[12] == 0 and c_off[13] == 0
        assert taken > 0.8 * n_tok
        assert launched - taken == ended_by_eot                     # only the row after an end-of-text token is launched in vain
        assert c_on[1] == c_off[1] + ended_by_eot                   # every row taken replaces one ordinary row
    finally:
        L.whisper_free(ctx)


def test_timestamps_on_rejects_and_recomputes(lib, model):
    L = _bind(lib)
    ctx = _context(L, model)
    try:
        clips = [synth.synth_audio(seed=400 + i, seconds=s) for i, s in enumerate([30.0, 47.0, 12.0, 61.0] * 16)]
        fp = _params(L, no_timestamps=False)
        on, c_on, off, c_off = _on_off(L, ctx, lambda: _batch(L, ctx, fp, clips))
        assert on == off
        print(f"timestamps on: {sum(len(r) for r in on)} segments, run-ahead rows {c_on[12]:.0f} launched, {c_on[13]:.0f} taken")
        assert 0 < c_on[13] < c_on[12]
    finally:
        L.whisper_free(ctx)


def _threads(L, ctx, fps, clips, delays, late=None):
    """one whisper_full_with_state caller per clip, started after its delay; the caller `late` creates its state when it starts,
    which grows the pool while the others transcribe"""
    n = len(clips)
    states = [None if i == late else L.whisper_init_state(ctx) for i in range(n)]
    rcs = [None] * n
    c0 = _counters(L)

    def work(i):
        time.sleep(delays[i])
        if states[i] is None:
            states[i] = L.whisper_init_state(ctx)
        rcs[i] = L.whisper_full_with_state(ctx, states[i], fps[i], clips[i].ctypes.data_as(vp), len(clips[i]))
    th = [threading.Thread(target=work, args=(i,)) for i in range(n)]
    for t in th: t.start()
    for t in th: t.join()
    d = _counters(L) - c0
    assert rcs == [0] * n, (rcs, L.wb200_last_error())
    res = [_result(L, st) for st in states]
    for st in states:
        L.whisper_free_state(st)
    return res, d


def test_staggered_callers_and_pool_growth(lib, model):
    L = _bind(lib)
    ctx = _context(L, model)
    try:
        clips = [synth.synth_audio(seed=500 + i, seconds=s) for i, s in enumerate((30.0, 47.0, 21.0, 30.0, 66.0))]
        # one sampler configuration for all: a batch that mixes configurations samples on the host, and which requests share a batch
        # depends on the callers' timing
        fps = [_params(L, no_timestamps=False) for _ in clips]
        delays = (0.0, 0.05, 0.2, 0.4, 0.3)
        on, c_on, off, c_off = _on_off(L, ctx, lambda: _threads(L, ctx, fps, clips, delays, late=4))
        assert on == off
        assert c_on[13] > 0 and c_off[12] == 0
    finally:
        L.whisper_free(ctx)


def test_mixed_audio_ctx_in_one_pool(lib, model):
    L = _bind(lib)
    ctx = _context(L, model)
    try:
        clips = [synth.synth_audio(seed=600 + i, seconds=s) for i, s in enumerate((14.0, 25.0, 14.0, 30.0))]
        fps = [_params(L, no_timestamps=True, audio_ctx=T) for T in (768, 0, 768, 0)]
        on, c_on, off, c_off = _on_off(L, ctx, lambda: _threads(L, ctx, fps, clips, (0.0, 0.0, 0.0, 0.0)))
        assert on == off
        assert sum(len(s[3]) for r in on for s in r) > 20
    finally:
        L.whisper_free(ctx)


@pytest.mark.parametrize("case", ["dtw", "beam5", "fallback"])
def test_paths_that_do_not_run_ahead(lib, model, case):
    L = _bind(lib)
    ctx = _context(L, model, dtw=(case == "dtw"))
    try:
        clips = [synth.synth_audio(seed=700 + i, seconds=s) for i, s in enumerate((30.0, 19.0, 30.0))]
        if case == "beam5":
            fp = _params(L, no_timestamps=True, strategy=1, beam_search__beam_size=5)
        elif case == "fallback":
            # an unreachable log-probability threshold fails every attempt: t = 0 runs greedy on the device, t > 0 samples on the host
            fp = _params(L, no_timestamps=True, temperature_inc=0.4, logprob_thold=10.0, greedy__best_of=2)
        else:
            fp = _params(L, no_timestamps=True)
        on, c_on, off, c_off = _on_off(L, ctx, lambda: _batch(L, ctx, fp, clips))
        assert on == off
        assert sum(len(s[3]) for r in on for s in r) > 0
        if case != "fallback":
            assert c_on[12] == 0 and c_on[13] == 0
    finally:
        L.whisper_free(ctx)
