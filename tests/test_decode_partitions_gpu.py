"""GPU: partitions of a persistent-kernel decode pass (wb_decode_mk.cu, WB200_MK_PARTS) change no bit.

A pass of 32 rows or more is cut into 2 or 4 partitions of whole 16-row groups, each on its own range of CTAs and its own barrier; the
partitions take turns streaming cross K/V.  Every row's arithmetic is the one of the single-partition schedule, so logits, sampled tokens
and DTW times must equal those of WB200_MK_PARTS=1 exactly:
  * wb200_decode_explicit at large-v3 width (d = 1280, 20 heads, 3 text layers), Q5_0 / F16 / Q4_K: a prompt pass with three tokens per
    sequence (rows that attend to cells other rows append in the same pass: stays on one barrier), then passes of 64, 48, 33 and 17 rows
    (full, three partitions of one group, a ragged last partition, too few rows to partition);
  * 64 ragged chunks through wb200_full_batch with timestamps on: chunks finish at different steps, so the rows of a pass -- and with them the
    number of partitions -- change from pass to pass;
  * a DTW context: the capture passes (several tokens per sequence) and the token times.
"""
import ctypes as C
import os

import numpy as np
import pytest

from wbtest import DATA_DIR, F16, Q4_K, Q5_0, FullParams, TokenData, bind_whisper_api
from e2e_util import synth

pytestmark = pytest.mark.gpu
vp = C.c_void_p
WIDE = (51864, 1500, 1280, 20, 2, 448, 1280, 20, 3, 80)                # large-v3 width: d = 1280, 20 heads; 2 audio + 3 text layers
_LOG_CB = C.CFUNCTYPE(None, C.c_int, C.c_char_p, vp)
_quiet = _LOG_CB(lambda level, text, ud: None)


def _bind(L):
    bind_whisper_api(L)
    L.whisper_log_set.argtypes = [_LOG_CB, vp]; L.whisper_log_set(_quiet, None)
    L.wb200_last_error.restype = C.c_char_p
    L.wb200_ctx_state.restype = vp; L.wb200_ctx_state.argtypes = [vp]
    L.wb200_decode_explicit.argtypes = [vp, vp, vp, vp, C.c_int, vp, vp, C.c_int, vp, C.c_int, vp]
    L.wb200_full_batch.argtypes = [vp, FullParams, C.POINTER(vp), C.POINTER(C.c_int), C.c_int, C.POINTER(vp)]
    L.whisper_full_get_token_data_from_state.restype = TokenData; L.whisper_full_get_token_data_from_state.argtypes = [vp, C.c_int, C.c_int]
    return L


def _model(tmp_path, wt, seed):
    path = str(tmp_path / f"wide-{wt}-{seed}.bin")
    if not os.path.exists(path):
        synth.write_model(path, WIDE, wt, seed=seed, vocab_from=os.path.join(DATA_DIR, "for-tests-ggml-tiny.en.bin"))
    return path


def _context(L, path, parts, dtw=False):
    """the number of partitions is read when the context is created"""
    os.environ["WB200_MK_PARTS"] = str(parts)
    try:
        cp = L.whisper_context_default_params()
        if dtw:
            cp.flash_attn = False; cp.dtw_token_timestamps = True; cp.dtw_aheads_preset = 1; cp.dtw_n_top = 2
        ctx = L.whisper_init_from_file_with_params(path.encode(), cp)
    finally:
        os.environ.pop("WB200_MK_PARTS")
    assert ctx, L.wb200_last_error()
    return ctx


def _explicit_passes(L, ctx, pcm):
    """logits of a 48-row prompt pass (16 sequences x 3 tokens) and of generation passes of 64, 48, 33 and 17 rows"""
    st = L.wb200_ctx_state(ctx)
    assert L.whisper_pcm_to_mel(ctx, pcm.ctypes.data_as(vp), len(pcm), 4) == 0
    assert L.whisper_encode(ctx, 0, 4) == 0, L.wb200_last_error()
    V = L.whisper_n_vocab(ctx)
    n_cells, ld = 256, 8
    rng = np.random.default_rng(3)
    out = []

    def decode(tok, pos, cells, idx, nkv):
        n = len(tok)
        logits = np.empty((n, V), np.float32)
        a = [np.ascontiguousarray(x, np.int32) for x in (tok, pos, cells, idx, nkv)]
        rc = L.wb200_decode_explicit(ctx, st, a[0].ctypes.data, a[1].ctypes.data, n, a[2].ctypes.data, a[3].ctypes.data, ld, a[4].ctypes.data, n_cells, logits.ctypes.data)
        assert rc == 0, L.wb200_last_error()
        assert np.isfinite(logits).all()
        return logits

    # prompt: sequence s = rows 3s .. 3s+2 in cells 3s .. 3s+2, causal inside the sequence (sequence 5 straddles two 16-row groups)
    idx = np.zeros((48, ld), np.int32)
    for s in range(16):
        for j in range(3):
            idx[3 * s + j, :j + 1] = np.arange(3 * s, 3 * s + j + 1)
    out.append(decode(rng.integers(0, 50000, 48), np.tile(np.arange(3), 16), np.arange(48), idx, np.tile(np.arange(1, 4), 16)))
    # generation: row r continues sequence r % 16 from its prompt (every row a branch of its own: its new cell is seen by no other row)
    cell0 = 48
    for n in (64, 48, 33, 17):
        idx = np.zeros((n, ld), np.int32)
        for r in range(n):
            s = r % 16
            idx[r, :4] = [3 * s, 3 * s + 1, 3 * s + 2, cell0 + r]
        out.append(decode(rng.integers(0, 50000, n), np.full(n, 3), cell0 + np.arange(n), idx, np.full(n, 4)))
        cell0 += n
    return out


@pytest.mark.parametrize("wt", [Q5_0, F16, Q4_K])
def test_partitioned_passes_give_the_bits_of_one_partition(lib, tmp_path, wt):
    L = _bind(lib)
    path = _model(tmp_path, wt, seed=2)
    pcm = synth.synth_audio(seed=5, seconds=10.0)
    got = {}
    for parts in (1, 2, 4):
        ctx = _context(L, path, parts)
        try:
            got[parts] = _explicit_passes(L, ctx, pcm)
        finally:
            L.whisper_free(ctx)
    assert len({float(x[0, 0]) for x in got[1]}) > 1                # the passes are not all the same
    for parts in (2, 4):
        for i, (a, b) in enumerate(zip(got[1], got[parts])):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (parts, i, float(np.abs(a - b).max()))
            assert np.array_equal(a.argmax(axis=1), b.argmax(axis=1)), (parts, i)


def _batch(L, ctx, fp, chunks):
    """per chunk: [(token id, p, t_dtw)] of all its segments"""
    n = len(chunks)
    ptrs = (vp * n)(*[c.ctypes.data for c in chunks]); lens = (C.c_int * n)(*[len(c) for c in chunks]); outs = (vp * n)()
    assert L.wb200_full_batch(ctx, fp, ptrs, lens, n, outs) == 0, L.wb200_last_error()
    res = []
    for i in range(n):
        st = outs[i]
        toks = [L.whisper_full_get_token_data_from_state(st, s, j) for s in range(L.whisper_full_n_segments_from_state(st))
                for j in range(L.whisper_full_n_tokens_from_state(st, s))]
        res.append([(t.id, np.float32(t.p).view(np.uint32).item(), t.t_dtw) for t in toks])
        L.whisper_free_state(st)
    return res


def _counters(L):
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    a = (C.c_double * 8)(); L.wb200_counters(a, 8)
    return [a[i] for i in range(8)]


@pytest.mark.parametrize("dtw", [False, True], ids=["timestamps", "dtw"])
def test_ragged_batch_equals_one_partition_token_for_token(lib, tmp_path, dtw):
    L = _bind(lib)
    path = _model(tmp_path, Q5_0, seed=4)
    n = 40 if dtw else 64
    chunks = [synth.synth_audio(seed=40 + i, seconds=3.0 + 0.5 * (i % 13)) for i in range(n)]
    got = {}
    for parts in (1, 4, 2):
        ctx = _context(L, path, parts, dtw=dtw)
        try:
            fp = L.whisper_full_default_params(0)
            fp.print_progress = False; fp.greedy.best_of = 1; fp.temperature_inc = 0.0; fp.no_timestamps = False; fp.max_tokens = 40; fp.n_threads = 4
            c0 = _counters(L)
            got[parts] = _batch(L, ctx, fp, chunks)
            c1 = _counters(L)
            passes, rows = c1[0] - c0[0], c1[1] - c0[1]
            print("parts %d: %d decode passes, %.1f rows per pass" % (parts, passes, rows / max(1.0, passes)))
            assert rows / passes > 1.5                                # passes are shared: all chunks in the first ones, stragglers alone at the end
        finally:
            L.whisper_free(ctx)
    assert sum(len(c) for c in got[1]) > n
    assert got[2] == got[1]
    assert got[4] == got[1]
