"""Q4_1 / Q5_1 models on their own device kernels: planar and tile-major records, Q8_1 activation rows, the integer block dot with the
block minimum (d_w d_x sumi + m_w s_x, ggml_vec_dot_q4_1_q8_1 / _q5_1_q8_1), the encoder's f16 expansion, the persistent decode kernel
against the kernel chain and the unmodified reference CPU build, batching, free-running parity, the load path and DTW.

NumPy side: tests/q1_ref.py (pinned to the reference's own type traits by tests/test_q8_1_cpu.py).  Tolerances are those the Q4_0 / Q5_0
tests of equal bit width use (tests/test_kernels_gpu.py, tests/test_e2e_gpu.py)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

os.environ["WB200_DEBUG_TAPS"] = "1"
import q1_ref as q1
from wbtest import DATA_DIR, F16, FullParams, TokenData, bind_whisper_api, ref_quantize, ref_dequantize, _api
from e2e_util import Side, synth, rms_err, _LOG_CB, _quiet

pytestmark = pytest.mark.gpu
vp = C.c_void_p
Q4_1, Q5_1 = synth.Q4_1, synth.Q5_1
#        logits rms (of std), margin needed for argmax equality: the tolerances of the equal-width format (Q4_0 / Q5_0)
TOL = {Q4_1: (7e-2, 0.4), Q5_1: (5e-2, 0.3)}


def _ptr(a):
    return a.ctypes.data_as(vp) if a is not None else None


def _err(x, r):
    return rms_err(x - r.mean(), r - r.mean())


def _build(tmp_path, ref, cfg, wt, seed=5):
    path = str(tmp_path / f"{cfg}-{wt}-{seed}.bin")
    synth.write_model(path, cfg, wt, seed=seed, vocab_from=os.path.join(DATA_DIR, "for-tests-ggml-tiny.en.bin"), quantizer=lambda t, w: ref_quantize(ref, t, w))
    return path


def _ulp_close(got, want):
    """equal, or one f32 ulp apart (ggml's own build may contract q * d + m into one fma)"""
    d = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    return int(d.max()) <= 1


@pytest.mark.parametrize("wt", [Q4_1, Q5_1])
@pytest.mark.parametrize("N,K", [(1000, 384), (1000, 3072), (51864, 768)])
def test_records_dequantise_exactly(lib, ref, wt, N, K):
    """file blocks -> tile-major records and planar arrays on the device -> the token-embedding reader: q * d + m bit for bit (rows past N
    pad the last tile and must not leak)"""
    rng = np.random.default_rng(N + K + wt)
    w = (rng.standard_normal((N, K)) * 0.05 * (1.0 + rng.random((N, 1)))).astype(np.float32)
    raw = np.frombuffer(ref_quantize(ref, wt, w), dtype=np.uint8)
    want = q1.dequantize(wt, raw.tobytes(), N, K)
    assert _ulp_close(want, ref_dequantize(ref, wt, raw.tobytes(), N, K))
    for hook in (lib.wb200_dbg_tm_dequant, lib.wb200_dbg_planar_dequant):
        out = np.empty((N, K), np.float32)
        assert hook(wt, N, K, _ptr(raw), _ptr(out)) == 0, lib.wb200_last_error()
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), np.abs(out - want).max()


@pytest.mark.parametrize("v2", [0, 4])
@pytest.mark.parametrize("wt", [Q4_1, Q5_1])
@pytest.mark.parametrize("N,K,n_tok", [(384, 384, 1), (1280, 1280, 1), (1000, 5120, 3), (51864, 384, 1), (640, 1280, 8), (1290, 1280, 5)])
def test_gemv_q8_1_matches_reference_arithmetic(lib, ref, wt, N, K, n_tok, v2):
    """both chain generations against the reference's Q8_1 arithmetic: only the f32 summation order differs -> 2e-5 of the output scale"""
    rng = np.random.default_rng(N + K + n_tok + wt)
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    x = rng.standard_normal((n_tok, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    scale = (0.5 + rng.random(N)).astype(np.float32)
    res = rng.standard_normal((n_tok, N)).astype(np.float32)
    raw = ref_quantize(ref, wt, w)
    out = np.empty((n_tok, N), np.float32)
    rawb = np.frombuffer(raw, dtype=np.uint8)
    rc = lib.wb200_dbg_gemv(wt, N, K, n_tok, _ptr(rawb), _ptr(x), _ptr(bias), _ptr(scale), _ptr(res), None, None, _ptr(out), v2)
    assert rc == 0, lib.wb200_last_error()
    y = q1.mul_mat_q(wt, raw, N, K, x)
    want = (y + bias[None, :]) * scale[None, :] + res
    assert np.abs(out - want).max() < 2e-5 * (np.abs(y).max() + 1.0), np.abs(out - want).max()


@pytest.mark.parametrize("wt", [Q4_1, Q5_1])
@pytest.mark.parametrize("flags", [0, 4, 5])
def test_encoder_gemm_equals_f16_gemm_on_expanded_matrix(lib, ref, wt, flags):
    """first generation (blocks decoded in the kernel), second generation with a per-launch f16 expansion (WB200_ENC_F16=0): the F16 GEMM
    on the f16 rounding of the dequantised matrix"""
    rng = np.random.default_rng(wt + flags)
    M, N, K, BN = 1280, 700, 1280, 256
    w = (rng.standard_normal((M, K)) * 0.05).astype(np.float32)
    x = rng.standard_normal((N, K)).astype(np.float32)
    bias = rng.standard_normal(M).astype(np.float32)
    raw = np.frombuffer(ref_quantize(ref, wt, w), dtype=np.uint8)
    w16 = np.frombuffer(q1.dequantize(wt, raw.tobytes(), M, K).astype(np.float16).tobytes(), dtype=np.uint8)

    def run(t, b):
        out = np.empty((N, M), np.float32)
        assert lib.wb200_dbg_gemm(C.c_int(t), M, N, K, _ptr(b), _ptr(x), _ptr(bias), _ptr(out), BN, flags) == 0, lib.wb200_last_error()
        return out
    got, want = run(wt, raw), run(F16, w16)
    if flags & 4:
        assert np.array_equal(got, want)
    else:
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


def _sides(lib, path):
    """(persistent kernel, persistent kernel, kernel chain): the layout is chosen when the context is created"""
    os.environ["WB200_MEGAKERNEL"] = "0"
    B = Side(lib, path, False)
    os.environ["WB200_MEGAKERNEL"] = "1"
    A = Side(lib, path, False); A2 = Side(lib, path, False)
    os.environ.pop("WB200_MEGAKERNEL")
    return A, A2, B


@pytest.mark.parametrize("wt", [Q4_1, Q5_1])
@pytest.mark.parametrize("cfg", ["test-2l.en", "test-2l-768.en"])
def test_persistent_kernel_matches_chain_and_reference(lib, ref, tmp_path, wt, cfg):
    path = _build(tmp_path, ref, cfg, wt)
    pcm = synth.synth_audio(seed=21, seconds=12.0)
    A, A2, B = _sides(lib, path)
    R = Side(ref, path, True)
    e_log, margin = TOL[wt]
    try:
        for S in (A, A2, B, R):
            S.pcm_to_mel(pcm); S.encode(0)
        sot = A.L.whisper_token_sot(A.ctx)
        toks = [sot, 100, 200, 300, 400]
        n_past = 0
        for step in range(12):
            feed = toks if step == 0 else toks[-1:]
            la = A.decode(feed, n_past); la2 = A2.decode(feed, n_past); lb = B.decode(feed, n_past); lr = R.decode(feed, n_past)
            n_past += len(feed)
            print("step %d: mk-chain %.2e  mk-ref %.2e  chain-ref %.2e" % (step, _err(la, lb), _err(la, lr), _err(lb, lr)))
            assert np.isfinite(la).all()
            assert np.array_equal(la, la2), step
            # the 5-row prompt pass carries the reference's multi-row F16 flash-attention accumulators: its tolerance against the reference
            # is scaled as in tests/test_kquant_decode_gpu.py::test_large_v3_width_q4_k
            assert _err(la, lb) < e_log and _err(la, lr) < e_log * (1.8 if step == 0 else 1.0), step
            assert _err(la, lr) <= 1.25 * _err(lb, lr) + 1e-3, step
            srt = np.sort(lr)
            if (srt[-1] - srt[-2]) / lr.std() > margin:
                assert int(la.argmax()) == int(lr.argmax()), step
            toks.append(int(lr.argmax()))
    finally:
        A.free(); A2.free(); B.free(); R.free()


def _counters(L):
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    a = (C.c_double * 8)(); L.wb200_counters(a, 8)
    return [a[i] for i in range(8)]


def _tokens(L, ctx):
    return [[L.whisper_full_get_token_id(ctx, s, j) for j in range(L.whisper_full_n_tokens(ctx, s))] for s in range(L.whisper_full_n_segments(ctx))]


def test_batch_of_19_chunks_equals_one_by_one_q5_1(lib, ref, tmp_path):
    """wb200_full_batch on a Q5_1 model: more than 8 rows share a pass, and every chunk gets exactly the tokens whisper_full gives it alone"""
    path = _build(tmp_path, ref, "test-2l.en", Q5_1)
    A = Side(lib, path, False)
    try:
        L = A.L
        chunks = [synth.synth_audio(seed=20 + i, seconds=4.0 + 1.5 * (i % 7)) for i in range(19)]
        fp = L.whisper_full_default_params(0); fp.print_progress = False; fp.temperature_inc = 0.0; fp.greedy.best_of = 1
        L.wb200_full_batch.argtypes = [vp, FullParams, C.POINTER(vp), C.POINTER(C.c_int), C.c_int, C.POINTER(vp)]
        n = len(chunks)
        ptrs = (vp * n)(*[c.ctypes.data for c in chunks]); lens = (C.c_int * n)(*[len(c) for c in chunks]); outs = (vp * n)()
        c0 = _counters(L)
        assert L.wb200_full_batch(A.ctx, fp, ptrs, lens, n, outs) == 0, L.wb200_last_error()
        c1 = _counters(L)
        batched = []
        for i in range(n):
            st = outs[i]
            batched.append([[L.whisper_full_get_token_id_from_state(st, s, j) for j in range(L.whisper_full_n_tokens_from_state(st, s))]
                            for s in range(L.whisper_full_n_segments_from_state(st))])
            L.whisper_free_state(st)
        rows_per_pass = (c1[1] - c0[1]) / (c1[0] - c0[0])
        print("rows per decode pass during the batch: %.1f" % rows_per_pass)
        assert rows_per_pass > 8.0
        single = []
        for c in chunks:
            assert L.whisper_full(A.ctx, fp, c.ctypes.data_as(vp), len(c)) == 0
            single.append(_tokens(L, A.ctx))
        assert batched == single
        assert sum(len(t) for c in batched for t in c) > 0
    finally:
        A.free()


LOGITS_CB = C.CFUNCTYPE(None, vp, vp, C.POINTER(TokenData), C.c_int, C.POINTER(C.c_float), vp)


def _greedy(S, pcm):
    """(token history, top-2 margin in units of the logits' std) of every sampling step of a greedy whisper_full"""
    L, V, record = S.L, S.n_vocab, []
    fp = L.whisper_full_default_params(0); fp.print_progress = False; fp.temperature_inc = 0.0; fp.greedy.best_of = 1; fp.n_threads = 4

    def rec(c, st, toks, nt, logits, ud):
        x = np.ctypeslib.as_array(logits, (V,)); fin = x[np.isfinite(x)]
        top = np.partition(fin, -2)[-2:]
        record.append((tuple(toks[k].id for k in range(nt)), float(top[1] - top[0]) / float(fin.std())))
    cb = LOGITS_CB(rec)
    fp.logits_filter_callback = C.cast(cb, vp)
    assert L.whisper_full(S.ctx, fp, pcm.ctypes.data_as(vp), len(pcm)) == 0
    return record


def test_free_running_parity_q5_1(lib, ref, tmp_path):
    """a well-conditioned Q5_1 model (synth.conditioned), greedy: the token history equals the reference's up to the first step where the
    reference's own top-2 margin is below 1e-2 sigma (the Q5_0 "margin" rule of tests/test_exact_tokens_gpu.py)"""
    path = str(tmp_path / "cond-q5_1.bin")
    synth.write_model(path, "test-3l.en", Q5_1, seed=0, vocab_from=os.path.join(DATA_DIR, "for-tests-ggml-tiny.en.bin"),
                      scale=lambda n: synth.conditioned(n, 0.0, 100.0))
    pcm = synth.synth_audio(seed=500, seconds=60.0)
    A = Side(lib, path, False); B = Side(ref, path, True)
    try:
        ra, rb = _greedy(A, pcm), _greedy(B, pcm)
        c = 0
        while c < min(len(ra), len(rb)) and ra[c][0] == rb[c][0]:
            c += 1
        print("sampling steps with identical history: %d of %d (reference), %d (here)" % (c, len(rb), len(ra)))
        assert len(rb) >= 100
        if c < min(len(ra), len(rb)):                            # histories part at step c: the decision of step c - 1 differed
            assert rb[c - 1][1] < 1e-2, (c, rb[c - 1][1])
        else:
            assert len(ra) == len(rb)
    finally:
        A.free(); B.free()


@pytest.mark.parametrize("wt", [Q4_1, Q5_1])
def test_load_keeps_the_file_bytes(lib, ref, tmp_path, wt):
    """ftype 3 / 9 load natively: no host expansion to F16, and the HBM image holds the file's bytes (not 2 B per weight)"""
    path = _build(tmp_path, ref, "test-2l.en", wt)
    log = []
    cb = _LOG_CB(lambda level, text, ud: log.append(text.decode("utf-8", "replace")))
    bind_whisper_api(lib)
    lib.whisper_log_set.argtypes = [_LOG_CB, vp]
    lib.whisper_log_set(cb, None)
    try:
        ctx = lib.whisper_init_from_file_with_params(path.encode(), lib.whisper_context_default_params())
        assert ctx, lib.wb200_last_error()
        lib.whisper_free(ctx)
    finally:
        lib.whisper_log_set(_quiet, None)
    err = "".join(log)
    assert "expanded to F16" not in err
    m = re.search(r"model size = ([0-9.]+) MB \(\d+ tensors\), HBM image = ([0-9.]+) MB", err)
    assert m, err[-2000:]
    file_mb, hbm_mb = float(m.group(1)), float(m.group(2))
    print("model size %.2f MB, HBM image %.2f MB" % (file_mb, hbm_mb))
    assert hbm_mb < 1.02 * file_mb


def test_dtw_q5_1(ref, tmp_path):
    """with DTW on, a Q5_1 model gives the tokens it gives with DTW off and a t_dtw for every text token"""
    path = _build(tmp_path, ref, "test-3l.en", Q5_1, seed=9)
    pcm = synth.synth_audio(seed=33, seconds=20.0)
    on = _api.WhisperB200(path, dtw_aheads_preset=1, dtw_n_top=2)
    off = _api.WhisperB200(path)
    try:
        assert on.full(pcm)[0] == 0 and off.full(pcm)[0] == 0
        ton, toff = on.tokens(), off.tokens()
        assert [[t[0] for t in s] for s in ton] == [[t[0] for t in s] for s in toff]
        eot = on.L.whisper_token_eot(on.ctx)
        text = [t for s in ton for t in s if t[0] < eot]
        assert text and all(t[3] >= 0 for t in text)
    finally:
        on.close(); off.close()
