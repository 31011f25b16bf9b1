"""Q3_K models on their own device kernels: tile-major records with a 288-byte header (16 rows x 16 integer scales + d), the verbatim
super-blocks of the encoder side and the kernel chain, Q8_K activation rows, the integer sub-block dot (two k16 products combined with
their 16-value scales, ggml_vec_dot_q3_K_q8_K), the encoder's f16 expansion, the persistent decode kernel against the kernel chain and
the unmodified reference CPU build, batching, partitions, the load path, DTW and beam search.

NumPy side: tests/kq_signed_ref.py (pinned to the reference's own type traits by tests/test_q8_k_signed_cpu.py).  Tolerances are those of
tests/test_wider_formats_gpu.py."""
import ctypes as C
import os
import re

import numpy as np
import pytest

os.environ["WB200_DEBUG_TAPS"] = "1"
import kq_signed_ref as kq
from wbtest import DATA_DIR, F16, FullParams, bind_whisper_api, ref_quantize, ref_dequantize, _api
from e2e_util import Side, synth, rms_err, taps, _LOG_CB, _quiet

pytestmark = pytest.mark.gpu
vp = C.c_void_p
Q3_K = synth.Q3_K
#        logits rms (of std) against the chain, margin needed for argmax equality with the reference
TOL = {Q3_K: (1.2e-1, 0.6)}


def _ptr(a):
    return a.ctypes.data_as(vp) if a is not None else None


def _err(x, r):
    return rms_err(x - r.mean(), r - r.mean())


def _build(tmp_path, ref, cfg, wt, seed=5, **kw):
    path = str(tmp_path / f"{cfg}-{wt}-{seed}.bin")
    synth.write_model(path, cfg, wt, seed=seed, vocab_from=os.path.join(DATA_DIR, "for-tests-ggml-tiny.en.bin"), quantizer=lambda t, w: ref_quantize(ref, t, w), **kw)
    return path


@pytest.mark.parametrize("wt", [Q3_K])
@pytest.mark.parametrize("N,K", [(1000, 256), (1000, 1280), (1000, 5120), (51866, 1280), (1003, 512)])
def test_records_dequantise_exactly(lib, ref, wt, N, K):
    """file super-blocks -> tile-major records / verbatim blocks on the device -> the token-embedding readers: dequantize_row_* bit for bit"""
    rng = np.random.default_rng(N + K + wt)
    w = (rng.standard_normal((N, K)) * 0.05 * (1.0 + rng.random((N, 1)))).astype(np.float32)
    raw = np.frombuffer(ref_quantize(ref, wt, w), dtype=np.uint8)
    want = ref_dequantize(ref, wt, raw.tobytes(), N, K)
    for hook in (lib.wb200_dbg_tm_dequant, lib.wb200_dbg_planar_dequant):
        out = np.empty((N, K), np.float32)
        assert hook(wt, N, K, _ptr(raw), _ptr(out)) == 0, lib.wb200_last_error()
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), np.abs(out - want).max()


@pytest.mark.parametrize("v2", [0, 4])
@pytest.mark.parametrize("wt", [Q3_K])
@pytest.mark.parametrize("N,K,n_tok", [(512, 512, 1), (1280, 1280, 2), (1000, 5120, 3), (51864, 512, 1), (640, 1280, 8), (1290, 1280, 5)])
def test_gemv_q8_k_matches_reference_arithmetic(lib, ref, wt, N, K, n_tok, v2):
    """both chain generations against the reference's Q8_K arithmetic: only the f32 summation order differs -> 2e-5 of the output scale"""
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
    y = kq.mul_mat_q(wt, raw, N, K, x)
    want = (y + bias[None, :]) * scale[None, :] + res
    assert np.abs(out - want).max() < 2e-5 * (np.abs(y).max() + 1.0), np.abs(out - want).max()


@pytest.mark.parametrize("wt", [Q3_K])
@pytest.mark.parametrize("flags", [0, 4, 5])
def test_encoder_gemm_equals_f16_gemm_on_expanded_matrix(lib, ref, wt, flags):
    """first generation (blocks decoded in the kernel), second generation with a per-launch f16 expansion: the F16 GEMM on the f16 rounding
    of the dequantised matrix"""
    rng = np.random.default_rng(wt + flags)
    M, N, K, BN = 1280, 700, 1280, 256
    w = (rng.standard_normal((M, K)) * 0.05).astype(np.float32)
    x = rng.standard_normal((N, K)).astype(np.float32)
    bias = rng.standard_normal(M).astype(np.float32)
    raw = np.frombuffer(ref_quantize(ref, wt, w), dtype=np.uint8)
    w16 = np.frombuffer(ref_dequantize(ref, wt, raw.tobytes(), M, K).astype(np.float16).tobytes(), dtype=np.uint8)

    def run(t, b):
        out = np.empty((N, M), np.float32)
        assert lib.wb200_dbg_gemm(C.c_int(t), M, N, K, _ptr(b), _ptr(x), _ptr(bias), _ptr(out), BN, flags) == 0, lib.wb200_last_error()
        return out
    got, want = run(wt, raw), run(F16, w16)
    if flags & 4:
        assert np.array_equal(got, want)
    else:
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


def _side(lib, path, env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return Side(lib, path, False)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.parametrize("wt", [Q3_K])
def test_persistent_kernel_matches_chain_and_reference(lib, ref, tmp_path, wt):
    path = _build(tmp_path, ref, "test-2l-512.en", wt)
    pcm = synth.synth_audio(seed=21, seconds=12.0)
    A, A2 = _side(lib, path, {"WB200_MEGAKERNEL": "1"}), _side(lib, path, {"WB200_MEGAKERNEL": "1"})
    B = _side(lib, path, {"WB200_MEGAKERNEL": "0"})
    F = _side(lib, path, {"WB200_KQUANT_AS_F16": "1"})
    R = Side(ref, path, True)
    e_log, margin = TOL[wt]
    try:
        for S in (A, A2, B, F, R):
            S.pcm_to_mel(pcm); S.encode(0)
        ta, tf = taps(A), taps(F)                                 # the encoder side: f16 expansion at load == the host expansion
        for tap in ("enc", "kc", "kv"):
            assert np.array_equal(ta[tap].view(np.uint32), tf[tap].view(np.uint32)), tap
        sot = A.L.whisper_token_sot(A.ctx)
        toks = [sot, 100, 200, 300, 400]
        n_past = 0
        for step in range(12):
            feed = toks if step == 0 else toks[-1:]
            la = A.decode(feed, n_past); la2 = A2.decode(feed, n_past); lb = B.decode(feed, n_past); lf = F.decode(feed, n_past)
            lr = R.decode(feed, n_past)
            n_past += len(feed)
            print("step %d: mk-chain %.2e  mk-ref %.2e  chain-ref %.2e  f16-ref %.2e" % (step, _err(la, lb), _err(la, lr), _err(lb, lr), _err(lf, lr)))
            assert np.isfinite(la).all()
            assert np.array_equal(la, la2), step
            assert _err(la, lb) < e_log, step
            assert _err(la, lr) <= 1.25 * _err(lb, lr) + 1e-3, step
            srt = np.sort(lr)
            if (srt[-1] - srt[-2]) / lr.std() > margin:
                assert int(la.argmax()) == int(lr.argmax()), step
            toks.append(int(lr.argmax()))
    finally:
        A.free(); A2.free(); B.free(); F.free(); R.free()


def _counters(L):
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    a = (C.c_double * 8)(); L.wb200_counters(a, 8)
    return [a[i] for i in range(8)]


def _tokens(L, ctx):
    return [[L.whisper_full_get_token_id(ctx, s, j) for j in range(L.whisper_full_n_tokens(ctx, s))] for s in range(L.whisper_full_n_segments(ctx))]


def test_batch_of_19_chunks_equals_one_by_one_q3_k(lib, ref, tmp_path):
    """wb200_full_batch on a Q3_K model: more than 8 rows share a pass, and every chunk gets exactly the tokens whisper_full gives it alone"""
    path = _build(tmp_path, ref, "test-2l-512.en", Q3_K)
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


@pytest.mark.parametrize("wt,ratio", [(Q3_K, 1.05)])
def test_load_keeps_the_file_bytes(lib, ref, tmp_path, wt, ratio):
    """ftype 11 loads natively: no host expansion to F16, and the HBM image is close to the file's bytes (not 2 B per weight)"""
    path = _build(tmp_path, ref, "test-2l-512.en", wt)
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
    assert hbm_mb <= ratio * file_mb


@pytest.mark.parametrize("wt", [Q3_K])
def test_dtw_and_beam(ref, tmp_path, wt):
    """DTW on / off give the same tokens and a t_dtw for every text token; beam 5 gives the same tokens on two contexts"""
    path = _build(tmp_path, ref, "test-3l-512.en", wt, seed=9)
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
    b1, b2 = _api.WhisperB200(path), _api.WhisperB200(path)
    try:
        for b in (b1, b2):
            fp = b.default_params(1); fp.beam_search.beam_size = 5
            assert b.full(pcm, fp)[0] == 0
        assert [[t[0] for t in s] for s in b1.tokens()] == [[t[0] for t in s] for s in b2.tokens()]
    finally:
        b1.close(); b2.close()


@pytest.mark.parametrize("wt", [Q3_K])
def test_partitioned_passes_give_the_bits_of_one_partition(lib, tmp_path, wt):
    """WB200_MK_PARTS=1 against the default partitions: logits and tokens of 64 / 48 / 33 / 17-row passes bit for bit"""
    from test_decode_partitions_gpu import _bind, _context, _explicit_passes, _model
    L = _bind(lib)
    path = _model(tmp_path, wt, seed=2)
    pcm = synth.synth_audio(seed=5, seconds=10.0)
    got = {}
    for parts in (1, 4):
        ctx = _context(L, path, parts)
        try:
            got[parts] = _explicit_passes(L, ctx, pcm)
        finally:
            L.whisper_free(ctx)
    assert len({float(x[0, 0]) for x in got[1]}) > 1
    for i, (a, b) in enumerate(zip(got[1], got[4])):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (i, float(np.abs(a - b).max()))
        assert np.array_equal(a.argmax(axis=1), b.argmax(axis=1)), i
