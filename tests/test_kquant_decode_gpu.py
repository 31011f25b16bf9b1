"""Q4_K / Q5_K models in the persistent decode kernel (wb_decode_mk.cu): tile-major K-quant records, Q8_K activation rows, and the
integer sub-block GEMV, against the NumPy dequantisation, the kernel chain (WB200_MEGAKERNEL=0) and the unmodified reference CPU build.

The persistent kernel and the chain run the same arithmetic (Q8_K activations, one integer dot per 32-value sub-block combined as
d_x * (d sc_j sumi - dmin m_j sumx)); they differ in f32 summation order only, so the cross-checks use the reference tolerances of
tests/test_e2e_gpu.py, require the persistent kernel to be as close to the reference as the chain, and two runs of it to agree bit for bit.
"""
import ctypes as C
import os
import numpy as np
import pytest

os.environ["WB200_DEBUG_TAPS"] = "1"
from wbtest import DATA_DIR, FullParams, Q4_K, Q5_K, ref_quantize, read_wav_f32
from e2e_util import Side, synth, rms_err
from oracle import ref_numpy as rn

pytestmark = pytest.mark.gpu
vp = C.c_void_p

#        logits rms (of std), margin needed for argmax equality (tests/test_e2e_gpu.py TOL)
TOL = {Q4_K: (7e-2, 0.4), Q5_K: (5e-2, 0.3)}


def _ptr(a):
    return a.ctypes.data_as(vp)


def _build(tmp_path, ref, cfg, wt, seed=5):
    stub = os.path.join(DATA_DIR, "for-tests-ggml-tiny.en.bin" if cfg.endswith(".en") else "for-tests-ggml-tiny.bin")
    path = str(tmp_path / f"{cfg}-{wt}.bin")
    synth.write_model(path, cfg, wt, seed=seed, vocab_from=stub, quantizer=lambda t, w: ref_quantize(ref, t, w))
    return path


def _sides(lib, path):
    """(persistent kernel, persistent kernel, kernel chain): the layout is chosen when the context is created"""
    os.environ["WB200_MEGAKERNEL"] = "0"
    B = Side(lib, path, False)
    os.environ["WB200_MEGAKERNEL"] = "1"
    A = Side(lib, path, False); A2 = Side(lib, path, False)
    os.environ.pop("WB200_MEGAKERNEL")
    return A, A2, B


def _err(x, r):
    return rms_err(x - r.mean(), r - r.mean())


@pytest.mark.parametrize("wt", [Q4_K, Q5_K])
@pytest.mark.parametrize("N,K", [(1000, 256), (1000, 1280), (1000, 5120), (51866, 256)])
def test_tile_major_records_dequantise_exactly(lib, ref, wt, N, K):
    """file super-blocks -> tile-major records on the device -> the token-embedding reader: dequantize_row_q4_K / _q5_K bit for bit
    (rows past N are padding of the last tile and must not leak into any row)"""
    rng = np.random.default_rng(N + K + wt)
    w = (rng.standard_normal((N, K)) * 0.05 * (1.0 + rng.random((N, 1)))).astype(np.float32)
    raw = np.frombuffer(ref_quantize(ref, wt, w), dtype=np.uint8)
    out = np.empty((N, K), np.float32)
    assert lib.wb200_dbg_tm_dequant(wt, N, K, _ptr(raw), _ptr(out)) == 0, lib.wb200_last_error()
    want = rn.dequantize(wt, raw.tobytes(), N, K)
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), np.abs(out - want).max()


@pytest.mark.parametrize("wt", [Q4_K, Q5_K])
def test_persistent_kernel_matches_chain_on_kquants(lib, ref, tmp_path, wt):
    path = _build(tmp_path, ref, "test-2l-512.en", wt)
    pcm = synth.synth_audio(seed=21, seconds=12.0)
    A, A2, B = _sides(lib, path)
    R = Side(ref, path, True)
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
            assert _err(la, lb) < TOL[wt][0], (step, _err(la, lb))
            assert _err(la, lr) < 1.25 * _err(lb, lr) + 1e-3, step
            toks.append(int(lb.argmax()))
    finally:
        A.free(); A2.free(); B.free(); R.free()


def test_large_v3_width_q4_k(lib, ref, tmp_path):
    """large-v3 shapes (d = 1280: 20 heads, 4 heads per super-block; FC2 K = 5120; 51866 ids) at 4 + 4 layers: a 3-row prompt pass
    and 5 single-row steps against the reference and the chain.  The prompt pass carries the reference's multi-row F16 flash-attention
    accumulators: its tolerance is scaled by the large4 ratio of tests/test_golden_large_gpu.py (9e-2 / 5e-2)."""
    path = _build(tmp_path, ref, "large-v3-4l", Q4_K, seed=3)
    pcm = synth.synth_audio(seed=8, seconds=20.0)
    A, A2, B = _sides(lib, path)
    A2.free()
    R = Side(ref, path, True)
    try:
        for S in (A, B):
            S.pcm_to_mel(pcm); S.encode(0)
        R.pcm_to_mel(pcm)
        assert R.L.whisper_encode(R.ctx, 0, max(4, os.cpu_count() or 4)) == 0
        sot = A.L.whisper_token_sot(A.ctx)
        toks = [sot, sot + 1, A.L.whisper_token_transcribe(A.ctx)]
        n_past = 0
        e_log, margin = TOL[Q4_K]
        for step in range(6):
            feed = toks if step == 0 else toks[-1:]
            la = A.decode(feed, n_past); lb = B.decode(feed, n_past); lr = R.decode(feed, n_past)
            n_past += len(feed)
            tol = e_log * (1.8 if step == 0 else 1.0)
            print("step %d: mk-chain %.2e  mk-ref %.2e  chain-ref %.2e" % (step, _err(la, lb), _err(la, lr), _err(lb, lr)))
            assert np.isfinite(la).all()
            assert _err(la, lr) < tol, (step, _err(la, lr))
            assert _err(la, lb) < e_log, (step, _err(la, lb))
            assert _err(la, lr) < 1.25 * _err(lb, lr) + 1e-3, step
            srt = np.sort(lr)
            if (srt[-1] - srt[-2]) / lr.std() > margin:
                assert int(la.argmax()) == int(lr.argmax()), step
            toks.append(int(lr.argmax()))
    finally:
        A.free(); B.free(); R.free()


def _counters(L):
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    a = (C.c_double * 8)(); L.wb200_counters(a, 8)
    return [a[i] for i in range(8)]


def _tokens(L, ctx):
    return [[L.whisper_full_get_token_id(ctx, s, j) for j in range(L.whisper_full_n_tokens(ctx, s))] for s in range(L.whisper_full_n_segments(ctx))]


def test_batch_of_19_chunks_equals_one_by_one_q4_k(lib, ref, tmp_path):
    """wb200_full_batch on a Q4_K model: more than 8 rows share a pass, and every chunk gets exactly the tokens whisper_full gives it alone"""
    path = _build(tmp_path, ref, "test-2l-512.en", Q4_K, seed=5)
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


def test_beam_search_q4_k(lib, ref, tmp_path):
    """beam 5 with the device draws on a Q4_K model: deterministic, and the same control flow as the reference (see
    test_whisper_full_beam_search_matches_reference for why random weights do not allow more)"""
    path = _build(tmp_path, ref, "test-2l-512.en", Q4_K, seed=11)
    pcm = read_wav_f32(os.path.join(DATA_DIR, "jfk.wav"))
    A = Side(lib, path, False); A2 = Side(lib, path, False); B = Side(ref, path, True)     # a fresh context each (no prompt from a previous call)
    try:
        ra, sa = A.full(pcm, strategy=1, beam_size=5, temperature_inc=0.0)
        ra2, sa2 = A2.full(pcm, strategy=1, beam_size=5, temperature_inc=0.0)
        rb, sb = B.full(pcm, strategy=1, beam_size=5, temperature_inc=0.0)
        assert ra == 0 and ra2 == 0 and rb == 0
        assert [s[2] for s in sa] == [s[2] for s in sa2]
        assert len(sa) >= 1 and len(sb) >= 1
        assert sa[0][0] == sb[0][0]
        assert all(0 <= t < A.n_vocab for s in sa for t in s[2])
    finally:
        A.free(); A2.free(); B.free()
