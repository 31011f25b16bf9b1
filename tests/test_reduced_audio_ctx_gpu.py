"""GPU: a reduced encoder context (whisper_full_params.audio_ctx = T < 1500) through every kernel that depends on it, against the reference.

`-ac 768` encodes half the positions of a 30-s window.  The conv stem then runs on 2T frames, the encoder attention on T queries over
pad256(T) keys, and the cross GEMM writes T rows per head into a cross K/V buffer laid out for the model's full padded context (Tp_max =
1536 rows per head).  Both decoders attend to pad256(T) keys of that buffer, the keys T .. pad256(T) - 1 being zero rows that stay in the
softmax as in the reference.  Asserted:
  * the decode kernel's cross-attention phase reads the producer's layout (1536 rows per head) at every key count, and gives the same bits
    as on a buffer of exactly n_keys rows per head; rows past the real keys hold NaN, so a read of any of them shows;
  * the encoder attention kernel at reduced T against a float64 softmax with pad256(T) - T zero keys;
  * conv, encoder output, cross K / V and 10 teacher-forced logits of the engine (persistent decode kernel and kernel chain) against the
    reference at T = 512, 750, 1000; the cross K / V rows past T are exactly zero; the DTW alignment weights at T = 768;
  * states of one context with different audio_ctx, run concurrently, give exactly what each gives alone (DESIGN.md section 1.1), also
    when a state with a third context length starts while the others are in the middle of their transcriptions.
"""
import ctypes as C
import os
import threading

import numpy as np
import pytest

os.environ["WB200_DEBUG_TAPS"] = "1"
import actq  # noqa: E402
from oracle import ref_numpy as rn  # noqa: E402
from wbtest import DATA_DIR, F16, Q4_K, Q5_0, read_wav_f32  # noqa: E402
from e2e_util import Side, rms_err, synth  # noqa: E402
from test_e2e_gpu import TOL, _build  # noqa: E402
from test_decode_phases_gpu import ATTN_CROSS, QUANT_ROWS, Q5_K, check_quantised, f32_out, probe, untouched, untouched_bytes  # noqa: E402
from test_dtw_pool_gpu import WIDE, SMALL, _bind, _context, _model, _params, _qks, _ref_tokens, _result, _tokens  # noqa: E402
from test_full_scripted_cpu import Script  # noqa: E402

pytestmark = pytest.mark.gpu
vp = C.c_void_p
F16_NAN = np.uint16(0x7E00)
TP_MAX = 1536                                                   # pad256(1500): rows per head of the engine's cross K/V buffer


def pad256(n):
    return (n + 255) // 256 * 256


# ---- kernel level -----------------------------------------------------------------------------------------------------------------------
def _cross_inputs(n_head, N, seed):
    """head-major cross K / V of 3 slots with TP_MAX rows per head: N real keys, NaN in every other row"""
    d, n_slots = 64 * n_head, 3
    rng = np.random.default_rng(seed)
    kx = np.full((n_slots, n_head, TP_MAX, 64), F16_NAN, np.uint16); vx = kx.copy()
    kx[:, :, :N] = (rng.standard_normal((n_slots, n_head, N, 64)) * 0.3).astype(np.float16).view(np.uint16)
    vx[:, :, :N] = rng.standard_normal((n_slots, n_head, N, 64)).astype(np.float16).view(np.uint16)
    q = rng.standard_normal((actq.ROWS, d)).astype(np.float32)
    slot = (np.arange(actq.ROWS) * 7 % n_slots).astype(np.int32)
    return kx, vx, q, slot


@pytest.mark.parametrize("n_head", [6, 20])
@pytest.mark.parametrize("N,n_keys", [(1, 256), (200, 256), (750, 768), (768, 768), (1000, 1024), (1280, 1280), (1500, 1536)])
def test_cross_phase_reads_the_producers_layout(lib, n_head, N, n_keys):
    """the cross GEMM writes head h of a layer at h * 1536 * 64; the phase attends to the first n_keys rows of each head, N of them real"""
    d = 64 * n_head
    kx, vx, q, slot = _cross_inputs(n_head, N, [n_head, N])
    scale = np.float32(64.0 ** -0.25)
    n_tok, row0, n_cta = (5, 16, 7) if n_head == 6 else (9, 3, 37)     # pairs split unevenly over the CTAs
    rows = list(range(row0, row0 + n_tok))
    kw = dict(d=d, n_head=n_head, n_keys=n_keys, n_slots=3, slot=slot, kq_scale=scale, N=N)
    full = dict(kw, xk=kx, xv=vx, kv_rows=TP_MAX)
    f = f32_out(3 * d)
    probe(lib, Q5_K, ATTN_CROSS, n_cta, row0, n_tok, f, q, **full)
    k64, v64 = kx.view(np.float16), vx.view(np.float16)
    for t in rows:
        want = np.concatenate([rn.attention(q[t:t + 1, 64 * h:64 * h + 64], k64[slot[t], h, :N].astype(np.float32),
                                            v64[slot[t], h, :N].astype(np.float32), float(scale), n_zero_keys=n_keys - N)[0]
                               for h in range(n_head)])
        err = np.abs(f[t, :d] - want)
        assert err.max() < 1e-4, (t, float(np.nanmax(err)), int(np.isnan(f[t, :d]).sum()))
    assert untouched(f, rows)
    # the same keys in a buffer of exactly n_keys rows per head: the same bits
    compact = dict(kw, xk=np.ascontiguousarray(kx[:, :, :n_keys]), xv=np.ascontiguousarray(vx[:, :, :n_keys]), kv_rows=n_keys)
    g = f32_out(3 * d)
    probe(lib, Q5_K, ATTN_CROSS, n_cta, row0, n_tok, g, q, **compact)
    assert np.array_equal(f[rows].view(np.uint32), g[rows].view(np.uint32))
    for wt in QUANT_ROWS:
        out = np.full(actq.nbytes(wt, d), 0xA5, np.uint8)
        probe(lib, wt, ATTN_CROSS, n_cta, row0, n_tok, out, q, **full)
        fq, fd = check_quantised(wt, d, out, rows, f[rows, :d], 0.0)
        assert fq < 1e-3 and fd < 0.01, (wt, fq, fd)
        assert untouched_bytes(wt, d, out, rows)


@pytest.mark.parametrize("T", [1, 64, 200, 750, 768, 1000, 1280])
def test_encoder_attention_at_reduced_context(lib, T):
    """fattn_enc_kernel with T queries over pad256(T) keys (T real, the rest all-zero and unmasked), two windows, against float64; tolerance
    of test_kernels_gpu.test_encoder_flash_attention_kernel (f16 probabilities on the tensor core, f16 output)"""
    rng = np.random.default_rng(T)
    Tp, H, n_win = pad256(T), 3, 2
    d = H * 64
    q = (rng.standard_normal((n_win, T, d)) * 1.5).astype(np.float32); k = rng.standard_normal((n_win, T, d)).astype(np.float32)
    v = rng.standard_normal((n_win, T, d)).astype(np.float32)
    out = np.full((n_win, T, d), np.nan, np.float32)
    scale = 1.0 / 8.0
    lib.wb200_dbg_fattn.restype = C.c_int
    p = lambda a: a.ctypes.data_as(vp)  # noqa: E731
    assert lib.wb200_dbg_fattn(p(q), p(k), p(v), T, Tp, H, n_win, C.c_float(scale), p(out)) == 0, lib.wb200_last_error()
    q16, k16, v16 = (x.astype(np.float16).astype(np.float64) for x in (q, k, v))
    worst = 0.0
    for w in range(n_win):
        for h in range(H):
            sl = slice(h * 64, h * 64 + 64)
            s_ = np.concatenate([q16[w, :, sl] @ k16[w, :, sl].T * scale, np.zeros((T, Tp - T))], axis=1)
            p_ = np.exp(s_ - s_.max(axis=1, keepdims=True)); p_ /= p_.sum(axis=1, keepdims=True)
            worst = max(worst, float(np.abs(out[w, :, sl] - p_[:, :T] @ v16[w, :, sl]).max()))
    assert worst < 4e-3, worst


# ---- engine against the reference -------------------------------------------------------------------------------------------------------
def _set_audio_ctx(S, T):
    """both libraries take the encoder context from the state, and only whisper_full sets it: a short whisper_full at audio_ctx = T"""
    clip = synth.synth_audio(seed=3, seconds=2.0)
    rc, _ = S.full(clip, audio_ctx=T, temperature_inc=0.0, greedy_best_of=1, max_tokens=4)
    assert rc == 0


def _taps_at(S, T):
    """conv [T][d], enc [T][d], kc / kv [Lt][T][d] of the last encode at context T; on the engine side also kc / kv rows T .. 1535"""
    L, d, Lt, Tp = S.L, S.d, S.Lt, pad256(T)
    p = lambda a: a.ctypes.data_as(vp)  # noqa: E731
    if S.is_ref:
        conv = np.empty((d, T), np.float32); assert L.wref_embd_conv(S.state, p(conv), conv.size) == conv.size
        enc = np.empty((T, d), np.float32); assert L.wref_embd_enc(S.state, p(enc), enc.size) == enc.size
        out = dict(conv=conv.T.copy(), enc=enc)
        for key, fn in (("kc", L.wref_kv_cross_k), ("kv", L.wref_kv_cross_v)):
            n = fn(S.state, None, 0)
            flat = np.empty(n, np.float16); assert fn(S.state, p(flat), n) == n
            # the reference's layer l starts at l * pad256(T) * d; its rows past T are not cleared between contexts and are not compared
            out[key] = np.stack([flat[l * Tp * d:l * Tp * d + T * d].reshape(T, d) for l in range(Lt)]).astype(np.float32)
        return out
    conv = np.empty((T, d), np.float32); enc = np.empty((T, d), np.float32)
    assert L.wb200_read_tensor(S.state, 1, p(conv), conv.size) == conv.size, L.wb200_last_error()
    assert L.wb200_read_tensor(S.state, 2, p(enc), enc.size) == enc.size
    out = dict(conv=conv, enc=enc)
    for key, which in (("kc", 3), ("kv", 4)):
        a = np.empty((Lt, TP_MAX, d), np.float32)
        assert L.wb200_read_tensor(S.state, which, p(a), a.size) == a.size
        out[key], out[key + "_pad"] = a[:, :T], a[:, T:]
    return out


@pytest.mark.parametrize("T", [512, 750, 1000])
@pytest.mark.parametrize("cfg,wt", [("test-2l.en", F16), ("test-2l.en", Q5_0), ("test-2l-512.en", Q4_K)])
def test_reduced_context_matches_reference(lib, ref, tmp_path, cfg, wt, T):
    path = _build(tmp_path, ref, cfg, wt)
    pcm = read_wav_f32(os.path.join(DATA_DIR, "jfk.wav"))
    os.environ["WB200_MEGAKERNEL"] = "1"
    A = Side(lib, path, False)
    os.environ["WB200_MEGAKERNEL"] = "0"
    B = Side(lib, path, False)
    os.environ.pop("WB200_MEGAKERNEL")
    R = Side(ref, path, True)                                     # a fresh reference context: no stale cross K/V rows of another T
    try:
        for S in (A, B):                                          # a full-context encode first: its rows T .. 1499 must not survive
            S.pcm_to_mel(pcm); S.encode(0)
        for S in (A, B, R):
            _set_audio_ctx(S, T)
            S.pcm_to_mel(pcm); S.encode(0)
        e_enc, e_kv, e_log, margin = TOL[wt]
        if A.d <= 256:
            e_enc, e_kv, e_log = 1.3 * e_enc, 1.3 * e_kv, 1.3 * e_log
        tr = _taps_at(R, T)
        for S in (A, B):
            ta = _taps_at(S, T)
            assert rms_err(ta["conv"], tr["conv"]) < 1e-3
            assert rms_err(ta["enc"], tr["enc"]) < e_enc
            assert rms_err(ta["kc"], tr["kc"]) < e_kv and rms_err(ta["kv"], tr["kv"]) < e_kv
            assert not ta["kc_pad"].any() and not ta["kv_pad"].any()        # exactly zero: attended to as zero keys up to pad256(T)
        sot = A.L.whisper_token_sot(A.ctx)
        toks, n_past = [sot], 0
        for step in range(10):
            feed = toks if step == 0 else toks[-1:]
            la, lb, lr = A.decode(feed, n_past), B.decode(feed, n_past), R.decode(feed, n_past)
            n_past += len(feed)
            e_mk, e_ch = rms_err(la - lr.mean(), lr - lr.mean()), rms_err(lb - lr.mean(), lr - lr.mean())
            assert np.isfinite(la).all() and np.isfinite(lb).all()
            assert e_ch < e_log, (step, e_ch)
            assert e_mk < e_log, (step, e_mk)
            assert e_mk < 1.25 * e_ch + 1e-3, (step, e_mk, e_ch)       # the persistent kernel is as close to the reference as the chain
            srt = np.sort(lr)
            if (srt[-1] - srt[-2]) / lr.std() > margin:
                assert int(la.argmax()) == int(lr.argmax()) == int(lb.argmax()), step
            toks.append(int(lr.argmax()))
    finally:
        A.free(); B.free(); R.free()


def _wide_run_ctx(L, path, pcm, T):
    ctx = _context(L, path, use_gpu=hasattr(L, "wb200_last_error"))
    script = Script(L, ctx, 77, "peaked")                         # alive until whisper_full returns: fp holds only its callback pointer
    fp = _params(L, script)
    fp.audio_ctx = T
    assert L.whisper_full(ctx, fp, pcm.ctypes.data_as(vp), len(pcm)) == 0
    return ctx


@pytest.mark.parametrize("wt,tol_ref", [(F16, 2e-2), (Q5_0, 8e-2)])
def test_dtw_at_reduced_context(lib, ref, tmp_path, wt, tol_ref):
    """large-v3 width at audio_ctx = 768: alignment weights of the persistent kernel against the kernel chain and the reference's
    aheads_cross_QKs, tolerances of test_dtw_pool_gpu.test_dtw_persistent_kernel_against_chain_and_reference"""
    T = 768
    L = _bind(lib)
    path = _model(tmp_path, WIDE, wt, 13, ref)
    pcm = synth.synth_audio(seed=5, seconds=14.0)
    runs = {}
    for mode in ("1", "0"):
        os.environ["WB200_MEGAKERNEL"] = mode
        try:
            ctx = _wide_run_ctx(L, path, pcm, T)
        finally:
            os.environ.pop("WB200_MEGAKERNEL")
        st = L.wb200_ctx_state(ctx)
        runs[mode] = (_result(L, st), *_qks(L, st))
        L.whisper_free(ctx)
    (res_mk, a, shape), (res_ch, b, shape_ch) = runs["1"], runs["0"]
    assert [[t[0] for t in s] for s in _tokens(res_mk)] == [[t[0] for t in s] for s in _tokens(res_ch)]
    assert shape == shape_ch and shape[1] == T and shape[2] == 40
    err = float(np.sqrt(((a - b) ** 2).mean()) / np.sqrt((b ** 2).mean()))
    print("wt %d: alignment weights %s at audio_ctx %d, persistent kernel vs chain relative rms %.2e" % (wt, shape, T, err))
    assert err < tol_ref / 2
    assert np.allclose(a.reshape(shape[2], shape[1], shape[0]).sum(axis=1), 1.0, atol=1e-4)
    R = _bind(ref)
    rctx = _wide_run_ctx(R, path, pcm, T)
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
        print("wt %d: vs reference relative rms %.2e" % (wt, err_ref))
        assert err_ref < tol_ref
    finally:
        R.whisper_free(rctx)


# ---- pool: states with different audio_ctx on one context -----------------------------------------------------------------------------
def _pool_params(L, ctx, mode, T, keep):
    """scripted: a fixed transcript with many text tokens (the alignment weights carry the cross-attention); greedy: the model's own
    tokens on the device sampler.  The Script goes to `keep`: fp holds only a pointer to its callback"""
    script = Script(L, ctx, 79, "peaked") if mode == "scripted" else None
    keep.append(script)
    fp = _params(L, script)
    fp.audio_ctx = T
    return fp


def _outcome(L, st):
    res = _result(L, st)
    qk, shape = _qks(L, st)
    return res, shape, qk.tobytes()


@pytest.mark.parametrize("mode", ["scripted", "greedy"])
def test_states_with_different_audio_ctx_share_the_pool(lib, tmp_path, mode):
    """three states with audio_ctx 768, 0 (1500) and 1000: run concurrently through whisper_full_with_state, each gives exactly what it
    gives alone -- tokens, segment times, t_dtw and the alignment weights of its last window.  DTW needs a window's frames within the
    context (2 T, as in the reference): clips of 14, 25 and 19 s"""
    L = _bind(lib)
    path = _model(tmp_path, SMALL, Q5_0, 9)
    ctx = _context(L, path)
    try:
        Ts = (768, 0, 1000)
        clips = [synth.synth_audio(seed=120 + i, seconds=s) for i, s in enumerate((14.0, 25.0, 19.0))]
        keep = []
        fps = [_pool_params(L, ctx, mode, T, keep) for T in Ts]
        states = [L.whisper_init_state(ctx) for _ in Ts]
        assert all(states), L.wb200_last_error()

        def work(i, rcs):
            rcs[i] = L.whisper_full_with_state(ctx, states[i], fps[i], clips[i].ctypes.data_as(vp), len(clips[i]))
        alone = []
        for i in range(3):
            rcs = [None] * 3
            work(i, rcs)
            assert rcs[i] == 0, L.wb200_last_error()
            alone.append(_outcome(L, states[i]))
        assert sum(len(s[2]) for r in alone for s in r[0]) > 10
        if mode == "scripted":
            assert all(o[1][0] > 0 and o[1][1] == (T or 1500) for o, T in zip(alone, Ts))
        rcs = [None] * 3
        th = [threading.Thread(target=work, args=(i, rcs)) for i in range(3)]
        for t in th: t.start()
        for t in th: t.join()
        assert rcs == [0] * 3, (rcs, L.wb200_last_error())
        for i in range(3):
            got = _outcome(L, states[i])
            assert got[0] == alone[i][0], (Ts[i], "tokens / segment times / t_dtw")
            assert got[1] == alone[i][1] and got[2] == alone[i][2], (Ts[i], "alignment weights")
        for s in states: L.whisper_free_state(s)
    finally:
        L.whisper_free(ctx)


def test_encode_at_another_context_leaves_running_states_alone(lib, tmp_path):
    """two states at audio_ctx 768 and 0 transcribe 70 s each; at the second window of the first, a third state at audio_ctx 1000 starts:
    the encodes of the newcomer at another context length must leave the cross K/V of the running states untouched.  Greedy on the
    device sampler, so every token depends on the cross-attention; DTW off (its windows would exceed 2 T frames)"""
    L = _bind(lib)
    path = _model(tmp_path, SMALL, Q5_0, 10)
    ctx = _context(L, path, dtw=False)
    try:
        Ts = (768, 0, 1000)
        clips = [synth.synth_audio(seed=140 + i, seconds=s) for i, s in enumerate((70.0, 70.0, 20.0))]
        keep = []
        fps = [_pool_params(L, ctx, "greedy", T, keep) for T in Ts]
        states = [L.whisper_init_state(ctx) for _ in Ts]
        assert all(states), L.wb200_last_error()
        rcs = [None] * 3

        def work(i):
            rcs[i] = L.whisper_full_with_state(ctx, states[i], fps[i], clips[i].ctypes.data_as(vp), len(clips[i]))
        alone = []
        for i in range(3):
            work(i)
            assert rcs[i] == 0, L.wb200_last_error()
            alone.append(_result(L, states[i]))
        windows, late = [], []
        ENC = C.CFUNCTYPE(C.c_bool, vp, vp, vp)

        def on_window(c, st, ud):
            windows.append(None)
            if len(windows) == 2:
                t = threading.Thread(target=work, args=(2,)); t.start(); late.append(t)
            return True
        cb = ENC(on_window)
        fps[0].encoder_begin_callback = C.cast(cb, vp)
        rcs[:] = [None] * 3
        th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
        for t in th: t.start()
        for t in th: t.join()
        for t in late: t.join()
        assert len(windows) >= 2 and len(late) == 1
        assert rcs == [0] * 3, (rcs, L.wb200_last_error())
        assert sum(len(s[2]) for r in alone for s in r) > 10
        for i in range(3):
            assert _result(L, states[i]) == alone[i], (Ts[i], "tokens / segment times")
        for s in states: L.whisper_free_state(s)
    finally:
        L.whisper_free(ctx)
