"""oracle/ref_numpy.py -- TEST INFRASTRUCTURE ONLY.  NumPy restatement of the reference arithmetic on the hot path.

Nothing under whisper.cpp_b200/ imports this module; only tests/, bench.py's cpu_baseline leg and
__graft_entry__.smoke() do, and only as a checker.

Pinning: every function here is checked in tests/test_oracle_cpu.py against the UNMODIFIED reference built from
/root/reference (oracle/_ref/libwhisper_ref.so): block decoders against ggml's own `to_float` traits, the Q8_0
activation quantiser + integer dot against ggml_quantize_chunk output, log-mel against `whisper_pcm_to_mel`, the
conv stem / encoder / cross K,V (EncoderOracle) and the decoder step (DecoderOracle) against the reference's own tensors and logits.  The reference ships no numeric golden vectors for this path
(SURVEY.md section 8c), so the compiled reference is the pin.

Citations are file:line in ggml-org/whisper.cpp @ 233fe1fc.
"""
import numpy as np

F32, F16, Q4_0, Q5_0, Q8_0, Q4_K, Q5_K = 0, 1, 2, 6, 8, 12, 13


# ----------------------------------------------------------------------------------------------------------------------
# block formats  (ggml/src/ggml-common.h:194-356, ggml/src/ggml-quants.c:459-567, 880-887, 1529-1551, 1731-1756)
# ----------------------------------------------------------------------------------------------------------------------
def _f16(b):
    return np.frombuffer(np.ascontiguousarray(b).tobytes(), dtype=np.float16).astype(np.float32)


def dequantize(wtype, raw, rows, k):
    """file bytes -> float32 [rows][k]; exact f32 arithmetic as dequantize_row_*"""
    raw = np.frombuffer(raw, dtype=np.uint8)
    if wtype == F16:
        return np.frombuffer(raw.tobytes(), dtype=np.float16).astype(np.float32).reshape(rows, k)
    if wtype == F32:
        return np.frombuffer(raw.tobytes(), dtype=np.float32).reshape(rows, k).copy()
    if wtype in (Q4_0, Q5_0, Q8_0):
        bs = {Q4_0: 18, Q5_0: 22, Q8_0: 34}[wtype]
        blk = raw.reshape(-1, bs)
        d = _f16(blk[:, 0:2]).reshape(-1, 1)
        if wtype == Q8_0:
            q = blk[:, 2:34].view(np.int8).astype(np.float32)
            return (q * d).reshape(rows, k)
        if wtype == Q4_0:
            qs = blk[:, 2:18]
            lo = (qs & 0xF).astype(np.int32) - 8
            hi = (qs >> 4).astype(np.int32) - 8
            return (np.concatenate([lo, hi], axis=1).astype(np.float32) * d).reshape(rows, k)
        qh = blk[:, 2:6].copy().view(np.uint32).reshape(-1, 1)
        qs = blk[:, 6:22]
        bits = (qh >> np.arange(32, dtype=np.uint32)[None, :]) & 1
        lo = ((qs & 0xF).astype(np.int32) | (bits[:, :16].astype(np.int32) << 4)) - 16
        hi = ((qs >> 4).astype(np.int32) | (bits[:, 16:].astype(np.int32) << 4)) - 16
        return (np.concatenate([lo, hi], axis=1).astype(np.float32) * d).reshape(rows, k)
    if wtype in (Q4_K, Q5_K):
        bs = 144 if wtype == Q4_K else 176
        blk = raw.reshape(-1, bs)
        d = _f16(blk[:, 0:2]); dmin = _f16(blk[:, 2:4])
        sc8 = blk[:, 4:16].astype(np.int32)
        sc = np.empty((blk.shape[0], 8), np.int32); mn = np.empty_like(sc)
        for j in range(8):                                   # get_scale_min_k4
            if j < 4:
                sc[:, j] = sc8[:, j] & 63; mn[:, j] = sc8[:, j + 4] & 63
            else:
                sc[:, j] = (sc8[:, j + 4] & 0xF) | ((sc8[:, j - 4] >> 6) << 4)
                mn[:, j] = (sc8[:, j + 4] >> 4) | ((sc8[:, j] >> 6) << 4)
        qoff = 16 + (32 if wtype == Q5_K else 0)
        qs = blk[:, qoff:qoff + 128].astype(np.int32)
        out = np.empty((blk.shape[0], 256), np.float32)
        for j in range(8):
            q = (qs[:, 32 * (j // 2):32 * (j // 2) + 32] >> (4 * (j & 1))) & 0xF
            if wtype == Q5_K:
                q = q | (((blk[:, 16:48].astype(np.int32) >> j) & 1) << 4)
            d1 = (d * sc[:, j].astype(np.float32)).astype(np.float32)[:, None]
            m1 = (dmin * mn[:, j].astype(np.float32)).astype(np.float32)[:, None]
            out[:, 32 * j:32 * j + 32] = d1 * q.astype(np.float32) - m1
        return out.reshape(rows, k)
    raise ValueError(wtype)


# ----------------------------------------------------------------------------------------------------------------------
# CPU mul_mat on quantised weights: activations -> Q8_0, integer dot per block
# (ggml-cpu/ggml-cpu.c:1181-1357; quantize_row_q8_0 AVX2 form ggml-cpu/arch/x86/quants.c; vec_dot ggml-cpu/quants.c:365-406)
# ----------------------------------------------------------------------------------------------------------------------
def quantize_q8_0(x):
    x = np.asarray(x, np.float32).reshape(-1, 32)
    amax = np.abs(x).max(axis=1, keepdims=True)
    d = (amax / np.float32(127.0)).astype(np.float32)
    idv = np.where(amax != 0, np.float32(127.0) / np.where(amax != 0, amax, 1), 0).astype(np.float32)
    q = np.rint(x * idv).astype(np.int32)                     # _MM_ROUND_NEAREST = ties to even
    return q, d.astype(np.float16).astype(np.float32)


def q8_0_bytes(x):
    """block_q8_0 records (ggml-common.h: f16 d, int8 qs[32]) of quantize_q8_0(x)"""
    q, d = quantize_q8_0(x)
    out = np.empty((q.shape[0], 34), np.uint8)
    out[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(-1, 2)
    out[:, 2:] = q.astype(np.int8).view(np.uint8)
    return out.tobytes()


def _block_ints(wtype, raw):
    raw = np.frombuffer(raw, dtype=np.uint8)
    bs = {Q4_0: 18, Q5_0: 22, Q8_0: 34}[wtype]
    blk = raw.reshape(-1, bs)
    d = _f16(blk[:, 0:2])
    if wtype == Q8_0:
        return blk[:, 2:34].view(np.int8).astype(np.int32), d
    if wtype == Q4_0:
        qs = blk[:, 2:18]
        return np.concatenate([(qs & 0xF).astype(np.int32) - 8, (qs >> 4).astype(np.int32) - 8], axis=1), d
    qh = blk[:, 2:6].copy().view(np.uint32).reshape(-1, 1)
    qs = blk[:, 6:22]
    bits = ((qh >> np.arange(32, dtype=np.uint32)[None, :]) & 1).astype(np.int32)
    lo = ((qs & 0xF).astype(np.int32) | (bits[:, :16] << 4)) - 16
    hi = ((qs >> 4).astype(np.int32) | (bits[:, 16:] << 4)) - 16
    return np.concatenate([lo, hi], axis=1), d


def mul_mat_q(wtype, raw, rows, k, x):
    """y[t][n] as ggml's CPU mul_mat computes it for Q4_0/Q5_0/Q8_0 weights (f32 sum over blocks in block order)."""
    x = np.asarray(x, np.float32).reshape(-1, k)
    wi, wd = _block_ints(wtype, raw)
    wi = wi.reshape(rows, k // 32, 32); wd = wd.reshape(rows, k // 32)
    out = np.empty((x.shape[0], rows), np.float32)
    for t in range(x.shape[0]):
        xq, xd = quantize_q8_0(x[t])
        sumi = np.einsum("nbk,bk->nb", wi, xq.reshape(k // 32, 32)).astype(np.float32)
        out[t] = (sumi * (wd * xd.reshape(1, -1))).astype(np.float32).sum(axis=1, dtype=np.float32)
    return out


def mul_mat_f16(raw, rows, k, x):
    """F16 weights: activations rounded to f16, f32 accumulation (ggml-cpu.c vec_dot_f16)"""
    w = np.frombuffer(raw, dtype=np.float16).astype(np.float32).reshape(rows, k)
    xh = np.asarray(x, np.float32).reshape(-1, k).astype(np.float16).astype(np.float32)
    return (xh.astype(np.float64) @ w.astype(np.float64).T).astype(np.float32)


# ----------------------------------------------------------------------------------------------------------------------
# element-wise pieces
# ----------------------------------------------------------------------------------------------------------------------
def gelu(x):
    """ggml_vec_gelu_f32 with GGML_GELU_FP16 (ggml-cpu/vec.h:46, 963-1001): f16 table lookup"""
    x = np.asarray(x, np.float32)
    xh = x.astype(np.float16).astype(np.float32)
    g = np.float32(0.5) * xh * (np.float32(1.0) + np.tanh(np.float32(0.79788456080286535587989211986876) * xh *
                                                         (np.float32(1.0) + np.float32(0.044715) * xh * xh)))
    g = g.astype(np.float16).astype(np.float32)
    return np.where(x <= -10, np.float32(0), np.where(x >= 10, x, g)).astype(np.float32)


def layernorm(x, w, b, eps=1e-5):
    """ggml_compute_forward_norm_f32 (ggml-cpu/ops.cpp:3698-3765) followed by mul + add (whisper.cpp:2108-2115)"""
    x = np.asarray(x, np.float32)
    mean = x.mean(axis=-1, keepdims=True, dtype=np.float32)
    y = x - mean
    var = (y * y).mean(axis=-1, keepdims=True, dtype=np.float32)
    return (y * (np.float32(1.0) / np.sqrt(var + np.float32(eps)))) * w + b


def attention(q, k, v, scale, n_zero_keys=0):
    """one head: softmax(scale * q k^T) v with `n_zero_keys` extra all-zero, UNMASKED keys (whisper.cpp:2148-2165)
    q is rounded to f16 like the CPU flash-attn path (ggml-cpu/ops.cpp:8590); f64 accumulation here."""
    qh = np.asarray(q, np.float32).astype(np.float16).astype(np.float64)
    s = (qh @ np.asarray(k, np.float64).T) * scale
    if n_zero_keys:
        s = np.concatenate([s, np.zeros((s.shape[0], n_zero_keys))], axis=1)
        v = np.concatenate([np.asarray(v, np.float64), np.zeros((n_zero_keys, v.shape[1]))], axis=0)
    m = s.max(axis=1, keepdims=True)
    p = np.exp(s - m)
    return ((p @ np.asarray(v, np.float64)) / p.sum(axis=1, keepdims=True)).astype(np.float32)


# ----------------------------------------------------------------------------------------------------------------------
# log-mel spectrogram (src/whisper.cpp:3005-3272) in float64 -- "exact" version used to bound both implementations
# ----------------------------------------------------------------------------------------------------------------------
def log_mel(pcm, filters):
    pcm = np.asarray(pcm, np.float64)
    n = pcm.shape[0]
    n_mel = filters.shape[0]
    padded = np.zeros(n + 480000 + 400)
    padded[200:200 + n] = pcm
    n_reflect = min(200, max(0, n - 1))
    if n_reflect:
        padded[200 - n_reflect:200] = pcm[1:1 + n_reflect][::-1]
    n_len = (padded.shape[0] - 400) // 160
    n_eff = n + 200
    n_comp = min(n_eff // 160 + 1, n_len)
    hann = 0.5 * (1.0 - np.cos(2.0 * np.pi * np.arange(400) / 400))
    mel = np.full((n_mel, n_len), -10.0)
    idx = np.arange(400)[None, :] + 160 * np.arange(n_comp)[:, None]
    frames = padded[idx]
    valid = idx < n_eff
    frames = np.where(valid, frames, 0.0) * hann[None, :]
    spec = np.abs(np.fft.rfft(frames, axis=1)) ** 2
    mel[:, :n_comp] = np.log10(np.maximum(filters.astype(np.float64) @ spec.T, 1e-10))
    mmax = mel.max() - 8.0
    mel = np.maximum(mel, mmax)
    return ((mel + 4.0) / 4.0).astype(np.float32)


# ----------------------------------------------------------------------------------------------------------------------
# model file (legacy ggml container, src/whisper.cpp:1485-1962) and the text decoder step (src/whisper.cpp:2466-2844)
# ----------------------------------------------------------------------------------------------------------------------
def read_model(path):
    """-> (hparams dict, {tensor name: (ggml type, shape as stored [rows, cols] or [n], raw bytes)})"""
    import struct
    with open(path, "rb") as f:
        blob = f.read()
    off = 0

    def rd(fmt):
        nonlocal off
        v = struct.unpack_from(fmt, blob, off)
        off += struct.calcsize(fmt)
        return v
    assert rd("<I")[0] == 0x67676d6c
    names = ["n_vocab", "n_audio_ctx", "n_audio_state", "n_audio_head", "n_audio_layer", "n_text_ctx", "n_text_state", "n_text_head", "n_text_layer", "n_mels", "ftype"]
    hp = dict(zip(names, rd("<11i")))
    n_mel, n_fft = rd("<2i")
    off += n_mel * n_fft * 4
    for _ in range(rd("<i")[0]):
        n_bytes = rd("<I")[0]                              # (rd advances `off`: read it before adding)
        off += n_bytes
    bpb = {F32: (1, 4), F16: (1, 2), Q4_0: (32, 18), Q5_0: (32, 22), Q8_0: (32, 34), Q4_K: (256, 144), Q5_K: (256, 176)}
    tensors = {}
    while off < len(blob):
        n_dims, length, ttype = rd("<3i")
        ne = list(rd("<%di" % n_dims))
        name = blob[off:off + length].decode(); off += length
        n = int(np.prod(ne))
        nbytes = n // bpb[ttype][0] * bpb[ttype][1]
        shape = [ne[1], ne[0]] if n_dims == 2 else ([ne[2], ne[1], ne[0]] if n_dims == 3 else [ne[0]])
        tensors[name] = (ttype, shape, blob[off:off + nbytes]); off += nbytes
    return hp, tensors


def _vec(t):
    ttype, shape, raw = t
    return (np.frombuffer(raw, np.float32) if ttype == F32 else np.frombuffer(raw, np.float16).astype(np.float32)).reshape(shape)


def _mul_mat(t, x):
    """ggml_mul_mat(W, x) as the CPU backend computes it for this weight type (ggml-cpu/ggml-cpu.c:1254-1452)"""
    ttype, (rows, k), raw = t
    if ttype == F16:
        return mul_mat_f16(raw, rows, k, x)
    if ttype == F32:
        return (np.asarray(x, np.float64).reshape(-1, k) @ np.frombuffer(raw, np.float32).reshape(rows, k).astype(np.float64).T).astype(np.float32)
    return mul_mat_q(ttype, raw, rows, k, x)


def _rows(t, ids):
    ttype, (rows, k), raw = t
    if ttype == F32:
        return np.frombuffer(raw, np.float32).reshape(rows, k)[ids]
    return dequantize(ttype, raw, rows, k)[ids]                 # get_rows on a quantised table dequantises exactly (ops.cpp:4850)


class DecoderOracle:
    """whisper_build_graph_decoder for ONE sequence, step by step (flash-attention path, CPU arithmetic):
    Q/K scaled by 64^-1/4, K/V stored as f16, Q rounded to f16 inside attention, cross-attention over all padded keys."""

    def __init__(self, path):
        self.hp, self.t = read_model(path)
        L, d = self.hp["n_text_layer"], self.hp["n_text_state"]
        self.k = [np.zeros((0, d), np.float32) for _ in range(L)]
        self.v = [np.zeros((0, d), np.float32) for _ in range(L)]

    def step(self, tokens, n_past, cross_k, cross_v):
        """tokens: ids fed in this call (positions n_past..); cross_k/v: [L][Tp][d] float32 views of the f16 cross KV.
        Returns the logits of the LAST fed token."""
        hp, t = self.hp, self.t
        d, H, L = hp["n_text_state"], hp["n_text_head"], hp["n_text_layer"]
        kq = np.float32(64.0) ** np.float32(-0.25)
        ids = np.asarray(tokens, np.int64)
        n = len(ids)
        x = _rows(t["decoder.token_embedding.weight"], ids) + _vec(t["decoder.positional_embedding"])[n_past:n_past + n]
        f16 = lambda a: np.asarray(a, np.float32).astype(np.float16).astype(np.float32)   # noqa: E731
        for l in range(L):
            p = "decoder.blocks.%d." % l
            cur = layernorm(x, _vec(t[p + "attn_ln.weight"]), _vec(t[p + "attn_ln.bias"]))
            q = (_mul_mat(t[p + "attn.query.weight"], cur) + _vec(t[p + "attn.query.bias"])) * kq
            k = _mul_mat(t[p + "attn.key.weight"], cur) * kq
            v = _mul_mat(t[p + "attn.value.weight"], cur) + _vec(t[p + "attn.value.bias"])
            self.k[l] = np.concatenate([self.k[l][:n_past], f16(k)]); self.v[l] = np.concatenate([self.v[l][:n_past], f16(v)])
            att = np.empty((n, d), np.float32)
            for i in range(n):                                   # causal: token i sees positions <= n_past + i
                nk = n_past + i + 1
                for h in range(H):
                    sl = slice(64 * h, 64 * h + 64)
                    att[i, sl] = attention(q[i:i + 1, sl], self.k[l][:nk, sl], self.v[l][:nk, sl], 1.0)[0]
            x = x + _mul_mat(t[p + "attn.out.weight"], att) + _vec(t[p + "attn.out.bias"])
            cur = layernorm(x, _vec(t[p + "cross_attn_ln.weight"]), _vec(t[p + "cross_attn_ln.bias"]))
            qc = _mul_mat(t[p + "cross_attn.query.weight"], cur) + _vec(t[p + "cross_attn.query.bias"])
            att = np.empty((n, d), np.float32)
            for h in range(H):
                sl = slice(64 * h, 64 * h + 64)
                att[:, sl] = attention(qc[:, sl], cross_k[l][:, sl], cross_v[l][:, sl], float(kq))    # all Tp keys, zero rows included
            x = x + _mul_mat(t[p + "cross_attn.out.weight"], att) + _vec(t[p + "cross_attn.out.bias"])
            cur = layernorm(x, _vec(t[p + "mlp_ln.weight"]), _vec(t[p + "mlp_ln.bias"]))
            hcur = gelu(_mul_mat(t[p + "mlp.0.weight"], cur) + _vec(t[p + "mlp.0.bias"]))
            x = x + _mul_mat(t[p + "mlp.2.weight"], hcur) + _vec(t[p + "mlp.2.bias"])
        cur = layernorm(x[-1:], _vec(t["decoder.ln.weight"]), _vec(t["decoder.ln.bias"]))
        return _mul_mat(t["decoder.token_embedding.weight"], cur)[0]


# ----------------------------------------------------------------------------------------------------------------------
# conv stem, encoder and cross K/V (src/whisper.cpp:1982-2042, 2044-2275, 2278-2354) on one 30-second window
# ----------------------------------------------------------------------------------------------------------------------
def _mul_mat_rows(t, x, chunk=128):
    """_mul_mat for many activation rows (the encoder has 1500): same arithmetic, evaluated in row chunks"""
    ttype, (rows, k), raw = t
    x = np.asarray(x, np.float32).reshape(-1, k)
    if ttype in (F16, F32):
        return _mul_mat(t, x)
    wi, wd = _block_ints(ttype, raw)
    wi = wi.reshape(rows, k // 32, 32).astype(np.float32); wd = wd.reshape(rows, k // 32)      # |sum of 32 products| < 2^24: exact in f32
    out = np.empty((x.shape[0], rows), np.float32)
    for r0 in range(0, x.shape[0], chunk):
        xs = x[r0:r0 + chunk]
        xq, xd = quantize_q8_0(xs.reshape(-1))
        xq = xq.reshape(len(xs), k // 32, 32).astype(np.float32); xd = xd.reshape(len(xs), k // 32)
        sumi = np.einsum("nbk,tbk->tnb", wi, xq)
        out[r0:r0 + chunk] = (sumi * (wd[None] * xd[:, None, :])).astype(np.float32).sum(axis=2, dtype=np.float32)
    return out


def conv1d_f16(w_t, x, stride):
    """ggml_conv_1d_ph (3 taps, padding 1) as the CPU backend runs it: im2col in F16, F16 x F16 products summed in f32
    (ggml/src/ggml.c ggml_conv_1d -> ggml_im2col(..., GGML_TYPE_F16) + ggml_mul_mat).  w_t: (type, [oc, ic, 3], raw); x: [ic][T] -> [oc][T/stride]"""
    ttype, (oc, ic, kw), raw = w_t
    assert kw == 3 and ttype in (F16, F32)
    w = (np.frombuffer(raw, np.float16) if ttype == F16 else np.frombuffer(raw, np.float32).astype(np.float16)).astype(np.float64).reshape(oc, ic, 3)
    xh = np.asarray(x, np.float32).astype(np.float16).astype(np.float64)
    T = xh.shape[1]
    xp = np.pad(xh, ((0, 0), (1, 1)))
    To = (T + 2 - 3) // stride + 1
    cols = np.stack([xp[:, k:k + stride * To:stride] for k in range(3)], axis=1)          # [ic][3][To]
    return np.einsum("oik,ikt->ot", w, cols).astype(np.float32)


class EncoderOracle:
    """whisper_build_graph_conv / _encoder / _cross for one window (flash-attention path, CPU arithmetic: F16 im2col, F16-rounded
    activations in front of F16 matrices / Q8_0 blocks in front of quantised ones, K and V of the attention rounded to F16 and padded with
    unmasked zero keys to 1536, f16-table GELU).  Accumulations are f64 here where the reference sums in f32 (or, for P.V of many query
    rows, in F16): the comparison with the compiled reference in tests/test_oracle_cpu.py carries that as its tolerance."""

    def __init__(self, path):
        self.hp, self.t = read_model(path)

    def conv(self, mel_window):
        """mel_window: [n_mels][2*n_ctx] f32 (frames past n_len zero, src/whisper.cpp:2389-2411) -> embd_conv [d][n_ctx]"""
        t = self.t
        x = conv1d_f16(t["encoder.conv1.weight"], mel_window, 1) + _vec(t["encoder.conv1.bias"]).reshape(-1, 1)
        x = gelu(x)
        x = conv1d_f16(t["encoder.conv2.weight"], x, 2) + _vec(t["encoder.conv2.bias"]).reshape(-1, 1)
        return gelu(x)

    def encode(self, embd_conv):
        """embd_conv [d][T] -> embd_enc [T][d]"""
        hp, t = self.hp, self.t
        d, H, L = hp["n_audio_state"], hp["n_audio_head"], hp["n_audio_layer"]
        T = embd_conv.shape[1]
        Tp = (T + 255) // 256 * 256                                                       # GGML_PAD(n_ctx, 256): 36 zero keys at T = 1500
        x = embd_conv.T + _vec(t["encoder.positional_embedding"])[:T]
        f16 = lambda a: np.asarray(a, np.float32).astype(np.float16).astype(np.float32)   # noqa: E731
        for l in range(L):
            p = "encoder.blocks.%d." % l
            cur = layernorm(x, _vec(t[p + "attn_ln.weight"]), _vec(t[p + "attn_ln.bias"]))
            q = _mul_mat_rows(t[p + "attn.query.weight"], cur) + _vec(t[p + "attn.query.bias"])
            k = f16(_mul_mat_rows(t[p + "attn.key.weight"], cur))
            v = f16(_mul_mat_rows(t[p + "attn.value.weight"], cur) + _vec(t[p + "attn.value.bias"]))
            att = np.empty((T, d), np.float32)
            for h in range(H):
                sl = slice(64 * h, 64 * h + 64)
                att[:, sl] = attention(q[:, sl], k[:, sl], v[:, sl], 1.0 / np.sqrt(64.0), n_zero_keys=Tp - T)
            x = x + _mul_mat_rows(t[p + "attn.out.weight"], att) + _vec(t[p + "attn.out.bias"])
            cur = layernorm(x, _vec(t[p + "mlp_ln.weight"]), _vec(t[p + "mlp_ln.bias"]))
            hcur = gelu(_mul_mat_rows(t[p + "mlp.0.weight"], cur) + _vec(t[p + "mlp.0.bias"]))
            x = x + _mul_mat_rows(t[p + "mlp.2.weight"], hcur) + _vec(t[p + "mlp.2.bias"])
        return layernorm(x, _vec(t["encoder.ln_post.weight"]), _vec(t["encoder.ln_post.bias"]))

    def cross(self, embd_enc):
        """-> (K [L][T][d], V [L][T][d]) as stored in kv_cross: K scaled by 64^-1/4 before the F16 rounding, V with bias"""
        hp, t = self.hp, self.t
        kq = np.float32(64.0) ** np.float32(-0.25)
        ks, vs = [], []
        for l in range(hp["n_text_layer"]):
            p = "decoder.blocks.%d." % l
            ks.append((_mul_mat_rows(t[p + "cross_attn.key.weight"], embd_enc) * kq).astype(np.float16).astype(np.float32))
            vs.append((_mul_mat_rows(t[p + "cross_attn.value.weight"], embd_enc) + _vec(t[p + "cross_attn.value.bias"])).astype(np.float16).astype(np.float32))
        return np.stack(ks), np.stack(vs)
