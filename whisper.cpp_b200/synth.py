"""Synthetic Whisper model files in the legacy "ggml" container (no network => no real checkpoints here).

Writes exactly the byte layout `models/convert-pt-to-ggml.py:268-339` produces and `whisper_model_load`
(src/whisper.cpp:1485-1962) reads: magic, 11 x i32 hparams, mel filters, vocabulary, then the tensor records with
reversed dims and no padding.  2-D weights are quantised like `whisper-quantize` does it
(examples/quantize/quantize.cpp:160-168, examples/common-ggml.cpp:141): every 2-D tensor except the conv biases and
the two positional embeddings; conv kernels stay F16, 1-D tensors F32; ftype in the header becomes 2000 + ftype.

The block quantisers restate ggml's reference quantisers (ggml/src/ggml-quants.c: quantize_row_q4_0_ref :113-147,
quantize_row_q5_0_ref :187-229, quantize_row_q8_0_ref :276-299, quantize_row_q4_1_ref :150-185, quantize_row_q5_1_ref :231-274);
tests/test_synth_cpu.py and tests/test_q8_1_cpu.py check them bit-for-bit against the compiled reference.  Host-side tooling only: no dependency on oracle/.
"""
import struct
import zlib

import numpy as np

F32, F16, Q4_0, Q5_0, Q8_0, Q4_K, Q5_K = 0, 1, 2, 6, 8, 12, 13
Q4_1, Q5_1 = 3, 7
Q2_K, Q3_K, Q6_K, BF16 = 10, 11, 14, 30              # Q2_K, Q6_K, BF16: no NumPy quantiser here (pass quantizer=, ggml's own via the oracle build)
FTYPE_OF = {F32: 0, F16: 1, Q4_0: 2, Q8_0: 7, Q5_0: 8, Q4_K: 12, Q5_K: 13, Q4_1: 3, Q5_1: 9, Q2_K: 10, Q3_K: 11, Q6_K: 14, BF16: 24}

CONFIGS = {
    # name: n_vocab, n_audio_ctx, n_audio_state, n_audio_head, n_audio_layer, n_text_ctx, n_text_state, n_text_head, n_text_layer, n_mels
    "tiny.en":        (51864, 1500, 384, 6, 4, 448, 384, 6, 4, 80),
    "base.en":        (51864, 1500, 512, 8, 6, 448, 512, 8, 6, 80),
    "large-v3":       (51866, 1500, 1280, 20, 32, 448, 1280, 20, 32, 128),
    "large-v3-turbo": (51866, 1500, 1280, 20, 32, 448, 1280, 20, 4, 128),
    # the large-v3 width (d = 1280, 20 heads, 128 mels, 51866 ids) at a depth the CPU reference finishes in seconds
    "large-v3-4l":    (51866, 1500, 1280, 20, 4, 448, 1280, 20, 4, 128),
    # reduced shapes for parity tests the CPU reference finishes in seconds
    "test-2l.en":     (51864, 1500, 384, 6, 2, 448, 384, 6, 2, 80),     # NB: 2 text layers + an English vocabulary = "distilled": whisper_full forces no_timestamps (whisper.cpp:7078-7084)
    "test-3l.en":     (51864, 1500, 384, 6, 2, 448, 384, 6, 3, 80),     # 3 text layers: timestamps stay on
    "test-2l-512.en": (51864, 1500, 512, 8, 2, 448, 512, 8, 2, 80),
    "test-3l-512.en": (51864, 1500, 512, 8, 2, 448, 512, 8, 3, 80),     # a K-quant width (d % 256 == 0) with timestamps on
    "test-2l-multi":  (51866, 1500, 256, 4, 2, 448, 256, 4, 2, 128),
    "small.en":       (51864, 1500, 768, 12, 12, 448, 768, 12, 12, 80),
    "test-2l-768.en": (51864, 1500, 768, 12, 2, 448, 768, 12, 2, 80),     # the small.en width at a depth the CPU reference finishes in seconds
}


# ----------------------------------------------------------------------------------------------------------------------
def mel_filters(n_mels, n_fft=400, sr=16000):
    """Slaney-style mel filterbank (what OpenAI's mel_filters.npz holds; librosa.filters.mel defaults)."""
    def hz_to_mel(f):
        f = np.asarray(f, np.float64)
        mels = f / (200.0 / 3)
        min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / (200.0 / 3), np.log(6.4) / 27.0
        return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, mels)

    def mel_to_hz(m):
        m = np.asarray(m, np.float64)
        f = m * (200.0 / 3)
        min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / (200.0 / 3), np.log(6.4) / 27.0
        return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f)

    fftfreqs = np.linspace(0, sr / 2, n_fft // 2 + 1)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(sr / 2), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, n_fft // 2 + 1))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return w.astype(np.float32)


# ----------------------------------------------------------------------------------------------------------------------
def quantize(wtype, w):
    """float32 [rows][k] -> file bytes"""
    w = np.ascontiguousarray(w, np.float32)
    if wtype == F32:
        return w.tobytes()
    if wtype == F16:
        return w.astype(np.float16).tobytes()
    x = w.reshape(-1, 32)
    nb = x.shape[0]
    if wtype == Q8_0:
        amax = np.abs(x).max(axis=1)
        d = (amax / np.float32(127.0)).astype(np.float32)
        idv = np.where(d != 0, np.float32(1.0) / np.where(d != 0, d, 1), 0).astype(np.float32)
        q = np.round(x * idv[:, None])  # roundf: half away from zero == np.round only for non-ties; fix ties below
        t = x * idv[:, None]
        q = np.where(np.abs(t - np.trunc(t)) == 0.5, np.trunc(t) + np.sign(t), np.rint(t)).astype(np.int8)
        out = np.empty((nb, 34), np.uint8)
        out[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(nb, 2)
        out[:, 2:] = q.view(np.uint8)
        return out.tobytes()
    # signed value of maximum magnitude (first occurrence, as the scalar loop finds it)
    idx = np.abs(x).argmax(axis=1)
    mx = x[np.arange(nb), idx]
    if wtype == Q4_0:
        d = (mx / np.float32(-8.0)).astype(np.float32)
        idv = np.where(d != 0, np.float32(1.0) / np.where(d != 0, d, 1), 0).astype(np.float32)
        t = (x * idv[:, None]).astype(np.float32) + np.float32(8.5)
        q = np.minimum(15, t.astype(np.int8).astype(np.int32)).astype(np.uint8)
        out = np.empty((nb, 18), np.uint8)
        out[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(nb, 2)
        out[:, 2:] = q[:, :16] | (q[:, 16:] << 4)
        return out.tobytes()
    if wtype == Q5_0:
        d = (mx / np.float32(-16.0)).astype(np.float32)
        idv = np.where(d != 0, np.float32(1.0) / np.where(d != 0, d, 1), 0).astype(np.float32)
        t = (x * idv[:, None]).astype(np.float32) + np.float32(16.5)
        q = np.minimum(31, t.astype(np.int8).astype(np.int32)).astype(np.uint32)
        out = np.empty((nb, 22), np.uint8)
        out[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(nb, 2)
        hi = (q >> 4) & 1
        qh = (hi << np.arange(32, dtype=np.uint32)[None, :]).sum(axis=1, dtype=np.uint64).astype(np.uint32)
        out[:, 2:6] = qh.view(np.uint8).reshape(nb, 4)
        out[:, 6:] = ((q[:, :16] & 0xF) | ((q[:, 16:] & 0xF) << 4)).astype(np.uint8)
        return out.tobytes()
    if wtype in (Q4_1, Q5_1):
        return quantize_q1(wtype, x)
    if wtype == Q4_K:
        return quantize_q4_k_simple(w)
    if wtype == Q3_K:
        return quantize_q3_k_simple(w)
    raise ValueError(f"synth.quantize: type {wtype} needs an external quantiser (pass quantizer=...)")


def quantize_q1(wtype, x):
    """[nb][32] float32 -> block_q4_1 / block_q5_1 bytes (quantize_row_q4_1_ref / _q5_1_ref): d = (max - min) / 15 (31), m = min,
    q = (x - min) * (1/d) + 0.5 truncated (Q4_1: capped at 15)"""
    nb = x.shape[0]
    mn = x.min(axis=1); mx = x.max(axis=1)
    d = ((mx - mn) / np.float32(15.0 if wtype == Q4_1 else 31.0)).astype(np.float32)
    idv = np.where(d != 0, np.float32(1.0) / np.where(d != 0, d, 1), 0).astype(np.float32)
    t = ((x - mn[:, None]).astype(np.float32) * idv[:, None]).astype(np.float32) + np.float32(0.5)
    q = t.astype(np.int32)
    out = np.empty((nb, 20 if wtype == Q4_1 else 24), np.uint8)
    out[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(nb, 2)
    out[:, 2:4] = mn.astype(np.float16).view(np.uint8).reshape(nb, 2)
    if wtype == Q4_1:
        q = np.minimum(15, q).astype(np.uint8)
        out[:, 4:] = q[:, :16] | (q[:, 16:] << 4)
        return out.tobytes()
    q = q.astype(np.uint32)
    qh = (((q >> 4) & 1) << np.arange(32, dtype=np.uint32)[None, :]).sum(axis=1, dtype=np.uint64).astype(np.uint32)
    out[:, 4:8] = qh.view(np.uint8).reshape(nb, 4)
    out[:, 8:] = ((q[:, :16] & 0xF) | ((q[:, 16:] & 0xF) << 4)).astype(np.uint8)
    return out.tobytes()


def quantize_q4_k_simple(w):
    """float32 [rows][k] -> block_q4_K bytes (ggml-common.h:327-340).  A plain min/max quantiser, NOT ggml's iterative make_qkx2_quants:
    every output is a valid Q4_K super-block that dequantises (ggml-quants.c:1529-1551) close to the input, which is all the multi-GB
    benchmark model of BASELINE config 3 needs; parity tests quantise with the reference's own ggml_quantize_chunk instead."""
    x = np.ascontiguousarray(w, np.float32).reshape(-1, 8, 32)
    nb = x.shape[0]
    mn = np.minimum(x.min(axis=2), 0.0); mx = x.max(axis=2)
    mf = -mn                                                    # >= 0
    sf = np.maximum((mx + mf) / np.float32(15.0), 1e-12)
    d = (sf.max(axis=1) / np.float32(63.0)).astype(np.float16).astype(np.float32); d = np.where(d > 0, d, 1e-8).astype(np.float32)
    dmin = (mf.max(axis=1) / np.float32(63.0)).astype(np.float16).astype(np.float32); dmin_safe = np.where(dmin > 0, dmin, 1.0).astype(np.float32)
    sc = np.clip(np.rint(sf / d[:, None]), 1, 63).astype(np.uint8)
    m = np.clip(np.rint(mf / dmin_safe[:, None]), 0, 63).astype(np.uint8)
    q = np.clip(np.rint((x + (dmin[:, None] * m)[:, :, None]) / (d[:, None] * sc)[:, :, None]), 0, 15).astype(np.uint8)
    out = np.zeros((nb, 144), np.uint8)
    out[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(nb, 2)
    out[:, 2:4] = dmin.astype(np.float16).view(np.uint8).reshape(nb, 2)
    scales = np.zeros((nb, 12), np.uint8)
    for j in range(4):
        scales[:, j] = (sc[:, j] & 63) | ((sc[:, j + 4] >> 4) << 6)
        scales[:, j + 4] = (m[:, j] & 63) | ((m[:, j + 4] >> 4) << 6)
        scales[:, j + 8] = (sc[:, j + 4] & 0xF) | ((m[:, j + 4] & 0xF) << 4)
    out[:, 4:16] = scales
    for jp in range(4):                                          # 64 values per 32 bytes: low nibbles = sub-block 2jp, high = 2jp+1
        out[:, 16 + 32 * jp:16 + 32 * (jp + 1)] = q[:, 2 * jp] | (q[:, 2 * jp + 1] << 4)
    return out.tobytes()


def _kq_signed_scales(x, qmax, smax):
    """[nb][256] -> (f16 d [nb], integer scales [nb][16] in 0 .. smax, q [nb][256] in -qmax .. qmax - 1): one scale per 16 values"""
    g = x.reshape(-1, 16, 16)
    s = np.abs(g).max(axis=2) / np.float32(qmax)
    d = (s.max(axis=1) / np.float32(smax)).astype(np.float16).astype(np.float32)
    sc = np.clip(np.rint(s / np.where(d > 0, d, 1.0)[:, None]), 0, smax).astype(np.int32)
    step = (d[:, None] * sc).astype(np.float32)
    q = np.clip(np.rint(g / np.where(step > 0, step, 1.0)[:, :, None]), -qmax, qmax - 1).astype(np.int32)
    return d, sc, q.reshape(-1, 256)


def quantize_q3_k_simple(w):
    """float32 [rows][k] -> block_q3_K bytes (hmask[32] qs[64] packed 6-bit scales[12] f16 d).  A plain absmax quantiser, not ggml's
    make_q3_quants search: valid super-blocks that dequantise (dequantize_row_q3_K) close to the input, for the benchmark models; parity
    tests quantise with the reference's own ggml_quantize_chunk."""
    x = np.ascontiguousarray(w, np.float32).reshape(-1, 256)
    nb = x.shape[0]
    d, sc, q = _kq_signed_scales(x, 4, 31)
    u = (q + 4).astype(np.uint8)                                 # q = (u & 3) - (hmask bit ? 0 : 4)
    out = np.zeros((nb, 110), np.uint8)
    for n in range(2):
        for r in range(4):
            v = u[:, 128 * n + 32 * r:128 * n + 32 * r + 32]
            out[:, 32 + 32 * n:64 + 32 * n] |= (v & 3) << (2 * r)
            out[:, 0:32] |= (v >> 2) << (4 * n + r)
    st = (sc + 32).astype(np.uint8)                              # stored 6-bit scale = sc + 32
    for k in range(4):
        for i in range(4):
            v = st[:, 4 * k + i]
            out[:, 96 + (k & 1) * 4 + i] |= (v & 0xF) << (4 * (k >> 1))
            out[:, 104 + i] |= (v >> 4) << (2 * k)
    out[:, 108:110] = d.astype(np.float16).view(np.uint8).reshape(nb, 2)
    return out.tobytes()


# ----------------------------------------------------------------------------------------------------------------------
def tensor_list(cfg):
    """(name, shape as torch would have it, kind) in the order whisper_model_load creates them; kind: 'mat','vec','conv','pos','cbias'"""
    n_vocab, n_actx, d, n_ah, La, n_tctx, dt, n_th, Lt, n_mels = cfg
    out = [("encoder.positional_embedding", (n_actx, d), "pos"),
           ("encoder.conv1.weight", (d, n_mels, 3), "conv"), ("encoder.conv1.bias", (d, 1), "cbias"),
           ("encoder.conv2.weight", (d, d, 3), "conv"), ("encoder.conv2.bias", (d, 1), "cbias"),
           ("encoder.ln_post.weight", (d,), "lnw"), ("encoder.ln_post.bias", (d,), "vec")]
    for i in range(La):
        p = f"encoder.blocks.{i}."
        out += [(p + "mlp_ln.weight", (d,), "lnw"), (p + "mlp_ln.bias", (d,), "vec"),
                (p + "mlp.0.weight", (4 * d, d), "mat"), (p + "mlp.0.bias", (4 * d,), "vec"),
                (p + "mlp.2.weight", (d, 4 * d), "mat"), (p + "mlp.2.bias", (d,), "vec"),
                (p + "attn_ln.weight", (d,), "lnw"), (p + "attn_ln.bias", (d,), "vec"),
                (p + "attn.query.weight", (d, d), "mat"), (p + "attn.query.bias", (d,), "vec"),
                (p + "attn.key.weight", (d, d), "mat"),
                (p + "attn.value.weight", (d, d), "mat"), (p + "attn.value.bias", (d,), "vec"),
                (p + "attn.out.weight", (d, d), "mat"), (p + "attn.out.bias", (d,), "vec")]
    out += [("decoder.positional_embedding", (n_tctx, dt), "pos"),
            ("decoder.token_embedding.weight", (n_vocab, dt), "mat"),
            ("decoder.ln.weight", (dt,), "lnw"), ("decoder.ln.bias", (dt,), "vec")]
    for i in range(Lt):
        p = f"decoder.blocks.{i}."
        out += [(p + "mlp_ln.weight", (dt,), "lnw"), (p + "mlp_ln.bias", (dt,), "vec"),
                (p + "mlp.0.weight", (4 * dt, dt), "mat"), (p + "mlp.0.bias", (4 * dt,), "vec"),
                (p + "mlp.2.weight", (dt, 4 * dt), "mat"), (p + "mlp.2.bias", (dt,), "vec"),
                (p + "attn_ln.weight", (dt,), "lnw"), (p + "attn_ln.bias", (dt,), "vec"),
                (p + "attn.query.weight", (dt, dt), "mat"), (p + "attn.query.bias", (dt,), "vec"),
                (p + "attn.key.weight", (dt, dt), "mat"),
                (p + "attn.value.weight", (dt, dt), "mat"), (p + "attn.value.bias", (dt,), "vec"),
                (p + "attn.out.weight", (dt, dt), "mat"), (p + "attn.out.bias", (dt,), "vec"),
                (p + "cross_attn_ln.weight", (dt,), "lnw"), (p + "cross_attn_ln.bias", (dt,), "vec"),
                (p + "cross_attn.query.weight", (dt, dt), "mat"), (p + "cross_attn.query.bias", (dt,), "vec"),
                (p + "cross_attn.key.weight", (dt, dt), "mat"),
                (p + "cross_attn.value.weight", (dt, dt), "mat"), (p + "cross_attn.value.bias", (dt,), "vec"),
                (p + "cross_attn.out.weight", (dt, dt), "mat"), (p + "cross_attn.out.bias", (dt,), "vec")]
    return out


def read_vocab_blob(stub_path):
    """raw bytes of the vocabulary section (i32 count + (u32 len, bytes)*) of an existing legacy model file"""
    with open(stub_path, "rb") as f:
        data = f.read()
    off = 4 + 44
    n_mel, n_fft = struct.unpack_from("<2i", data, off)
    off += 8 + n_mel * n_fft * 4
    start = off
    n, = struct.unpack_from("<i", data, off)
    off += 4
    for _ in range(n):
        ln, = struct.unpack_from("<I", data, off)
        off += 4 + ln
    return data[start:off]


def synthetic_vocab_blob(n):
    """n distinct printable tokens; token 220 is " " (needed by suppress_blank, src/whisper.cpp:6238)"""
    parts = [struct.pack("<i", n)]
    for i in range(n):
        s = b" " if i == 220 else (b" w%d" % i if i % 3 else b"w%d" % i)
        parts.append(struct.pack("<I", len(s)) + s)
    return b"".join(parts)


def write_model(path, config="test-2l.en", wtype=F16, seed=0, sigma=0.02, vocab_from=None, quantizer=None, fast_pool=False, scale=None):
    """Write a synthetic model.  Weights: matrices/embeddings N(0, sigma^2), LN weight 1+N(0,.02^2), biases N(0,.02^2),
    per-tensor seed = crc32(name) ^ seed (SURVEY.md section 8d).  fast_pool=True draws matrix blocks from one pre-quantised
    pool of 2^22 values (for the multi-GB benchmark models; same marginal distribution, seconds instead of minutes).
    scale: optional function name -> multiplier applied to that tensor's values (conditioned test models, see CONDITIONED)."""
    cfg = CONFIGS[config] if isinstance(config, str) else tuple(config)
    n_vocab, n_actx, d, n_ah, La, n_tctx, dt, n_th, Lt, n_mels = cfg
    q = quantizer or quantize
    ftype = FTYPE_OF[wtype] + (2000 if wtype not in (F32, F16) else 0)
    blk = {Q4_0: (32, 18), Q5_0: (32, 22), Q8_0: (32, 34), Q4_1: (32, 20), Q5_1: (32, 24), Q4_K: (256, 144), Q5_K: (256, 176), Q3_K: (256, 110)}.get(wtype)
    pool = None
    if fast_pool:
        prng = np.random.default_rng(seed ^ 0x5EED)
        pool_w = (prng.standard_normal(1 << 22) * sigma).astype(np.float32)
        if blk:
            pool = np.frombuffer(q(wtype, pool_w.reshape(-1, blk[0])), dtype=np.uint8).reshape(-1, blk[1])
        elif wtype == F16:
            pool = pool_w.astype(np.float16).reshape(-1, 32)
        else:
            pool = pool_w.reshape(-1, 32)
    with open(path, "wb") as f:
        f.write(struct.pack("<I", 0x67676d6c))
        f.write(struct.pack("<11i", n_vocab, n_actx, d, n_ah, La, n_tctx, dt, n_th, Lt, n_mels, ftype))
        filt = mel_filters(n_mels)
        f.write(struct.pack("<2i", n_mels, 201))
        f.write(filt.tobytes())
        if vocab_from:
            f.write(read_vocab_blob(vocab_from))
        else:
            f.write(synthetic_vocab_blob(n_vocab - (1 if n_vocab >= 51865 else 0) * 0))
        for name, shape, kind in tensor_list(cfg):
            rng = np.random.default_rng((zlib.crc32(name.encode()) ^ seed) & 0xFFFFFFFF)
            n_el = int(np.prod(shape))
            mul = np.float32(scale(name)) if scale else np.float32(1.0)
            if kind == "mat":
                ttype = wtype
                if pool is not None and mul == 1.0:
                    per = pool.shape[1] if not blk else blk[0]
                    nblk = n_el // (blk[0] if blk else 32)
                    idx = rng.integers(0, pool.shape[0], size=nblk)
                    data = pool[idx].tobytes()
                else:
                    data = q(wtype, (rng.standard_normal(shape) * sigma).astype(np.float32) * mul)
            elif kind == "conv":
                ttype = F16 if wtype != F32 else F32
                w = (rng.standard_normal(shape) * sigma * 2).astype(np.float32)
                data = w.astype(np.float16).tobytes() if ttype == F16 else w.tobytes()
            elif kind == "pos":
                ttype = F32
                data = (rng.standard_normal(shape) * sigma).astype(np.float32).tobytes()
            elif kind == "lnw":
                ttype = F32
                data = ((1.0 + rng.standard_normal(shape) * 0.02).astype(np.float32) * mul).tobytes()
            else:
                ttype = F32
                data = ((rng.standard_normal(shape) * 0.02).astype(np.float32) * mul).tobytes()
            nb = name.encode()
            f.write(struct.pack("<3i", len(shape), len(nb), ttype))
            for dim in reversed(shape):
                f.write(struct.pack("<i", dim))
            f.write(nb)
            f.write(data)
    return path


def conditioned(name, attn=1e-2, gain=100.0):
    """`scale` function of a WELL-CONDITIONED test model (tests/test_exact_tokens_gpu.py).  Random weights give logits whose top-2
    gap is routinely below the ~1e-2 relative noise between two arithmetic paths, so free-running transcripts of two correct
    implementations part ways at the first near-tie.  Two changes make the decode deterministic in the sense a trained model is:
      * the value projections of the text decoder's self- and cross-attention are scaled by `attn`: what attention adds to the residual
        stream (the part of the decoder whose reference arithmetic -- F16 accumulators in ggml's CPU flash attention, per-thread KV
        chunks, int8 activations in the encoder -- cannot be reproduced bit for bit) is attenuated but not removed: different audio
        still changes the transcript;
      * the final LayerNorm gain is multiplied by `gain`: logits spread over tens of nats, so softmax is peaked and the categorical
        draws of beam search land on the same ids unless a probability boundary moves by more than ~1e-6."""
    if name.startswith("decoder.") and ("attn.value.weight" in name or "attn.value.bias" in name):
        return attn
    if name in ("decoder.ln.weight", "decoder.ln.bias"):
        return gain
    return 1.0


def cached_model(config, wtype, seed=0, fast_pool=False, tag=None):
    """a synthetic model in the temp directory, written once per box (the multi-GB ones take a while); returns its path"""
    import os
    import tempfile
    names = {F16: "f16", Q4_0: "q4_0", Q5_0: "q5_0", Q8_0: "q8_0", Q4_K: "q4_k", Q4_1: "q4_1", Q5_1: "q5_1", Q3_K: "q3_k"}
    path = os.path.join(tempfile.gettempdir(), "wb200-%s-%s%s.bin" % (config, names[wtype], ("-" + tag) if tag else ""))
    if not os.path.exists(path):
        tmp = path + ".tmp.%d" % os.getpid()
        write_model(tmp, config, wtype, seed=seed, fast_pool=fast_pool)
        os.replace(tmp, path)
    return path


def synth_audio(seed=1234, seconds=30.0, sr=16000):
    """SURVEY.md section 8d, config 2: sum of 8 sinusoids 80-3800 Hz with random phases x slow AM + N(0, 0.01^2), peak 0.5"""
    rng = np.random.default_rng(seed)
    n = int(seconds * sr)
    t = np.arange(n) / sr
    x = np.zeros(n)
    for f0 in rng.uniform(80, 3800, size=8):
        x += np.sin(2 * np.pi * f0 * t + rng.uniform(0, 2 * np.pi)) * (0.5 + 0.5 * np.sin(2 * np.pi * rng.uniform(0.1, 2.0) * t + rng.uniform(0, 6.28)))
    x += rng.standard_normal(n) * 0.01
    x *= 0.5 / np.abs(x).max()
    return x.astype(np.float32)
