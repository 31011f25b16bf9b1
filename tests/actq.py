"""The persistent decode kernel's quantised activation rows ("actq", wb_decode_mk.cu) built from the reference's activation records, and
read back.  A buffer holds the pass's 64 rows: the row values [64][K] (int8; F16 weights: f16), then one K/8-byte record per row:
  Q8_0 (Q4_0 / Q5_0 / Q8_0 weights): f32 d[K/32]                (block_q8_0: f16 d, int8 qs[32])
  Q8_1 (Q4_1 / Q5_1):                {f16 d, f16 s}[K/32]       (block_q8_1: f16 d, f16 s, int8 qs[32])
  Q8_K (Q3_K / Q4_K / Q5_K):         f32 d[K/256] | int16 sum[K/32] of each 32 values (block_q8_K: f32 d, int8 qs[256], int16 bsums[16])
F16 rows have no record.  Test infrastructure only.
"""
import numpy as np

ROWS = 64
F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q3_K, Q4_K, Q5_K = 1, 2, 3, 6, 7, 8, 11, 12, 13
KQ = (Q3_K, Q4_K, Q5_K)
Q1 = (Q4_1, Q5_1)


def row_format(wtype):
    return "f16" if wtype == F16 else "q8_k" if wtype in KQ else "q8_1" if wtype in Q1 else "q8_0"


def nbytes(wtype, K):
    return ROWS * K * 2 if wtype == F16 else ROWS * K + ROWS * (K // 8)


def _rows_of(fmt, blocks, K):
    """one row of reference activation records -> (row bytes [K or 2K], record bytes [K/8] or None)"""
    b = np.frombuffer(blocks, np.uint8)
    if fmt == "f16":
        return b.copy(), None
    if fmt == "q8_0":
        blk = b.reshape(-1, 34)
        d = blk[:, 0:2].copy().view(np.float16).astype(np.float32).reshape(-1)
        return blk[:, 2:].reshape(-1).copy(), d.view(np.uint8)
    if fmt == "q8_1":
        blk = b.reshape(-1, 36)
        return blk[:, 4:].reshape(-1).copy(), blk[:, 0:4].reshape(-1).copy()
    blk = b.reshape(-1, 292)
    sums = blk[:, 260:].copy().view(np.int16).astype(np.int32).reshape(-1, 8, 2).sum(axis=2).astype(np.int16)
    return blk[:, 4:260].reshape(-1).copy(), np.concatenate([blk[:, 0:4].reshape(-1), sums.reshape(-1).view(np.uint8)])


def pack(wtype, K, rows):
    """rows: {row index: reference activation records of that row (bytes; F16: the f16 values)} -> actq buffer (uint8); other rows zero"""
    fmt = row_format(wtype)
    out = np.zeros(nbytes(wtype, K), np.uint8)
    rb = 2 * K if fmt == "f16" else K
    for t, blocks in rows.items():
        v, rec = _rows_of(fmt, blocks, K)
        out[t * rb:(t + 1) * rb] = v
        if rec is not None:
            out[ROWS * K + t * (K // 8):ROWS * K + t * (K // 8) + len(rec)] = rec      # Q8_K: 5K/64 bytes used of K/8
    return out


def unpack(wtype, K, buf, t):
    """row t of an actq buffer -> dict: q (int64 [K]; F16: f32 values), and d (f32 per block / super-block), s (Q8_1, f32), sum (Q8_K)"""
    fmt = row_format(wtype)
    buf = np.asarray(buf, np.uint8)
    if fmt == "f16":
        return {"q": buf[t * 2 * K:(t + 1) * 2 * K].view(np.float16).astype(np.float32)}
    q = buf[t * K:(t + 1) * K].view(np.int8).astype(np.int64)
    rec = buf[ROWS * K + t * (K // 8):ROWS * K + (t + 1) * (K // 8)]
    if fmt == "q8_0":
        return {"q": q, "d": rec.view(np.float32).copy()}
    if fmt == "q8_1":
        h = rec.view(np.float16).astype(np.float32).reshape(-1, 2)
        return {"q": q, "d": h[:, 0].copy(), "s": h[:, 1].copy()}
    o = K // 256 * 4
    return {"q": q, "d": rec[:o].view(np.float32).copy(), "sum": rec[o:o + K // 16].view(np.int16).astype(np.int64)}
