"""The persistent decode kernel (wb_decode_mk.cu) phase by phase, through its probe (wb200_dbg_mk_phase): one phase function run on a view
(CTA count, first row, rows) chosen here, with weights repacked tile-major as the engine does.

GEMV phases take their activation rows as actq bytes built from the reference's activation records (tests/actq.py), so the integer dot
is checked apart from the quantisers, against the reference's arithmetic on the same ints (oracle/ref_numpy.py, tests/q1_ref.py,
tests/kq_signed_ref.py; each pinned to the compiled reference's from_float / vec_dot on the CPU) at 2e-5 of the output scale: only the
f32 summation order differs.  The quantisers are checked against the reference's from_float bytes, attention against a float64 softmax.
"""
import ctypes as C
import functools

import numpy as np
import pytest

import actq
import kq_signed_ref as kq
import q1_ref as q1
from oracle import ref_numpy as rn

pytestmark = pytest.mark.gpu
vp = C.c_void_p
F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q3_K, Q4_K, Q5_K = actq.F16, actq.Q4_0, actq.Q4_1, actq.Q5_0, actq.Q5_1, actq.Q8_0, actq.Q3_K, actq.Q4_K, actq.Q5_K
ALL = [F16, Q4_0, Q5_0, Q8_0, Q4_1, Q5_1, Q3_K, Q4_K, Q5_K]
BLOCK32 = [Q4_0, Q5_0, Q8_0, Q4_1, Q5_1]
LNQ, Q8K, GEMV, PAIR, LOGITS_WARP, ATTN_SELF, ATTN_CROSS = range(7)
SENT_F32 = np.uint32(0x7FC0DEAD)                                 # a NaN no phase writes
SENT_F16 = np.uint16(0x7E5A)


class Io(C.Structure):
    _fields_ = [("wtype", C.c_int), ("phase", C.c_int), ("n_cta", C.c_int), ("row0", C.c_int), ("n_tok", C.c_int),
                ("N", C.c_int), ("K", C.c_int), ("lds", C.c_int), ("act", C.c_int), ("kv_d", C.c_int),
                ("w_file", vp), ("inp", vp), ("in_bytes", C.c_int64), ("bias", vp), ("scale", vp), ("res", vp),
                ("out", vp), ("out_bytes", C.c_int64), ("cell", vp), ("kc", vp), ("vc", vp), ("n_cells", C.c_int),
                ("d", C.c_int), ("n_head", C.c_int), ("ld_idx", C.c_int), ("nkv", vp), ("idx", vp),
                ("xk", vp), ("xv", vp), ("n_keys", C.c_int), ("n_slots", C.c_int), ("slot", vp), ("kq_scale", C.c_float), ("eps", C.c_float),
                ("kv_rows", C.c_int)]


def _p(a):
    return None if a is None else a.ctypes.data_as(vp)


def probe(lib, wtype, phase, n_cta, row0, n_tok, out, inp, **kw):
    """run one phase; `out` (numpy, sentinel-filled by the caller) is updated in place"""
    io = Io(wtype=wtype, phase=phase, n_cta=n_cta, row0=row0, n_tok=n_tok, inp=_p(inp), in_bytes=inp.nbytes, out=_p(out), out_bytes=out.nbytes)
    for k, v in kw.items():
        setattr(io, k, _p(v) if isinstance(v, np.ndarray) else v)
    rc = lib.wb200_dbg_mk_phase(C.byref(io))
    assert rc == 0, (rc, lib.wb200_last_error())


# ---- weights: random file blocks with sane scales (every bit pattern of the quants and of the 6-bit scales occurs) ----------------------
_BB = {Q4_0: 18, Q5_0: 22, Q8_0: 34, Q4_1: 20, Q5_1: 24, Q3_K: 110, Q4_K: 144, Q5_K: 176}
_BK = {Q3_K: 256, Q4_K: 256, Q5_K: 256}


@functools.lru_cache(maxsize=4)
def weights(wtype, N, K, seed=0):
    rng = np.random.default_rng([wtype, N, K, seed])
    if wtype == F16:
        return (rng.standard_normal((N, K)) * 0.05).astype(np.float16).tobytes()
    blk = rng.integers(0, 256, (N * K // _BK.get(wtype, 32), _BB[wtype]), dtype=np.uint8)
    d = lambda lo, hi, neg=False: (rng.uniform(lo, hi, len(blk)) * (rng.choice([-1, 1], len(blk)) if neg else 1)).astype(np.float16).view(np.uint8).reshape(-1, 2)  # noqa: E731
    if wtype == Q3_K:
        blk[:, 108:110] = d(2e-3, 6e-3)
    elif wtype in (Q4_K, Q5_K):
        blk[:, 0:2] = d(2e-4, 8e-4); blk[:, 2:4] = d(2e-4, 8e-4)
    else:
        blk[:, 0:2] = d(5e-3, 2e-2, neg=True)
        if wtype in (Q4_1, Q5_1):
            blk[:, 2:4] = d(5e-2, 2e-1, neg=True)
    return blk.tobytes()


def _rows_of(wtype, raw, N, K, rows):
    rb = len(raw) // N
    return b"".join(raw[r * rb:(r + 1) * rb] for r in rows)


# ---- activation rows ----------------------------------------------------------------------------------------------------------------------
def ref_records(wtype, x):
    """the reference's activation records of the f32 row x for weights of type wtype (NumPy from_float, pinned on the CPU)"""
    fmt = actq.row_format(wtype)
    if fmt == "f16":
        return np.asarray(x, np.float32).astype(np.float16).tobytes()
    return {"q8_0": rn.q8_0_bytes, "q8_1": q1.q8_1_bytes, "q8_k": kq.q8_k_bytes}[fmt](x)


def act_rows(wtype, K, seed, n=actq.ROWS):
    rng = np.random.default_rng([wtype, K, seed])
    X = (rng.standard_normal((n, K)) * rng.uniform(0.3, 3.0, (n, 1))).astype(np.float32)
    return X, actq.pack(wtype, K, {t: ref_records(wtype, X[t]) for t in range(n)})


def oracle(wtype, raw, N, K, buf, rows):
    """y [len(rows)][N] (float64) and the sum of the terms' magnitudes, from the actq rows `rows` of buf and the weight file bytes"""
    U = [actq.unpack(wtype, K, buf, t) for t in rows]
    T = len(rows)
    if wtype == F16:
        w = np.frombuffer(raw, np.float16).astype(np.float64).reshape(N, K)
        x = np.stack([u["q"] for u in U]).astype(np.float64)
        return x @ w.T, np.abs(x) @ np.abs(w).T
    xq = np.stack([u["q"] for u in U]).astype(np.float32)
    xd = np.stack([u["d"] for u in U]).astype(np.float64)
    if wtype in actq.KQ:
        return kq.dot_q8_k(wtype, raw, N, K, xq, xd.astype(np.float32))
    if wtype in actq.Q1:
        wi, wd, wm = q1.block_ints(wtype, raw)
    else:
        (wi, wd), wm = rn._block_ints(wtype, raw), None
    nb = K // 32
    sumi = np.matmul(wi.astype(np.float32).reshape(N, nb, 32).transpose(1, 0, 2), xq.reshape(T, nb, 32).transpose(1, 2, 0)).transpose(2, 1, 0)
    a = sumi.astype(np.float64) * (wd.reshape(1, N, nb).astype(np.float64) * xd[:, None, :])
    y, mag = a.sum(axis=2), np.abs(a).sum(axis=2)
    if wm is not None:
        xs = np.stack([u["s"] for u in U]).astype(np.float64)
        b = wm.reshape(1, N, nb).astype(np.float64) * xs[:, None, :]
        y, mag = y + b.sum(axis=2), mag + np.abs(b).sum(axis=2)
    return y, mag


def f32_out(n):
    return np.full((actq.ROWS, n), SENT_F32, np.uint32).view(np.float32)


def untouched(out, rows):
    """every row outside `rows` still holds the sentinel"""
    mask = np.ones(out.shape[0], bool); mask[list(rows)] = False
    return (out.view(np.uint32)[mask] == SENT_F32).all()


# ---- GEMV phases ------------------------------------------------------------------------------------------------------------------------
SHAPES = {"qkv": (3, 1), "o": (1, 1), "fc1": (4, 1), "fc2": (1, 4)}
N_TOK = [1, 2, 7, 8, 9, 15, 16, 17, 33, 64]


def _views(wtype, d, shape, K):
    """(n_tok, row0, n_cta) cases of one test: every n_tok of N_TOK over the tests of a format, CTA counts from the number of row groups
    (8-row groups for the widest F16 rows) up to 132, including counts that do not divide the tile count"""
    rg = 8 if wtype == F16 and 16 * (2 * K + 16) > 64 * (1280 + 16) else 16
    i = ALL.index(wtype) + list(SHAPES).index(shape) + d
    out = []
    for j in range(3):
        n_tok = N_TOK[(i + 3 * j) % len(N_TOK)]
        row0 = 16 * ((i + j) % 2) if n_tok <= 48 else 0
        groups = -(-n_tok // rg)
        n_cta = [groups, 132, 37 + groups, 97][(i + j) % 4]
        out.append((n_tok, row0, max(groups, n_cta)))
    return out


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("d", [384, 512, 1280])
@pytest.mark.parametrize("wtype", ALL)
def test_gemv_phase_matches_reference_arithmetic(lib, wtype, d, shape):
    """y = (W x + bias) * scale + res for every output of the view's rows, nothing written elsewhere; QKV also appends its K and V parts
    to the f16 caches at the rows' cells (sentinel-filled: nothing else changes, the Q part is not appended)"""
    N, K = SHAPES[shape][0] * d, SHAPES[shape][1] * d
    if wtype in actq.KQ and K % 256:
        pytest.skip("K-quant rows are whole 256-value super-blocks")
    raw = weights(wtype, N, K)
    X, buf = act_rows(wtype, K, 1)
    rng = np.random.default_rng([wtype, d, N])
    bias = rng.standard_normal(N).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, N).astype(np.float32)
    res = rng.standard_normal((actq.ROWS, N)).astype(np.float32)
    y, _ = oracle(wtype, raw, N, K, buf, range(actq.ROWS))
    want = (y + bias) * scale + res
    tol = 2e-5 * np.abs(y * scale).max()
    n_cells = 200
    for n_tok, row0, n_cta in _views(wtype, d, shape, K):
        rows = range(row0, row0 + n_tok)
        out = f32_out(N)
        kw = dict(w_file=np.frombuffer(raw, np.uint8), N=N, K=K, bias=bias, scale=scale, res=res)
        if shape == "qkv":
            cell = rng.permutation(n_cells)[:actq.ROWS].astype(np.int32)
            kc = np.full((n_cells, d), SENT_F16, np.uint16); vc = kc.copy()
            kw.update(kv_d=d, cell=cell, kc=kc, vc=vc, n_cells=n_cells)
        probe(lib, wtype, GEMV, n_cta, row0, n_tok, out, buf, **kw)
        err = np.abs(out[rows] - want[rows])
        assert err.max() <= tol, (n_tok, row0, n_cta, err.max(), tol, np.unravel_index(err.argmax(), err.shape))
        assert untouched(out, rows)
        if shape == "qkv":
            c = cell[list(rows)]
            assert np.array_equal(kc[c], out[rows, d:2 * d].astype(np.float16).view(np.uint16))
            assert np.array_equal(vc[c], out[rows, 2 * d:].astype(np.float16).view(np.uint16))
            other = np.setdiff1d(np.arange(n_cells), c)
            assert (kc[other] == SENT_F16).all() and (vc[other] == SENT_F16).all()


def test_gemv_phase_f16_fc2_takes_8_row_groups(lib):
    """F16 rows of K = 5120 do not fit 16 to a group: the 8-row group path of mk_rows, all n_tok, CTA counts around the group count"""
    N, K = 1280, 5120
    raw = weights(F16, N, K)
    X, buf = act_rows(F16, K, 2)
    y, _ = oracle(F16, raw, N, K, buf, range(actq.ROWS))
    tol = 2e-5 * np.abs(y).max()
    for i, n_tok in enumerate(N_TOK):
        row0 = 16 * (i % 2) if n_tok <= 48 else 0
        groups = -(-n_tok // 8)
        for n_cta in (groups, groups + 1 + i, 132):
            out = f32_out(N)
            probe(lib, F16, GEMV, n_cta, row0, n_tok, out, buf, w_file=np.frombuffer(raw, np.uint8), N=N, K=K)
            rows = range(row0, row0 + n_tok)
            assert np.abs(out[rows] - y[rows]).max() <= tol, (n_tok, n_cta)
            assert untouched(out, rows)


def _f16_boundary(v, tol):
    """v within tol (>= 0) of a rounding boundary of f16"""
    return np.float16(v - tol).astype(np.float32) != np.float16(v + tol).astype(np.float32)


def check_quantised(wtype, K, out, rows, Y, dv):
    """The device's quantised rows `rows` of `out` against the reference quantiser of the format (Q8_0, Q8_1, Q8_K; f16) applied to Y
    (float32 [len(rows)][K]): the values the device quantised, known to within dv (>= 0, same shape).  Everything -- ints, d, Q8_1 s,
    Q8_K sub-block sums -- must be equal, except where the oracle computes that dv, or the kernel's reciprocal quotients (Q8_0: __fdividef
    and amax * (1 / 127), 2 ulp), reach a rounding boundary: an int may then differ by 1, a scale by its rounding.  The f32 d of Q8_K
    (1 / (-127 / mx)) is exact when dv = 0 and within the bound of amax otherwise.  A Q8_K super-block may have q and d negated only when
    +m and -m tie for its largest magnitude (q8k_pick).  Returns the fractions of ints (f16: values) and of f16 scales that were exempt."""
    fmt = actq.row_format(wtype)
    Y = np.asarray(Y, np.float32); dv = np.asarray(dv, np.float64) * np.ones(Y.shape)
    n_q = n_d = 0
    for i, t in enumerate(rows):
        u, y, e = actq.unpack(wtype, K, out, t), Y[i], dv[i]
        if fmt == "f16":
            ref = y.astype(np.float16).astype(np.float32)
            free = _f16_boundary(y, e) & (np.abs(u["q"] - y) <= e + np.spacing(np.abs(y).astype(np.float16)).astype(np.float64))
            bad = u["q"] != ref
            assert not (bad & ~free).any(), (t, np.flatnonzero(bad & ~free)[:6], u["q"][bad & ~free][:4], y[bad & ~free][:4])
            n_q += _f16_boundary(y, e).sum()
            continue
        bs = 256 if fmt == "q8_k" else 32
        yb, eb = y.reshape(-1, bs).astype(np.float64), e.reshape(-1, bs)
        amax = np.abs(yb).max(axis=1)
        da = np.maximum((np.abs(yb) + eb).max(axis=1) - amax, eb[np.arange(len(yb)), np.abs(yb).argmax(axis=1)])   # amax of the device
        if fmt == "q8_k":
            wq, wd = kq.quantize_q8_k(y)
            pos, neg = yb.max(axis=1), -yb.min(axis=1)
            tie = np.abs(pos - neg) <= 2 * da
            flip = (np.sign(u["d"]) != np.sign(wd)) & (wd != 0)
            assert not (flip & ~tie).any(), (t, np.flatnonzero(flip & ~tie))
            sg = np.where(flip, -1, 1)
            gq, gd = u["q"].reshape(-1, bs) * sg[:, None], u["d"] * sg
            iscale = np.where(amax > 0, 127.0 / np.where(amax > 0, amax, 1), 0)
        else:
            if fmt == "q8_1":
                wq, wd, ws = q1.quantize_q8_1(y)
            else:
                wq, wd = rn.quantize_q8_0(y)
            gq, gd = u["q"].reshape(-1, bs), u["d"]
            iscale = np.where(amax > 0, 127.0 / np.where(amax > 0, amax, 1), 0)
        wq, wd = wq.reshape(-1, bs), wd.reshape(-1)
        r = np.abs(yb) * iscale[:, None]
        dr = iscale[:, None] * eb + r * (da / np.where(amax > 0, amax, 1))[:, None] + r * 2.0 ** -21
        q_free = np.abs(r - np.floor(r) - 0.5) <= dr
        bad = gq != wq
        assert (np.abs(gq - wq) <= 1).all() and not (bad & ~q_free).any(), (t, np.argwhere(bad & ~q_free)[:6])
        if fmt == "q8_k":                                        # f32 d = 1 / (-127 / mx)
            d_free = np.zeros(len(amax), bool)
            assert (np.abs(gd - wd) <= np.abs(wd) * 2 * da / np.where(amax > 0, amax, 1)).all(), (t, gd, wd)
            sums = gq.reshape(-1, 32).sum(axis=1)
            assert np.array_equal(u["sum"] * np.repeat(sg, 8), sums), t             # the record holds the sums of the ints written
            ok = ~q_free.reshape(-1, 32).any(axis=1)
            assert np.array_equal(sums[ok], wq.reshape(-1, 32).sum(axis=1)[ok]), t
        else:
            a127 = amax / 127.0
            d_free = _f16_boundary(a127, da / 127.0 + a127 * 2.0 ** -22)
            assert np.array_equal(gd[~d_free], wd[~d_free]), (t, np.flatnonzero((gd != wd) & ~d_free))
            if fmt == "q8_1":                                    # s = f16(d * sum q) with the unrounded d
                s_free = d_free | q_free.any(axis=1) | _f16_boundary(a127 * wq.sum(axis=1), np.abs(wq.sum(axis=1)) * (da / 127.0 + a127 * 2.0 ** -22))
                assert np.array_equal(u["s"][~s_free], ws[~s_free]), (t, np.flatnonzero((u["s"] != ws) & ~s_free))
        n_q += q_free.sum(); n_d += d_free.sum()
    n = len(rows) * K
    return n_q / n, n_d / max(1, n // (256 if fmt == "q8_k" else 32))


def _gelu_uncertainty(x):
    """how far the device's GELU of the f32 input x may lie from rn.gelu(x).  Both are the f16 rounding of an f32 value g (the reference's
    table); the two g differ by a few f32 ulp (tanhf against the CPU's tanh, FMA contraction): 4e-6 |g|, and below x = -1.6, where 1 + tanh
    cancels, 4 ulp of tanh near -1 (tanhf is within 2 ulp), up to 0.5 |x| 2^-22.  So the results are equal unless that interval around g crosses an f16 rounding
    edge; then they may differ by it plus one f16 step"""
    xh = x.astype(np.float16).astype(np.float32)
    g32 = np.float32(0.5) * xh * (np.float32(1.0) + np.tanh(np.float32(0.79788456080286535587989211986876) * xh * (np.float32(1.0) + np.float32(0.044715) * xh * xh)))
    dg = np.abs(g32).astype(np.float64) * 4e-6 + np.where(xh < np.float32(-1.6), 0.5 * np.abs(xh.astype(np.float64)) * 2.0 ** -22, 0.0)
    step = np.spacing(np.abs(rn.gelu(x)).astype(np.float16)).astype(np.float64)
    return np.where((x > -10) & (x < 10) & _f16_boundary(g32, dg), dg + step, 0.0)


@pytest.mark.parametrize("d", [384, 1280])
@pytest.mark.parametrize("wtype", [F16] + BLOCK32)
def test_fc1_pair_phase_writes_quantised_gelu_rows(lib, wtype, d):
    """FC1 + GELU written straight as FC2 input rows.  The pre-activation y + bias is taken from the GEMV phase on the same rows (a row's
    f32 outputs do not depend on the view or on how tiles are dealt out: test_gemv_row_bits_do_not_depend_on_the_view); the rows must be the
    reference quantisation of gelu of it, ints, d and s, except at the rounding boundaries check_quantised computes"""
    N, K = 4 * d, d
    raw = weights(wtype, N, K)
    X, buf = act_rows(wtype, K, 3)
    bias = np.random.default_rng(d).standard_normal(N).astype(np.float32)
    n_tok, row0, n_cta = (17, 16, 61) if d == 384 else (64, 0, 132)
    rows = list(range(row0, row0 + n_tok))
    w_file = np.frombuffer(raw, np.uint8)
    pre = f32_out(N)
    probe(lib, wtype, GEMV, n_cta, row0, n_tok, pre, buf, w_file=w_file, N=N, K=K, bias=bias)
    y, _ = oracle(wtype, raw, N, K, buf, rows)
    assert np.abs(pre[rows] - (y + bias)).max() <= 2e-5 * np.abs(y).max()
    out = np.full(actq.nbytes(wtype, N), 0xA5, np.uint8)
    probe(lib, wtype, PAIR, n_cta, row0, n_tok, out, buf, w_file=w_file, N=N, K=K, bias=bias)
    unc = _gelu_uncertainty(pre[rows])
    # outside the cancelling range of 1 + tanh only values within 4e-6 of an f16 edge are exempt: about 2 * 4e-6 / 2^-11 = 1.6 %
    assert (unc[pre[rows] >= -1.6] > 0).mean() < 0.02
    fq, fd = check_quantised(wtype, N, out, rows, rn.gelu(pre[rows]), unc)
    # f16 rows keep the small GELU values of the cancelling range at full precision, so those may be one f16 step off; Q8 rows round them away
    assert fq < ((pre[rows] < -1.6).mean() + 0.02 if wtype == F16 else 0.01) and fd < 0.02, (fq, fd)
    assert untouched_bytes(wtype, N, out, rows)


@pytest.mark.parametrize("wtype", [Q3_K, Q4_K, Q5_K])
def test_kquant_fc1_gelu_rows_then_q8k(lib, wtype):
    """K-quant FC1: the GEMV epilogue with GELU writes f32 rows gelu((y + bias) * scale) + res (the pre-activation from the same phase
    without GELU), and mk_q8k_rows turns those 4d-value rows into the reference's Q8_K records, as the pass does"""
    d = 512
    N, K = 4 * d, d
    raw = weights(wtype, N, K)
    X, buf = act_rows(wtype, K, 6)
    rng = np.random.default_rng(wtype)
    bias = rng.standard_normal(N).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, N).astype(np.float32)
    res = rng.standard_normal((actq.ROWS, N)).astype(np.float32)
    n_tok, row0, n_cta = 33, 16, 45
    rows = list(range(row0, row0 + n_tok))
    w_file = np.frombuffer(raw, np.uint8)
    pre = f32_out(N)
    probe(lib, wtype, GEMV, n_cta, row0, n_tok, pre, buf, w_file=w_file, N=N, K=K, bias=bias, scale=scale)
    y, _ = oracle(wtype, raw, N, K, buf, rows)
    assert np.abs(pre[rows] - (y + bias) * scale).max() <= 2e-5 * np.abs(y * scale).max()
    h = f32_out(N)
    probe(lib, wtype, GEMV, n_cta, row0, n_tok, h, buf, w_file=w_file, N=N, K=K, bias=bias, scale=scale, res=res, act=1)
    want = (rn.gelu(pre[rows]) + res[rows]).astype(np.float32)
    e = _gelu_uncertainty(pre[rows])
    bad = h[rows] != want
    assert not (bad & ~(np.abs(h[rows] - want) <= e + np.spacing(np.abs(want)))).any()
    assert not (bad & (e == 0)).any(), np.argwhere(bad & (e == 0))[:6]
    assert untouched(h, rows)
    q = np.full(actq.nbytes(wtype, N), 0xA5, np.uint8)
    probe(lib, wtype, Q8K, n_cta, row0, n_tok, q, h, K=N, lds=N)
    fq, fd = check_quantised(wtype, N, q, rows, h[rows], 0.0)
    assert fq < 1e-3 and fd == 0, (fq, fd)


@pytest.mark.parametrize("wtype", ALL)
def test_gemv_row_bits_do_not_depend_on_the_view(lib, wtype):
    """a row's outputs are the same uint32 alone, inside a 64-row pass, at another position, at another CTA count and at another row0
    (batching and partitioning rely on it); the same for the warp-per-tile logits phase"""
    for N, K in ((3 * 512, 512), (1280, 5120)):
        raw = weights(wtype, N, K)
        X, buf = act_rows(wtype, K, 4)
        one = actq.pack(wtype, K, {p: ref_records(wtype, X[0]) for p in range(actq.ROWS)})   # the same row everywhere
        for phase in (GEMV, LOGITS_WARP):
            got = []
            for n_tok, row0, n_cta, t in ((1, 0, 132, 0), (64, 0, 132, 37), (20, 3, 17, 5), (33, 16, 50, 40), (9, 48, 3, 56)):
                src = _replace_row(wtype, K, buf, one, 37) if t == 37 else one     # the full pass: the row among 63 others
                out = f32_out(N)
                probe(lib, wtype, phase, n_cta, row0, n_tok, out, src, w_file=np.frombuffer(raw, np.uint8), N=N, K=K)
                got.append(out[t].view(np.uint32).copy())
            for g in got[1:]:
                assert np.array_equal(g, got[0]), (N, K, phase)


def _replace_row(wtype, K, buf, src, t):
    out = buf.copy()
    rb = 2 * K if wtype == F16 else K
    out[t * rb:(t + 1) * rb] = src[t * rb:(t + 1) * rb]
    if wtype != F16:
        o = actq.ROWS * K + t * (K // 8)
        out[o:o + K // 8] = src[o:o + K // 8]
    return out


# ---- logits ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,K", [(51866, 1280), (51864, 384)])
@pytest.mark.parametrize("wtype", ALL)
def test_logits_phases(lib, wtype, N, K):
    """both logits phases (warp per tile; split-K GEMV over the whole grid) on a vocabulary that is not a multiple of 16: the last tile's
    rows and a sample of the others against the oracle, nothing written past N or outside the rows"""
    if wtype in actq.KQ and K % 256:
        pytest.skip("K-quant rows are whole 256-value super-blocks")
    raw = weights(wtype, N, K)
    X, buf = act_rows(wtype, K, 5)
    rng = np.random.default_rng([wtype, N])
    check = np.unique(np.concatenate([np.arange(N - 42, N), rng.choice(N, 300, replace=False)]))
    for n_tok in (1, 3, 17):
        rows = list(range(n_tok))
        y, _ = oracle(wtype, _rows_of(wtype, raw, N, K, check), len(check), K, buf, rows)
        tol = 2e-5 * np.abs(y).max()
        for phase in (LOGITS_WARP, GEMV):
            io_out = f32_out(N)                                  # [64][N]: a write past N of row t lands in row t + 1 (outside the rows)
            probe(lib, wtype, phase, 132, 0, n_tok, io_out, buf, w_file=np.frombuffer(raw, np.uint8), N=N, K=K)
            assert np.abs(io_out[rows][:, check] - y).max() <= tol, (n_tok, phase)
            assert np.isfinite(io_out[rows]).all()
            assert untouched(io_out, rows)


# ---- quantisers -------------------------------------------------------------------------------------------------------------------------
def _edge_rows(K, rng):
    """f32 rows with the quantisers' edges: a zero row, a zero super-block, a negative largest value, +m and -m as the largest magnitude of
    one super-block, a large dynamic range, and ordinary rows"""
    X = (rng.standard_normal((actq.ROWS, K)) * rng.uniform(0.1, 5.0, (actq.ROWS, 1))).astype(np.float32)
    X[0] = 0.0
    X[1, :256] = 0.0
    X[2, 7] = -40.0
    X[3, 10] = 30.0; X[3, 200] = -30.0
    X[4] *= (np.float32(10.0) ** rng.integers(-5, 4, K)).astype(np.float32)
    return X


def test_q8k_rows_phase_matches_reference_bytes(lib):
    """mk_q8k_rows writes the reference's quantize_row_q8_K bytes, except that a super-block whose largest magnitude is held by both +m and
    -m may come out with the signs of q and d flipped (q8k_pick: the tie goes to +m): its dot product with any weights is unchanged"""
    rng = np.random.default_rng(9)
    for K, lds, n_tok, row0, n_cta in ((384 * 4, 384 * 4, 64, 0, 132), (1280, 3 * 1280, 17, 16, 5), (512, 512, 9, 0, 1)):
        X = _edge_rows(K, rng)
        src = np.zeros((actq.ROWS, lds), np.float32); src[:, :K] = X
        out = np.full(actq.nbytes(Q4_K, K), 0xA5, np.uint8)
        probe(lib, Q4_K, Q8K, n_cta, row0, n_tok, out, src, K=K, lds=lds)
        want = actq.pack(Q4_K, K, {t: kq.q8_k_bytes(X[t]) for t in range(actq.ROWS)})
        flips = 0
        for t in range(row0, row0 + n_tok):
            g, w = actq.unpack(Q4_K, K, out, t), actq.unpack(Q4_K, K, want, t)
            for sb in range(K // 256):
                s = slice(256 * sb, 256 * sb + 256)
                if np.array_equal(g["q"][s], w["q"][s]) and g["d"][sb] == w["d"][sb]:
                    continue
                xs = X[t, s]
                m = np.abs(xs).max()
                assert (xs == m).any() and (xs == -m).any(), (t, sb)
                assert np.array_equal(g["q"][s], -w["q"][s]) and g["d"][sb] == -w["d"][sb], (t, sb)
                wts = np.random.default_rng(sb).integers(-31, 32, 256)
                assert float(g["d"][sb]) * float(g["q"][s] @ wts) == float(w["d"][sb]) * float(w["q"][s] @ wts)
                flips += 1
            sign = np.where(np.repeat(g["d"], 8) == np.repeat(w["d"], 8), 1, -1)
            assert np.array_equal(g["sum"], sign * w["sum"]), t
        assert flips <= 2


def _layernorm64(x, w, b, eps):
    """LayerNorm in f64, and a bound on how far the kernel's f32 LayerNorm (two-pass mean / variance, then ((x - mean) rstd) w + b) may lie
    from it: 2^-20 of |w| rstd max|x - mean| + |b| + |y|"""
    x = x.astype(np.float64)
    m = x.mean(axis=-1, keepdims=True)
    rstd = 1.0 / np.sqrt(((x - m) ** 2).mean(axis=-1, keepdims=True) + eps)
    y = (x - m) * rstd * w + b
    return y, 2.0 ** -20 * (np.abs(w) * rstd * np.abs(x - m).max(axis=-1, keepdims=True) + np.abs(b) + np.abs(y))


@pytest.mark.parametrize("wtype", [F16, Q8_0, Q4_1, Q4_K])
def test_lnq_phase_matches_layernorm_and_reference_quantiser(lib, wtype):
    """LayerNorm in f64 followed by the reference quantiser of the format's rows (Q8_0, Q8_1, Q8_K, f16): ints, d, Q8_1 s, Q8_K sums, exact
    except at the rounding boundaries check_quantised computes from the f32 LayerNorm's bound; a constant row gives b exactly"""
    rng = np.random.default_rng(wtype)
    for K, n_tok, row0, n_cta in ((512, 64, 0, 132), (1280, 17, 16, 5)):
        X = (rng.standard_normal((actq.ROWS, K)) * 2 + 0.3).astype(np.float32)
        X[5] = np.float32(1.0)
        w = (1 + 0.1 * rng.standard_normal(K)).astype(np.float32); b = (0.1 * rng.standard_normal(K)).astype(np.float32)
        out = np.full(actq.nbytes(wtype, K), 0xA5, np.uint8)
        probe(lib, wtype, LNQ, n_cta, row0, n_tok, out, X, K=K, bias=b, scale=w, eps=np.float32(1e-5))
        Y, dv = _layernorm64(X, w, b, 1e-5)
        rows = list(range(row0, row0 + n_tok))
        fq, fd = check_quantised(wtype, K, out, rows, Y[rows], dv[rows])
        assert fq < (0.1 if wtype == F16 else 0.01) and fd < 0.05, (fq, fd)
        if 5 in rows:
            check_quantised(wtype, K, out, [5], b[None, :], 0.0)
        assert untouched_bytes(wtype, K, out, rows)


def untouched_bytes(wtype, K, out, rows):
    rb = 2 * K if wtype == F16 else K
    return all((out[t * rb:(t + 1) * rb] == 0xA5).all() for t in range(actq.ROWS) if t not in rows)


# ---- attention ----------------------------------------------------------------------------------------------------------------------
# The K-quant instantiation hands its f32 rows on (checked against a float64 softmax at 1e-4); the others quantise the same f32 values
# (the arithmetic before the store does not depend on the format): exact against the reference quantisation of the K-quant rows
QUANT_ROWS = [F16, Q8_0, Q4_1]


def _attn_self(lib, wtype, n_head, row0, n_tok, seed):
    d = 64 * n_head
    rng = np.random.default_rng(seed)
    counts = [1, 31, 32, 33, 255, 256, 257, 448]
    n_cells, ld = 512, 448
    kc = (rng.standard_normal((n_cells, d)) * 0.5).astype(np.float16); vc = rng.standard_normal((n_cells, d)).astype(np.float16)
    qkv = (rng.standard_normal((actq.ROWS, 3 * d))).astype(np.float32)
    nkv = np.zeros(actq.ROWS, np.int32); idx = np.full((actq.ROWS, ld), -7, np.int32)
    for i, t in enumerate(range(row0, row0 + n_tok)):
        nkv[t] = counts[i % len(counts)]
        idx[t, :nkv[t]] = rng.permutation(n_cells)[:nkv[t]]     # scattered cells
    out = f32_out(d) if wtype in actq.KQ else np.full(actq.nbytes(wtype, d), 0xA5, np.uint8)
    probe(lib, wtype, ATTN_SELF, 7, row0, n_tok, out, qkv, d=d, n_head=n_head, kc=kc.view(np.uint16), vc=vc.view(np.uint16), n_cells=n_cells,
          nkv=nkv, idx=idx, ld_idx=ld)
    want = {}
    for t in range(row0, row0 + n_tok):
        c = idx[t, :nkv[t]]
        want[t] = np.concatenate([rn.attention(qkv[t:t + 1, 64 * h:64 * h + 64], kc[c][:, 64 * h:64 * h + 64].astype(np.float32),
                                               vc[c][:, 64 * h:64 * h + 64].astype(np.float32), 1.0)[0] for h in range(n_head)]).astype(np.float64)
    return out, want


@pytest.mark.parametrize("n_head", [6, 20])
def test_attn_self_phase(lib, n_head):
    """key counts 1 .. 448 around the 32-key groups, scattered cells"""
    d = 64 * n_head
    n_tok, row0 = (24, 16) if n_head == 20 else (8, 0)
    rows = list(range(row0, row0 + n_tok))
    f, want = _attn_self(lib, Q4_K, n_head, row0, n_tok, n_head)
    for t in rows:
        assert np.abs(f[t] - want[t]).max() < 1e-4, t
    assert untouched(f, rows)
    for wt in QUANT_ROWS:
        out, _ = _attn_self(lib, wt, n_head, row0, n_tok, n_head)
        fq, fd = check_quantised(wt, d, out, rows, f[rows], 0.0)
        assert fq < 1e-3 and fd < 0.01, (wt, fq, fd)
        assert untouched_bytes(wt, d, out, rows)


def test_attn_cross_phase(lib):
    """1536 keys of which the last 36 are zero and not masked, rows mapped to different slots, (row, head) pairs split unevenly over CTAs"""
    n_head, n_keys, n_slots = 6, 1536, 3
    d = 64 * n_head
    rng = np.random.default_rng(5)
    kx = np.zeros((n_slots, n_head, n_keys, 64), np.float16); vx = np.zeros_like(kx)
    kx[:, :, :1500] = (rng.standard_normal((n_slots, n_head, 1500, 64)) * 0.3).astype(np.float16)
    vx[:, :, :1500] = rng.standard_normal((n_slots, n_head, 1500, 64)).astype(np.float16)
    q = rng.standard_normal((actq.ROWS, d)).astype(np.float32)
    slot = (np.arange(actq.ROWS) * 7 % n_slots).astype(np.int32)
    scale = np.float32(64.0 ** -0.25)
    n_tok, row0, n_cta = 5, 16, 7                                  # 30 pairs over 7 CTAs
    rows = list(range(row0, row0 + n_tok))
    kw = dict(d=d, n_head=n_head, xk=kx.view(np.uint16), xv=vx.view(np.uint16), n_keys=n_keys, n_slots=n_slots, slot=slot, kq_scale=scale)
    f = f32_out(3 * d)
    probe(lib, Q5_K, ATTN_CROSS, n_cta, row0, n_tok, f, q, **kw)
    for t in rows:
        want = np.concatenate([rn.attention(q[t:t + 1, 64 * h:64 * h + 64], kx[slot[t], h, :1500].astype(np.float32),
                                            vx[slot[t], h, :1500].astype(np.float32), float(scale), n_zero_keys=36)[0] for h in range(n_head)])
        assert np.abs(f[t, :d] - want).max() < 1e-4, t
    assert untouched(f, rows)
    for wt in QUANT_ROWS:
        out = np.full(actq.nbytes(wt, d), 0xA5, np.uint8)
        probe(lib, wt, ATTN_CROSS, n_cta, row0, n_tok, out, q, **kw)
        fq, fd = check_quantised(wt, d, out, rows, f[rows, :d], 0.0)
        assert fq < 1e-3 and fd < 0.01, (wt, fq, fd)
        assert untouched_bytes(wt, d, out, rows)
