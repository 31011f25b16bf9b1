"""The decode kernel's attention phases as streams (wb_decode_mk.cu: mk_attn_self, mk_attn_cross), through the phase probe
(wb200_dbg_mk_phase):

* the cross stream does not read the padding keys n_audio_ctx .. n_keys - 1 (NaN there changes no bit of what zeros give);
* a self-attention item's bits depend on the item alone, not on which warp pair, CTA or view streams it: a warp pair streams one item
  after another, and with one CTA it walks more than 100 of them.
"""
import numpy as np
import pytest

import actq
from oracle import ref_numpy as rn
from test_decode_phases_gpu import ATTN_CROSS, ATTN_SELF, Q5_0, Q5_K, f32_out, probe

pytestmark = pytest.mark.gpu
F16_NAN = np.uint16(0x7E00)
N_AUDIO_CTX, N_KEYS = 1500, 1536
SELF_COUNTS = [1, 2, 3, 255, 256, 257, 448, 116, 17, 8, 9, 24, 40, 228, 4, 100]


def _out(wtype, d, ncol):
    return f32_out(ncol) if wtype in actq.KQ else np.full(actq.nbytes(wtype, d), 0xA5, np.uint8)


def cross_case(n_head, pad_value, seed=5):
    """head-major cross K / V of 3 slots with N_AUDIO_CTX real keys of N_KEYS; the padding keys hold `pad_value` (f16 bits)"""
    d, n_slots = 64 * n_head, 3
    rng = np.random.default_rng(seed)
    kx = np.full((n_slots, n_head, N_KEYS, 64), pad_value, np.uint16).view(np.float16); vx = kx.copy()
    kx[:, :, :N_AUDIO_CTX] = (rng.standard_normal((n_slots, n_head, N_AUDIO_CTX, 64)) * 0.3).astype(np.float16)
    vx[:, :, :N_AUDIO_CTX] = rng.standard_normal((n_slots, n_head, N_AUDIO_CTX, 64)).astype(np.float16)
    q = rng.standard_normal((actq.ROWS, d)).astype(np.float32)
    slot = (np.arange(actq.ROWS) * 7 % n_slots).astype(np.int32)
    return q, dict(d=d, n_head=n_head, xk=kx.view(np.uint16), xv=vx.view(np.uint16), n_keys=N_KEYS, n_slots=n_slots, slot=slot,
                   kq_scale=np.float32(64.0 ** -0.25))


def run_cross(lib, wtype, n_cta, row0, n_tok, q, kw, n_audio_ctx):
    d = kw["d"]
    out = _out(wtype, d, 3 * d)
    probe(lib, wtype, ATTN_CROSS, n_cta, row0, n_tok, out, q, N=n_audio_ctx, **kw)
    return out


def self_case(n_head, n_rows, seed=11, ld=448):
    """n_rows logical rows: query, key count (SELF_COUNTS in turn) and scattered cells of their own; every cell no row attends to is NaN"""
    d = 64 * n_head
    rng = np.random.default_rng(seed)
    counts = np.array([SELF_COUNTS[j % len(SELF_COUNTS)] for j in range(n_rows)], np.int32)
    n_cells = 2 * int(counts.sum())
    perm = rng.permutation(n_cells)
    kc = np.full((n_cells, d), F16_NAN, np.uint16).view(np.float16); vc = kc.copy()
    idx = np.full((n_rows, ld), -7, np.int32)
    o = 0
    for j, n in enumerate(counts):
        cells = perm[o:o + n]; o += n
        idx[j, :n] = cells
        kc[cells] = (rng.standard_normal((n, d)) * 0.5).astype(np.float16)
        vc[cells] = rng.standard_normal((n, d)).astype(np.float16)
    qkv = rng.standard_normal((n_rows, 3 * d)).astype(np.float32)
    return dict(d=d, n_head=n_head, kc=kc, vc=vc, qkv=qkv, counts=counts, idx=idx, ld=ld)


def run_self(lib, wtype, case, n_cta, row0):
    """the logical rows at rows row0 .. row0 + n_rows - 1 of the pass; returns the output rows in logical order (uint8 / f32)"""
    d, n_rows, ld = case["d"], len(case["counts"]), case["ld"]
    qkv = np.zeros((actq.ROWS, 3 * d), np.float32); qkv[row0:row0 + n_rows] = case["qkv"]
    nkv = np.zeros(actq.ROWS, np.int32); nkv[row0:row0 + n_rows] = case["counts"]
    idx = np.full((actq.ROWS, ld), -7, np.int32); idx[row0:row0 + n_rows] = case["idx"]
    out = _out(wtype, d, d)
    probe(lib, wtype, ATTN_SELF, n_cta, row0, n_rows, out, qkv, d=d, n_head=case["n_head"], kc=case["kc"].view(np.uint16),
          vc=case["vc"].view(np.uint16), n_cells=case["kc"].shape[0], nkv=nkv, idx=idx, ld_idx=ld)
    if wtype in actq.KQ:
        return out[row0:row0 + n_rows]
    if wtype == actq.F16:                                        # halves
        return out.reshape(actq.ROWS, 2 * d)[row0:row0 + n_rows]
    q, s = out[:actq.ROWS * d].reshape(actq.ROWS, d), out[actq.ROWS * d:].reshape(actq.ROWS, d // 8)    # int8 values, 4 scale bytes per block
    return np.concatenate([q, s], axis=1)[row0:row0 + n_rows]


@pytest.mark.parametrize("wtype", [Q5_K, Q5_0])
def test_cross_stream_does_not_read_padding_keys(lib, wtype):
    """NaN in keys 1500 .. 1535 of every head gives the bits that zeros there give when every key is read (fails if padding is read)"""
    n_head, n_tok, row0, n_cta = 20, 5, 16, 7                    # 100 (row, head) pairs over 7 CTAs
    q, kw_zero = cross_case(n_head, 0)
    _, kw_nan = cross_case(n_head, F16_NAN)
    want = run_cross(lib, wtype, n_cta, row0, n_tok, q, kw_zero, 0)            # N = 0: every key is read, the padding is zero
    got = run_cross(lib, wtype, n_cta, row0, n_tok, q, kw_nan, N_AUDIO_CTX)
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    if wtype in actq.KQ:
        assert np.isfinite(got[row0:row0 + n_tok, :64 * n_head]).all()


SELF_VIEWS = [(1, 0), (3, 16), (7, 5), (33, 11), (132, 2)]      # (CTAs, first row); one CTA: 8 warp pairs stream 120 items each


@pytest.mark.parametrize("wtype", [Q5_K, Q5_0])
def test_self_stream_bits_do_not_depend_on_the_schedule(lib, wtype):
    """48 rows x 20 heads with key counts 1 .. 448 (1, 2, 3: fewer keys than the ring has stages), cells scattered over a cache whose
    unattended cells are NaN: equal bits for every (CTA count, first row), finite, and the float64 softmax at 1e-4 (f32 rows)"""
    case = self_case(20, 48)
    outs = [run_self(lib, wtype, case, n_cta, row0) for n_cta, row0 in SELF_VIEWS]
    for (n_cta, row0), o in zip(SELF_VIEWS[1:], outs[1:]):
        assert np.array_equal(o.view(np.uint8), outs[0].view(np.uint8)), (n_cta, row0)
    if wtype in actq.KQ:
        f = outs[0]
        assert np.isfinite(f).all()
        kc, vc, d = case["kc"], case["vc"], case["d"]
        for j, n in enumerate(case["counts"]):
            c = case["idx"][j, :n]
            want = np.concatenate([rn.attention(case["qkv"][j:j + 1, 64 * h:64 * h + 64], kc[c][:, 64 * h:64 * h + 64].astype(np.float32),
                                                vc[c][:, 64 * h:64 * h + 64].astype(np.float32), 1.0)[0] for h in range(case["n_head"])])
            assert np.abs(f[j] - want).max() < 1e-4, j
