"""CPU: the NumPy statement of the reference's Q4_1 / Q5_1 arithmetic (tests/q1_ref.py) and synth's Q4_1 / Q5_1 quantisers against the
compiled reference: Q8_1 activation bytes, per-row dots and weight blocks byte for byte."""
import numpy as np
import pytest

import q1_ref as q1
from wbtest import load_ref, ref_quantize
from e2e_util import synth


@pytest.fixture(scope="module")
def cpu():
    return q1.RefCpu(load_ref())


def _rows():
    rng = np.random.default_rng(3)
    zero = np.zeros(32, np.float32)
    tie = rng.uniform(-1, 1, 32).astype(np.float32); tie[3] = 2.0; tie[17] = -2.0                   # +amax and -amax in one block
    wide = (rng.standard_normal(32) * np.float32(10.0) ** rng.integers(-6, 4, 32)).astype(np.float32)  # large dynamic range
    half = ((np.arange(32) - 16).astype(np.float32) + np.float32(0.5)) * np.float32(127.0 / 15.5)    # x * 127 / amax on .5 boundaries
    half[0] = np.float32(127.0)
    normal = (rng.standard_normal(32 * 40) * 0.3).astype(np.float32)
    return np.concatenate([zero, tie, wide, half, normal])


@pytest.mark.parametrize("wt", [q1.Q4_1, q1.Q5_1])
def test_q8_1_rows_match_reference_bytes(cpu, wt):
    x = _rows()
    assert q1.q8_1_bytes(x) == cpu.quantize_act(wt, x)


@pytest.mark.parametrize("wt", [q1.Q4_1, q1.Q5_1])
@pytest.mark.parametrize("K", [384, 768, 1280, 5120])
def test_mul_mat_matches_reference_vec_dot(cpu, wt, K):
    rng = np.random.default_rng(K + wt)
    N, n_tok = 24, 3
    w = (rng.standard_normal((N, K)) * 0.02).astype(np.float32)
    raw = ref_quantize(cpu.ref, wt, w)
    x = (rng.standard_normal((n_tok, K))).astype(np.float32)
    mine = q1.mul_mat_q(wt, raw, N, K, x)
    rb = len(raw) // N
    theirs = np.array([[cpu.vec_dot(wt, K, raw[n * rb:(n + 1) * rb], cpu.quantize_act(wt, x[t])) for n in range(N)] for t in range(n_tok)], np.float32)
    assert np.abs(mine - theirs).max() <= 1e-6 * np.abs(theirs).max()


@pytest.mark.parametrize("wt", [synth.Q4_1, synth.Q5_1])
def test_numpy_quantisers_match_reference(cpu, wt):
    rng = np.random.default_rng(11)
    w = (rng.standard_normal((64, 768)) * 0.02).astype(np.float32)
    w[0, :32] = 0.0                                              # d = 0
    w[1, :32] = np.float32(0.25)                                 # max == min
    w[2, :32] = np.linspace(-1, 1, 32, dtype=np.float32)
    assert synth.quantize(wt, w) == ref_quantize(cpu.ref, wt, w)
