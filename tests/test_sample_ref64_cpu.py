"""CPU suite: the sampler's reference (tests/sample_ref64.py) -- Philox4x64-10 against numpy's independent implementation, the
exact kept sets, the bound, and negative controls: the checker must reject each kind of faulty sampler, naming the row and
the rule it breaks."""
import numpy as np
import pytest

from tests import sample_ref64 as R


def test_philox_matches_numpy_and_the_known_answer_vector():
    assert [hex(w) for w in R.philox4x64_10((0, 0), (0, 0, 0, 0))] == [
        "0x16554d9eca36314c", "0xdb20fe9d672d0fdc", "0xd7e772cee186176b", "0x7e68b68aec7ba23b"]
    rng = np.random.default_rng(3)
    cases = [(0, 0, 0), (1, 2, 3), (2 ** 64 - 1, 2 ** 63, 2 ** 64 - 1)] + \
            [tuple(int(x) for x in rng.integers(0, 2 ** 63, 3, dtype=np.int64)) for _ in range(20)]
    for k0, k1, c in cases:
        # numpy's Philox increments its 256-bit counter before each block: the block at counter c is counter = c - 1's next
        g = np.random.Philox(key=k0 | (k1 << 64), counter=(c - 1) % (1 << 256))
        assert R.philox4x64_10((k0, k1), (c, 0, 0, 0)) == [int(x) for x in g.random_raw(4)]
    assert R.uniform53((5, 7), 9) == R.philox4x64_10((5, 7), (9, 0, 0, 0))[0] >> 11


def _rows(rng, b, v):
    l = (rng.standard_normal((b, v)) * rng.choice([1.0, 4.0, 16.0], (b, 1))).astype(np.float16)
    l[0, :] = rng.integers(-3, 4, v)                 # many exact ties
    return l


@pytest.mark.parametrize("v", [128, 1000, 5000])
def test_numpy_sampler_passes_the_reference(v):
    rng = np.random.default_rng(v)
    b = 24
    l = _rows(rng, b, v)
    l[1, rng.integers(0, v, v // 3)] = -np.inf
    l[2, 5] = np.nan
    l[3, :] = -np.inf
    l[4, :2] = 65504
    l[4, 2:4] = -65504
    T = rng.choice([0.0, 0.5, 1.0, 1.7], b).astype(np.float32)
    K = rng.choice([0, 1, 5, 50, v], b)
    P = rng.choice([1.0, 0.9, 0.5, 0.05], b).astype(np.float32)
    keys = [(11, r) for r in range(b)]
    ctr = rng.integers(0, 1 << 40, b)
    tok = R.sample_np(l, T, K, P, keys, ctr)
    assert tok[2] == -1 and tok[3] == -1
    R.check_tokens(l, T, K, P, keys, ctr, tok)


def test_greedy_and_top1_are_the_first_argmax_with_ties_and_signed_zeros():
    l = np.array([[1, 3, 3, 2], [-0.0, 0.0, -1, -2], [0.0, -0.0, -1, -2]], np.float16)
    for T, k in [(0.0, 0), (0.7, 1)]:
        tok = R.sample_np(l, T, k, 1.0, [(0, 0)] * 3, [0] * 3)
        assert tok.tolist() == [1, 0, 0]
        R.check_tokens(l, T, k, 1.0, [(0, 0)] * 3, [0] * 3, tok)


def test_bound_is_small_positive_and_finite():
    for z, n in [(1.0, 1), (1.0, 128256), (5000.0, 1000)]:
        d = R.bound(z, n)
        assert 0 < d < 1e-4 * z + 1e-6


def _find_rejected(l, T, K, P, fault, rule, counters=range(4000), key=(7, 0), bad_token=None):
    """The first counter at which the faulty sampler's token differs from the correct one (and is `bad_token`, if given) must
    make the checker fail on that row, naming the rule."""
    for c in counters:
        good = R.sample_np(l, T, K, P, [key], [c])
        bad = R.sample_np(l, T, K, P, [key], [c], faults=(fault,))
        if good[0] != bad[0] and bad_token in (None, bad[0]):
            R.check_tokens(l, T, K, P, [key], [c], good)
            with pytest.raises(R.SampleMismatch, match=f"row 0: rule {rule}"):
                R.check_tokens(l, T, K, P, [key], [c], bad)
            return c
    raise AssertionError(f"fault {fault} never changed a token")


def test_checker_rejects_ties_broken_toward_the_higher_index():
    l = np.array([[2, 5, 1, 5, 5, 0, 3, 5]], np.float16)
    with pytest.raises(R.SampleMismatch, match="row 0: rule greedy"):
        R.check_tokens(l, 0.0, 0, 1.0, [(0, 0)], [0], R.sample_np(l, 0.0, 0, 1.0, [(0, 0)], [0], faults=("tie_high",)))
    _find_rejected(l, 1.0, 2, 1.0, "tie_high", "top-k")


def test_checker_rejects_a_top_p_set_one_token_short_or_long():
    # probabilities well apart around the boundary: 0.5, 0.25, 0.125, ... at T = 1 / ln 2
    l = np.array([[-np.float16(i) for i in range(12)]], np.float16)
    T = np.float32(1 / np.log(2))
    # exclusive masses 0, .5, .75, .875: top_p = 0.8 keeps tokens 0..2; the set one token long also draws token 3
    _find_rejected(l, T, 0, 0.8, "topp_long", "top-p", bad_token=3)
    _find_rejected(l, T, 0, 0.8, "topp_short", "draw")


@pytest.mark.parametrize("fault", ["counter+1", "word1"])
def test_checker_rejects_u_from_the_wrong_counter_or_word(fault):
    l = (np.random.default_rng(1).standard_normal((1, 300))).astype(np.float16)
    _find_rejected(l, 1.0, 0, 1.0, fault, "draw")


def test_checker_rejects_the_next_token_at_a_cdf_boundary():
    l = (np.random.default_rng(2).standard_normal((1, 64))).astype(np.float16)
    _find_rejected(l, 0.9, 0, 1.0, "cdf_next", "draw")


def test_checker_rejects_top_k_after_the_temperature():
    # T = 0.7 maps some adjacent FP16 logits onto one FP16 value of l / T: the tie then goes to the lower index, which on the
    # raw logits is the smaller one, and the set changes
    base = np.arange(1400, 1500, dtype=np.float64) * 2.0 ** -10       # adjacent FP16 values in [1.37, 1.46)
    vals = base.astype(np.float16)
    sc = (vals.astype(np.float32) / np.float32(0.7)).astype(np.float16)
    i = next(j for j in range(len(vals) - 1) if sc[j] == sc[j + 1])
    l = np.array([[float(vals[i]) + 0.5, vals[i], vals[i + 1]]], np.float16)      # raw top-2: {0, 2}; after T: {0, 1}
    assert l[0, 2] > l[0, 1]
    _find_rejected(l, np.float32(0.7), 2, 1.0, "topk_after_t", "top-k")


def test_distribution_chi_square_has_power_on_the_cpu_sampler():
    """The GPU test's statistic on the numpy sampler (fewer draws): accepts the right temperature, rejects 0.85."""
    rng = np.random.default_rng(5)
    row = (rng.standard_normal(1000) * 3).astype(np.float16)
    n = 8192
    tok = R.sample_np(np.broadcast_to(row, (n, 1000)), 0.8, 64, 0.9, [(123, 0)] * n, np.arange(n))
    assert _chi2_p(tok, R.probabilities(row, 0.8, 64, 0.9)) > 1e-4
    assert _chi2_p(tok, R.probabilities(row, 0.85, 64, 0.9)) < 1e-4


def _chi2_p(tok, prob):
    import scipy.stats
    n = len(tok)
    obs = np.bincount(tok, minlength=len(prob)).astype(np.float64)
    if obs[prob == 0].sum():
        return 0.0                                   # a draw the distribution cannot produce
    exp = prob * n
    keep = exp >= 5
    o = np.append(obs[keep], obs[~keep & (prob > 0)].sum())
    e = np.append(exp[keep], exp[~keep & (prob > 0)].sum())
    if e[-1] < 5:
        o[-2] += o[-1]; e[-2] += e[-1]
        o, e = o[:-1], e[:-1]
    return scipy.stats.chisquare(o, e).pvalue
