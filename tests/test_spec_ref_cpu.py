"""CPU suite: the references of speculative decoding (tests/spec_ref.py) -- the draft acceptance rule's properties (no candidate is
the plain sampler, greedy accepts exactly the argmax, emitted frequencies follow W / Z by a seeded chi-square, with negative
controls) and the prompt-lookup proposer's edge cases."""
import numpy as np
import pytest
import scipy.stats

from tests import sample_penalty_ref64 as RP
from tests import sample_ref64 as R
from tests import spec_ref as SR


def _rows(b, v, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((b, v)) * 2).astype(np.float16)
    x[:, :2] += np.float16(3)
    return x


@pytest.mark.parametrize("T,k,p,m", [(0.7, 0, 1.0, 0.0), (1.0, 20, 0.9, 0.0), (1.3, 0, 0.8, 0.05), (0.5, 5, 1.0, 0.1)])
def test_no_candidate_is_the_plain_sampler(T, k, p, m):
    x = _rows(40, 300, 1)
    keys = [(5, i) for i in range(40)]
    ctrs = list(range(100, 140))
    want = RP.sample_np(x, T, k, p, keys, ctrs, min_p=m)
    assert np.array_equal(SR.sample_draft_np(x, T, k, p, keys, ctrs, [-1] * 40, min_p=m), want)


def test_greedy_accepts_exactly_the_argmax():
    x = _rows(30, 200, 2)
    am = np.argmax(x.astype(np.float32), axis=1)
    for T, k in ((0.0, 0), (0.9, 1)):
        for d in (am, (am + 1) % 200, np.full(30, -1)):
            tok = SR.sample_draft_np(x, T, k, 1.0, [(1, i) for i in range(30)], list(range(30)), d)
            assert np.array_equal(tok, am)
            assert np.array_equal(tok == d, am == d)


def test_out_of_range_candidates_give_minus_one():
    x = _rows(3, 50, 3)
    tok = SR.sample_draft_np(x, 0.8, 0, 1.0, [(1, 0)] * 3, [0, 1, 2], [-2, 50, 7])
    assert tok.tolist()[:2] == [-1, -1] and tok[2] >= 0


def _frequencies(row, T, k, p, m, d, n=1 << 16, faults=()):
    V = len(row)
    counts = np.zeros(V, np.int64)
    for c in range(n):
        counts[SR.draft_row(row, T, k, p, (77, 3), c, d, m, faults)] += 1
    _, W = SR._kept(row, T, k, p, m)
    return counts, W.astype(np.float64) / float(W.sum())


def _chi2_p(counts, prob):
    kept = prob > 0
    assert counts[~kept].sum() == 0, "a token outside the kept set was emitted"
    n = counts.sum()
    stat = float((((counts[kept] - n * prob[kept]) ** 2) / (n * prob[kept])).sum())
    return scipy.stats.chi2.sf(stat, int(kept.sum()) - 1)


CHI_ROW = np.array([2.0, 1.6, 1.5, 0.9, 0.4, 0.0, -0.3, -1.0, -1.5, -2.5, -4.0, -9.0], dtype=np.float16)


@pytest.mark.parametrize("T,k,p,m,d", [
    (1.0, 0, 1.0, 0.0, 0),           # the top token proposed
    (0.8, 0, 1.0, 0.0, 3),           # a mid token
    (1.2, 6, 0.95, 0.0, 2),          # top-k and top-p, d kept
    (1.0, 6, 1.0, 0.0, 9),           # d cut by top-k: never accepted
    (1.0, 0, 1.0, 0.05, 10),         # d cut by min-p
    (0.9, 0, 0.8, 0.02, 1),          # top-p and min-p together
])
def test_emitted_frequencies_follow_the_kept_weights(T, k, p, m, d):
    counts, prob = _frequencies(CHI_ROW, T, k, p, m, d)
    assert _chi2_p(counts, prob) > 1e-4
    if prob[d] == 0:
        assert counts[d] == 0


@pytest.mark.parametrize("fault", ["keep_d", "accept_word0"])
def test_the_chi_square_rejects_faulty_rules(fault):
    # keep_d: the draw after a rejection may give d again (d is over-weighted); accept_word0: the acceptance and the draw read
    # the same uniform, which skews which tokens follow a rejection
    counts, prob = _frequencies(CHI_ROW, 1.0, 0, 1.0, 0.0, 1, faults=(fault,))
    assert _chi2_p(counts, prob) < 1e-6


def test_acceptance_uses_the_exact_product_and_word_one():
    x = _rows(64, 100, 4)
    keys = [(9, i) for i in range(64)]
    ctrs = list(range(64))
    for i in range(64):
        row = x[i]
        _, W = SR._kept(row, 1.0, 0, 1.0, 0.0)
        d = int(np.argsort(-row.astype(np.float32))[1])
        a = R.uniform53(keys[i], ctrs[i], 1)
        if (a * int(W.sum())) >> 53 < int(W[d]):
            assert SR.draft_row(row, 1.0, 0, 1.0, keys[i], ctrs[i], d) == d


def test_proposer_edge_cases():
    P = SR.propose_np
    assert P([], 4, 1, 3) == [] and P([5], 4, 1, 3) == []
    assert P([1, 2], 4, 2, 3) == []                  # history shorter than n + 1
    assert P([1, 2, 3], 4, 1, 3) == []               # the tail itself is no match
    assert P([7, 1, 2, 7], 4, 1, 1) == [1, 2, 7]     # drafts run to the end of the history
    assert P([7, 1, 7, 2, 7], 4, 1, 1) == [2, 7]     # ties: the latest occurrence
    assert P([7, 1, 7, 2, 7], 1, 1, 1) == [2]        # at most k drafts
    assert P([3, 7, 9, 1, 7, 8, 3, 7], 4, 1, 2) == [9, 1, 7, 8]   # the longest n wins over a later shorter match
    assert P([3, 7, 9, 1, 7, 8, 3, 7], 4, 3, 3) == []
    h = [1, 2, 3, 4, 1, 2, 3]
    assert P(h, 2, 1, 3) == [4, 1] and P(h, 7, 1, 3) == [4, 1, 2, 3]


def test_commit_stops_at_the_first_rejected_or_missing_candidate():
    hist, lens = np.zeros((2, 20), np.int32), np.array([3, 0], np.int32)
    hist[0, :3] = [4, 5, 6]
    out = np.zeros((2, 2 * 3 + 3), np.int32)
    tokens = np.array([4, 5, 9, 1, 8], np.int32)
    cands = np.array([4, 5, 6, -1, -1], np.int32)
    SR.commit_propose_np(tokens, cands, [0, 4, 5], [0, 1], hist, lens, out, 3, 1, 2)
    assert out[0, 0] == 3 and out[0, 2:6].tolist() == [4, 5, 9, -1]
    assert hist[0, :6].tolist() == [4, 5, 6, 4, 5, 9] and lens.tolist() == [6, 1]
    assert out[1, 0] == 1 and out[1, 2] == 8 and out[1, 1] == 0
    full = np.zeros((1, 4), np.int32)
    ln = np.array([3], np.int32)
    o = np.zeros((1, 9), np.int32)
    SR.commit_propose_np(np.array([1, 2], np.int32), np.array([1, -1], np.int32), [0, 2], [0], full, ln, o, 3, 1, 1)
    assert ln[0] == 4 and o[0, 0] == 2                 # emitted, but the slot holds no more than cap
