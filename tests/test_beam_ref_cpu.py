"""CPU suite: the beam-search reference (tests/beam_ref.py) -- one step's candidate order, stop ids of rank >= W, the length
penalty, the finished set, and the whole search against an exhaustive one on Markov stand-ins."""
import numpy as np
import pytest

from tests import beam_ref as BR


def _markov(V, seed):
    rng = np.random.default_rng(seed)
    table = (rng.standard_normal((V + 1, V)) * 2).astype(np.float16)
    return (lambda t: table[t]), table[V]


def test_step_order_and_ties():
    row = np.array([1.0, 3.0, 3.0, 2.0, -np.inf], np.float16)
    live, key, fin, fkey = BR.beam_select_np(row[None], [0, 1], [0.0], 3)
    assert live[0, :, 1].tolist() == [1, 2, 3]          # equal logits: the lower id first; -inf is never a candidate
    assert key[0, 0] == key[0, 1] > key[0, 2]
    assert (fin == -1).all()
    # two rows: equal keys go to the lower beam index (both of beam 0's tied tokens before beam 1's)
    live, key, _, _ = BR.beam_select_np(np.stack([row, row]), [0, 2], [-1.0, -1.0], 3)
    assert live[0].tolist() == [[0, 1], [0, 2], [1, 1]]


def test_stop_rank_and_skip():
    row = np.array([5.0, 4.0, 3.0, 2.0, 1.0], np.float16)
    live, _, fin, _ = BR.beam_select_np(row[None], [0, 1], [0.0], 2, stop_ids=(1, 4))
    assert fin[0, :, 1].tolist() == [1, -1]             # id 1 has rank 1 < W; id 4 has rank 4 >= W: skipped
    assert live[0, :, 1].tolist() == [0, 2]


def test_invalid_rows_and_empty_requests():
    rows = np.array([[1, np.nan, 0], [-np.inf] * 3, [0, 1, np.inf]], np.float16)
    live, _, fin, _ = BR.beam_select_np(rows, [0, 0, 3], [0, 0, 0], 3)
    assert (live == -1).all() and (fin == -1).all()
    req = BR.BeamRequest(2, 0.0, 5)
    req.step(live[1], np.full(2, -1, np.float32), fin[1], np.full(2, -1, np.float32), lambda r: r)
    assert req.done and req.best()[0] == []


def test_length_penalty_and_finished_set():
    req = BR.BeamRequest(2, 1.0, 10, stop_ids=(0,))
    req.offer([1, 0], np.float32(-3.0))                 # score -1.5
    req.offer([1, 2, 3, 0], np.float32(-4.0))           # score -1.0: better despite the lower sum
    assert req.best()[0] == [1, 2, 3, 0]
    req.offer([5, 0], np.float32(-3.0))                 # -1.5 is not strictly better than the worst (-1.5): kept out
    assert sorted(h[2] for h in req.finished) == [[1, 0], [1, 2, 3, 0]]
    req.offer([6, 0], np.float32(-2.0))                 # -1.0 ties the best: replaces the worst; the earlier one wins ties
    assert req.best()[0] == [1, 2, 3, 0]
    req0 = BR.BeamRequest(2, 0.0, 10)
    req0.offer([1, 0], np.float32(-3.0))
    req0.offer([1, 2, 3, 0], np.float32(-4.0))
    assert req0.best()[0] == [1, 0]


@pytest.mark.parametrize("V,L,stops,alpha", [(8, 2, (), 0.0), (2, 4, (), 0.0), (8, 2, (3,), 1.0), (2, 4, (1,), 0.7)])
def test_wide_beam_is_exhaustive(V, L, stops, alpha):
    for seed in range(4):
        nxt, first = _markov(V, seed)
        req = BR.beam_search_ref(nxt, first, 8, alpha, L, stops)
        tokens, _, score = req.best()
        best_score, best_tokens = BR.exhaustive_best(nxt, first, alpha, L, stops)
        assert score == pytest.approx(best_score, abs=1e-6) and tokens == best_tokens, (seed, tokens, best_tokens)


def test_width_one_is_greedy():
    nxt, first = _markov(50, 7)
    for stops in ((), (int(np.argmax(nxt(3))),)):
        req = BR.beam_search_ref(nxt, first, 1, 0.0, 12, stops)
        greedy, row = [], first
        for _ in range(12):
            t = int(np.argmax(row.astype(np.float32)))
            greedy.append(t)
            if t in stops:
                break
            row = nxt(t)
        assert req.best()[0] == greedy
