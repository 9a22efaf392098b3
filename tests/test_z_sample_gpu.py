"""GPU suite (-m gpu): atom_sample_f16 / ops.sample_tokens against the float64 reference of tests/sample_ref64.py -- every row
accepted, greedy bit for bit torch.argmax, rows independent of batch, position and pitch, graph replays equal to eager calls,
and the distribution of 65536 draws against the exact probabilities."""
import numpy as np
import pytest
import torch

from tests import sample_ref64 as R
from tests.test_sample_ref64_cpu import _chi2_p

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _logits(rng, b, v):
    """Row kinds by index: N(0, s) for s in 1, 4, 16; peaked; small integers (many exact ties); +-65504; -inf masks; one NaN
    row and one all -inf row when b >= 7."""
    l = np.empty((b, v), np.float32)
    for i in range(b):
        kind = i % 7
        if kind < 3:
            l[i] = rng.standard_normal(v) * (1.0, 4.0, 16.0)[kind]
        elif kind == 3:
            l[i] = rng.standard_normal(v)
            l[i, rng.integers(0, v, 3)] += 12.0
        elif kind == 4:
            l[i] = rng.integers(-4, 5, v)
        elif kind == 5:
            l[i] = rng.standard_normal(v) * 8
            l[i, rng.integers(0, v, 4)] = 65504
            l[i, rng.integers(0, v, 4)] = -65504
        else:
            l[i] = rng.standard_normal(v) * 2
            l[i, rng.random(v) < 0.5] = -np.inf
    l = l.astype(np.float16)
    if b >= 7:
        l[b // 2, rng.integers(0, v)] = np.nan
        l[b - 1] = -np.inf
    return l


def _params(rng, b, v):
    """Per-row mixes of greedy, temperature only, top-k, top-p and both."""
    T = rng.choice([0.0, 0.3, 0.8, 1.0, 1.5], b).astype(np.float32)
    K = rng.choice([0, 0, 1, 5, 50, max(1, v // 3), v + 1], b).astype(np.int32)
    P = rng.choice([1.0, 1.0, 0.95, 0.9, 0.5, 0.1], b).astype(np.float32)
    keys = np.stack([rng.integers(0, 2 ** 63, b), np.arange(b)], 1).astype(np.int64)
    ctr = rng.integers(0, 2 ** 40, b).astype(np.int64)
    return T, K, P, keys, ctr


def _dev(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in arrays]


def _sample(l, T, K, P, keys, ctr):
    from atom_b200 import ops
    lt = l if isinstance(l, torch.Tensor) else torch.from_numpy(l).to(DEV)
    return ops.sample_tokens(lt, *_dev(T, K, P, keys, ctr)).cpu().numpy()


AMBIGUOUS = []


@pytest.mark.parametrize("v", [128, 1000, 32000, 32001, 128256])
@pytest.mark.parametrize("b", [1, 7, 32, 64])
def test_every_row_is_accepted_by_the_reference(v, b):
    rng = np.random.default_rng(1000 * v + b)
    l = _logits(rng, b, v)
    T, K, P, keys, ctr = _params(rng, b, v)
    tok = _sample(l, T, K, P, keys, ctr)
    amb = R.check_tokens(l, T, K, P, keys, ctr, tok)
    AMBIGUOUS.append((amb, b))
    print(f"V={v} B={b}: {amb} of {b} draws ambiguous; in all so far {sum(a for a, _ in AMBIGUOUS)} of "
          f"{sum(n for _, n in AMBIGUOUS)}")


@pytest.mark.parametrize("v", [128, 32000, 128256])
def test_greedy_and_top1_equal_torch_argmax_with_planted_ties(v):
    rng = np.random.default_rng(v)
    b = 48
    l = (rng.standard_normal((b, v)) * 3).astype(np.float16)
    for i in range(b):                                   # ties at the maximum, spread over the row (and the cluster's slices)
        m = float(l[i].max()) + (i % 3)
        l[i, rng.choice(v, 1 + i % 5, replace=False)] = m
    l[0, :] = 0
    l[0, : v // 2] = -0.0                                # -0 before +0: argmax takes index 0
    lt = torch.from_numpy(l).to(DEV)
    want = torch.argmax(lt, dim=-1).cpu().numpy()
    for T, k in [(0.0, 0), (0.0, 7), (1.3, 1), (0.2, 1)]:
        tok = _sample(lt, np.full(b, T, np.float32), np.full(b, k, np.int32), np.full(b, 0.9, np.float32),
                      np.zeros((b, 2), np.int64), np.arange(b, dtype=np.int64))
        assert np.array_equal(tok, want), (T, k)


def test_rows_do_not_depend_on_batch_position_or_pitch():
    rng = np.random.default_rng(7)
    for v in (1000, 32001, 128256):
        b = 24
        l = _logits(rng, b, v)
        T, K, P, keys, ctr = _params(rng, b, v)
        T[:] = 0.9
        full = _sample(l, T, K, P, keys, ctr)
        perm = rng.permutation(b)
        assert np.array_equal(_sample(l[perm], T[perm], K[perm], P[perm], keys[perm], ctr[perm]), full[perm])
        parts = [_sample(l[i:j], T[i:j], K[i:j], P[i:j], keys[i:j], ctr[i:j]) for i, j in [(0, 1), (1, 8), (8, 24)]]
        assert np.array_equal(np.concatenate(parts), full)
        wide = torch.full((b, v + 37), 7.0, dtype=torch.float16, device=DEV)
        wide[:, :v] = torch.from_numpy(l).to(DEV)
        assert np.array_equal(_sample(wide[:, :v], T, K, P, keys, ctr), full)


def test_captured_call_replayed_with_new_values_equals_the_eager_call():
    from atom_b200 import ops
    rng = np.random.default_rng(3)
    b, v = 16, 32001
    l0 = _logits(rng, b, v)
    stat = _dev(l0, *_params(rng, b, v))
    ops.sample_tokens(*stat)                             # warm-up (kernel attributes) outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ops.sample_tokens(*stat)
    for it in range(3):
        new = [_logits(rng, b, v), *_params(rng, b, v)]
        for s, n in zip(stat, new):
            s.copy_(torch.from_numpy(np.ascontiguousarray(n)))
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), _sample(*new)), it
        R.check_tokens(*new, out.cpu().numpy())


def test_out_of_range_device_parameters_give_minus_one():
    b, v = 5, 300
    l = np.zeros((b, v), np.float16)
    T = np.array([-1.0, np.nan, np.inf, 1.0, 1.0], np.float32)
    P = np.array([1, 1, 1, 0.0, 1.5], np.float32)
    tok = _sample(l, T, np.zeros(b, np.int32), P, np.zeros((b, 2), np.int64), np.zeros(b, np.int64))
    assert tok.tolist() == [-1] * b
    tok = _sample(l[:1], np.ones(1, np.float32), np.full(1, -2, np.int32), np.ones(1, np.float32), np.zeros((1, 2), np.int64),
                  np.zeros(1, np.int64))
    assert tok.tolist() == [-1]


def test_host_parameters_are_validated_and_copied():
    from atom_b200 import ops
    l = torch.zeros(2, 64, dtype=torch.float16, device=DEV)
    for bad in [dict(temperature=[-1.0, 1.0]), dict(temperature=[float("nan"), 1.0]), dict(top_k=[-1, 0]), dict(top_p=[0.0, 1.0]),
                dict(top_p=[1.0, 1.01]), dict(keys=[(0, 0)]), dict(counters=[-1, 0])]:
        args = dict(temperature=[1.0, 1.0], top_k=[0, 0], top_p=[1.0, 1.0], keys=[(0, 0), (0, 1)], counters=[0, 0])
        args.update(bad)
        with pytest.raises(RuntimeError):
            ops.sample_tokens(l, **args)
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.sample_tokens(l, torch.ones(2), [0, 0], [1.0, 1.0], [(0, 0), (0, 1)], [0, 0])
    tok = ops.sample_tokens(l, 1.0, 0, 1.0, [(2 ** 64 - 1, 0), (5, 2 ** 63)], [2 ** 64 - 1, 0])
    assert tok.dtype == torch.int32 and tok.shape == (2,)
    R.check_tokens(l, 1.0, 0, 1.0, [(2 ** 64 - 1, 0), (5, 2 ** 63)], [2 ** 64 - 1, 0], tok)


def test_distribution_of_65536_draws_matches_the_reference_probabilities():
    """One row, V = 1000, T = 0.8, top-k 64, top-p 0.9, counters 0..65535 (fixed seeds: deterministic).  Pearson chi-square
    against the exact probabilities: p >= 1e-4; against T = 0.85 the same draws must fail, which shows the test has power."""
    rng = np.random.default_rng(2024)
    row = (rng.standard_normal(1000) * 3).astype(np.float16)
    n = 65536
    l = torch.from_numpy(row).to(DEV).expand(n, 1000).contiguous()
    tok = _sample(l, np.full(n, 0.8, np.float32), np.full(n, 64, np.int32), np.full(n, 0.9, np.float32),
                  np.tile(np.array([[77, 1]], np.int64), (n, 1)), np.arange(n, dtype=np.int64))
    p_ok = _chi2_p(tok, R.probabilities(row, 0.8, 64, 0.9))
    p_bad = _chi2_p(tok, R.probabilities(row, 0.85, 64, 0.9))
    print(f"chi-square p: {p_ok:.4g} at T = 0.8 (the truth), {p_bad:.3g} at T = 0.85")
    assert p_ok >= 1e-4 and p_bad < 1e-4
