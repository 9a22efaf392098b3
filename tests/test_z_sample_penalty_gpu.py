"""GPU suite (-m gpu): atom_sample_ex_f16 / ops.sample_tokens with penalties, min-p and log-probabilities, against the float64
reference of tests/sample_penalty_ref64.py -- every row, log-probability and top-n list accepted; greedy bit for bit the argmax of the
host-computed penalised logits; neutral options equal to the plain call; rows independent of batch, position and pitch; the
table incremented once per drawn token; graph replays equal to eager calls; and 65536 draws against the exact probabilities."""
import numpy as np
import pytest
import torch

from tests import sample_penalty_ref64 as R
from tests.test_sample_ref64_cpu import _chi2_p
from tests.test_z_sample_gpu import _dev, _logits, _params

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _table(rng, slots, v, saturate=False):
    """Random penalty state: ~10 % prompt tokens, ~5 % generated 1-8 times; rows of `saturate` at the 0x7FFF count."""
    t = np.zeros((slots, (v + 7) // 8 * 8), np.uint16)
    t[:, :v][rng.random((slots, v)) < 0.1] = 0x8000
    gen = rng.random((slots, v)) < 0.05
    t[:, :v] |= (gen * rng.integers(1, 9, (slots, v))).astype(np.uint16)
    if saturate:
        t[::3, :v] |= 0x7FFF
    return t


def _options(rng, b, slots):
    sl = rng.permutation(slots)[:b].astype(np.int32)
    sl[rng.random(b) < 0.15] = -1
    return dict(min_p=rng.choice([0.0, 0.0, 0.02, 0.1, 0.5], b).astype(np.float32),
                repetition_penalty=rng.choice([1.0, 0.7, 1.3, 2.0], b).astype(np.float32),
                frequency_penalty=rng.choice([0.0, 0.3, -0.4, 1.5], b).astype(np.float32),
                presence_penalty=rng.choice([0.0, 0.5, -0.8, -2.0], b).astype(np.float32), slots=sl)


def _call(l, T, K, P, keys, ctr, table, opts, n=None):
    """ops.sample_tokens with device tensors; returns numpy outputs and the table after the call."""
    from atom_b200 import ops
    lt = l if isinstance(l, torch.Tensor) else torch.from_numpy(l).to(DEV)
    tab = torch.from_numpy(table.view(np.int16).copy()).to(DEV)
    kw = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in opts.items()}
    out = ops.sample_tokens(lt, *_dev(T, K, P, keys, ctr), penalty_table=tab, logprobs=n, **kw)
    out = tuple(x.cpu().numpy() for x in out) if isinstance(out, tuple) else out.cpu().numpy()
    return out, tab.cpu().numpy().view(np.uint16)


def _recorded(before, slots, tok):
    want = before.copy()
    for s, t in zip(slots, tok):
        if s >= 0 and t >= 0 and (want[s, t] & 0x7FFF) != 0x7FFF:
            want[s, t] += 1
    return want


AMBIGUOUS = []


@pytest.mark.parametrize("v", [128, 1000, 32000, 32001, 128256])
@pytest.mark.parametrize("b", [1, 7, 32, 64])
def test_every_row_logprob_and_top_n_is_accepted_by_the_reference(v, b):
    rng = np.random.default_rng(5000 * v + b)
    l = _logits(rng, b, v)
    T, K, P, keys, ctr = _params(rng, b, v)
    table = _table(rng, b + 3, v, saturate=True)
    opts = _options(rng, b, b + 3)
    n = int(rng.choice([0, 1, 5, 20]))
    (tok, lp, ids, lps), after = _call(l, T, K, P, keys, ctr, table, opts, n)
    amb = R.check_tokens(l, T, K, P, keys, ctr, tok, penalty_table=table, logprob=lp, top_ids=ids, top_logprobs=lps, **opts)
    assert np.array_equal(after, _recorded(table, opts["slots"], tok))
    AMBIGUOUS.append((amb, b))
    print(f"V={v} B={b} n={n}: {amb} of {b} draws ambiguous; so far {sum(a for a, _ in AMBIGUOUS)} of {sum(m for _, m in AMBIGUOUS)}")


@pytest.mark.parametrize("v", [128, 32000, 128256])
def test_greedy_with_penalties_is_the_argmax_of_the_penalised_logits(v):
    rng = np.random.default_rng(v + 1)
    b = 40
    l = (rng.standard_normal((b, v)) * 3).astype(np.float16)
    l[:, rng.choice(v, 5, replace=False)] = l.max()                 # ties at the raw maximum, broken by the penalties
    table = _table(rng, b, v)
    opts = _options(rng, b, b)
    opts["min_p"][:] = 0.3
    T = np.where(np.arange(b) % 2, 0.0, 0.7).astype(np.float32)
    K = np.where(np.arange(b) % 2, 0, 1).astype(np.int32)
    (tok, lp, ids, lps), _ = _call(l, T, K, np.ones(b, np.float32), np.zeros((b, 2), np.int64), np.arange(b, dtype=np.int64), table,
                                   opts, 3)
    lp16 = R._penalised(l, table, opts["slots"], opts["repetition_penalty"], opts["frequency_penalty"], opts["presence_penalty"])
    want = torch.argmax(torch.from_numpy(lp16).to(DEV), dim=-1).cpu().numpy()
    assert np.array_equal(tok, want)
    assert np.array_equal(ids[:, 0], want)


def test_neutral_options_and_a_zero_table_equal_the_plain_call():
    from atom_b200 import ops
    rng = np.random.default_rng(8)
    for v in (1000, 32001, 128256):
        b = 21
        l = _logits(rng, b, v)
        prm = _params(rng, b, v)
        plain = ops.sample_tokens(torch.from_numpy(l).to(DEV), *_dev(*prm)).cpu().numpy()
        zero = np.zeros((b, (v + 7) // 8 * 8), np.uint16)
        opts = dict(min_p=np.zeros(b, np.float32), repetition_penalty=np.ones(b, np.float32),
                    frequency_penalty=np.zeros(b, np.float32), presence_penalty=np.zeros(b, np.float32),
                    slots=np.arange(b, dtype=np.int32))
        (tok, lp, ids, lps), _ = _call(l, *prm, zero, opts, 20)
        assert np.array_equal(tok, plain)
        tok2, _ = _call(l, *prm, zero, {**opts, "slots": np.full(b, -1, np.int32)})
        assert np.array_equal(tok2, plain)
        tok3 = ops.sample_tokens(torch.from_numpy(l).to(DEV), *_dev(*prm), min_p=0.0, logprobs=0)[0].cpu().numpy()
        assert np.array_equal(tok3, plain)


def test_rows_do_not_depend_on_batch_position_pitch_or_table_pitch():
    rng = np.random.default_rng(17)
    for v in (1000, 32001, 128256):
        b = 24
        l = _logits(rng, b, v)
        T, K, P, keys, ctr = _params(rng, b, v)
        T[:] = 0.9
        table = _table(rng, b, v)
        opts = _options(rng, b, b)
        (full, lp, ids, lps), after = _call(l, T, K, P, keys, ctr, table, opts, 4)
        perm = rng.permutation(b)
        po = {k: x[perm] for k, x in opts.items()}
        (pt, plp, pids, plps), pafter = _call(l[perm], T[perm], K[perm], P[perm], keys[perm], ctr[perm], table, po, 4)
        assert np.array_equal(pt, full[perm]) and np.array_equal(plp, lp[perm], equal_nan=True)
        assert np.array_equal(pids, ids[perm]) and np.array_equal(pafter, after)
        for i, j in [(0, 1), (1, 9), (9, 24)]:
            (pt, plp, _, _), _ = _call(l[i:j], T[i:j], K[i:j], P[i:j], keys[i:j], ctr[i:j], table,
                                       {k: x[i:j] for k, x in opts.items()}, 4)
            assert np.array_equal(pt, full[i:j]) and np.array_equal(plp, lp[i:j], equal_nan=True)
        wide_l = np.full((b, v + 37), 7.0, np.float16)
        wide_l[:, :v] = l
        wide_t = np.full((b, table.shape[1] + 64), 0x7FFF, np.uint16)
        wide_t[:, :table.shape[1]] = table
        (wt, wlp, wids, _), wafter = _call(torch.from_numpy(wide_l).to(DEV)[:, :v], T, K, P, keys, ctr, wide_t, opts, 4)
        assert np.array_equal(wt, full) and np.array_equal(wlp, lp, equal_nan=True) and np.array_equal(wids, ids)
        assert np.array_equal(wafter[:, :table.shape[1]], after)


def test_captured_call_replayed_with_new_values_equals_the_eager_call():
    from atom_b200 import ops
    rng = np.random.default_rng(4)
    b, v, n = 16, 32001, 6
    stat = _dev(_logits(rng, b, v), *_params(rng, b, v))
    o0 = _options(rng, b, b + 2)
    okeys = list(o0)
    sopts = {k: torch.from_numpy(o0[k]).to(DEV) for k in okeys}
    tab = torch.from_numpy(_table(rng, b + 2, v).view(np.int16)).to(DEV)
    ops.sample_tokens(*stat, penalty_table=tab, logprobs=n, **sopts)             # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ops.sample_tokens(*stat, penalty_table=tab, logprobs=n, **sopts)
    for it in range(3):
        new = [_logits(rng, b, v), *_params(rng, b, v)]
        o = _options(rng, b, b + 2)
        table = _table(rng, b + 2, v, saturate=it == 1)
        for s, x in zip(stat, new):
            s.copy_(torch.from_numpy(np.ascontiguousarray(x)))
        for k in okeys:
            sopts[k].copy_(torch.from_numpy(o[k]))
        tab.copy_(torch.from_numpy(table.view(np.int16)))
        g.replay()
        torch.cuda.synchronize()
        got = [x.cpu().numpy() for x in out]
        after = tab.cpu().numpy().view(np.uint16)
        want, wafter = _call(new[0], *new[1:], table, o, n)
        for x, y in zip(got, want):
            assert np.array_equal(x, y, equal_nan=True), it
        assert np.array_equal(after, wafter)
        R.check_tokens(*new, got[0], penalty_table=table, logprob=got[1], top_ids=got[2], top_logprobs=got[3], **o)


def test_slot_init_and_host_validation():
    from atom_b200 import ops
    tab = ops.penalty_table(4, 1001, DEV)
    assert tab.shape == (4, 1008) and tab.dtype == torch.int16
    tab.fill_(0x1234)
    ops.init_penalty_slot(tab, 2, [5, 7, 5, 1000])
    ops.init_penalty_slot(tab, 1, torch.tensor([0, 3, 5000, -4], dtype=torch.int32, device=DEV))
    t = tab.cpu().numpy().view(np.uint16)
    want = np.zeros(1008, np.uint16)
    want[[5, 7, 1000]] = 0x8000
    assert np.array_equal(t[2], want) and (t[[0, 3]] == 0x1234).all()
    want = np.zeros(1008, np.uint16)
    want[[0, 3]] = 0x8000
    assert np.array_equal(t[1], want)
    l = torch.zeros(2, 1001, dtype=torch.float16, device=DEV)
    base = dict(temperature=[1.0, 1.0], top_k=[0, 0], top_p=[1.0, 1.0], keys=[(0, 0), (0, 1)], counters=[0, 0])
    for bad in [dict(slots=[1, 1]), dict(slots=[0, 4]), dict(slots=[0]), dict(repetition_penalty=[0.0, 1.0]),
                dict(frequency_penalty=[np.nan, 0.0]), dict(presence_penalty=[np.inf, 0.0]), dict(min_p=[1.5, 0.0]),
                dict(logprobs=21), dict(penalty_table=None, repetition_penalty=1.2)]:
        kw = dict(penalty_table=tab, slots=[0, 1])
        kw.update(bad)
        if kw.get("penalty_table") is None:
            kw.pop("slots")
        with pytest.raises(RuntimeError):
            ops.sample_tokens(l, **base, **kw)
    with pytest.raises(RuntimeError):
        ops.init_penalty_slot(tab, 0, [1008])
    dev_bad = torch.tensor([-1.0, 1.0], device=DEV)
    tok = ops.sample_tokens(l, **base, penalty_table=tab, slots=[0, -1], repetition_penalty=dev_bad)
    assert tok.cpu().tolist()[0] == -1 and tok.cpu().tolist()[1] >= 0


def test_distribution_with_min_p_and_penalties_matches_the_exact_probabilities():
    """One row, V = 1000, T = 0.8, top-k 200, min-p 0.02, top-p 0.95, all penalties, counters 0..65535 (no slot recording: each
    draw sees the same state).  Pearson chi-square against the exact probabilities of l': p >= 1e-4; against min-p 0.05 the
    same draws must fail."""
    from atom_b200 import ops
    rng = np.random.default_rng(77)
    row = (rng.standard_normal(1000) * 3).astype(np.float16)
    ent = _table(rng, 1, 1000)[0, :1000]
    r, f, q = 1.4, 0.3, -0.5
    lp16 = R.penalise(row, ent, r, f, q)
    n = 65536
    l = torch.from_numpy(lp16).to(DEV).expand(n, 1000).contiguous()
    tok = ops.sample_tokens(l, *_dev(np.full(n, 0.8, np.float32), np.full(n, 200, np.int32), np.full(n, 0.95, np.float32),
                                     np.tile(np.array([[91, 2]], np.int64), (n, 1)), np.arange(n, dtype=np.int64)),
                            min_p=0.02).cpu().numpy()
    # the same draws through the penalty path: one row per draw with its own slot holding the same state
    tab = torch.from_numpy(np.tile(np.pad(ent, (0, 0)), (n, 1)).view(np.int16)).to(DEV)
    raw = torch.from_numpy(row).to(DEV).expand(n, 1000).contiguous()
    tok_pen = ops.sample_tokens(raw, *_dev(np.full(n, 0.8, np.float32), np.full(n, 200, np.int32), np.full(n, 0.95, np.float32),
                                           np.tile(np.array([[91, 2]], np.int64), (n, 1)), np.arange(n, dtype=np.int64)),
                                min_p=0.02, repetition_penalty=r, frequency_penalty=f, presence_penalty=q, penalty_table=tab,
                                slots=torch.arange(n, dtype=torch.int32, device=DEV)).cpu().numpy()
    assert np.array_equal(tok, tok_pen)

    def probs(m):
        v = lp16.astype(np.float64)
        order = R.total_order(v)
        w = np.exp((v[order[:200]] - v[order[0]]) / 0.8)
        keep = w >= m
        w = w[keep]
        o = order[:200][keep]
        M = np.concatenate([[0.0], np.cumsum(w)[:-1]])
        k = max(1, int(np.count_nonzero(M < 0.95 * w.sum())))
        out = np.zeros(1000)
        out[o[:k]] = w[:k] / w[:k].sum()
        return out
    p_ok, p_bad = _chi2_p(tok, probs(0.02)), _chi2_p(tok, probs(0.05))
    print(f"chi-square p: {p_ok:.4g} at min-p 0.02 (the truth), {p_bad:.3g} at min-p 0.05")
    assert p_ok >= 1e-4 and p_bad < 1e-4
