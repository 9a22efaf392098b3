"""CPU suite: the penalty, min-p and log-probability reference tests/sample_penalty_ref64.py -- the penalised logits bit for bit
against a float64 restatement, the numpy sampler accepted by the extended checker, and every deliberate fault rejected."""
import numpy as np
import pytest

from tests import sample_penalty_ref64 as R


def _setup(seed, b=24, v=300):
    rng = np.random.default_rng(seed)
    l = (rng.standard_normal((b, v)) * 3).astype(np.float16)
    l[:, rng.random(v) < 0.1] = -np.inf
    table = np.zeros((b + 2, (v + 7) // 8 * 8), np.uint16)
    for s in range(b + 2):
        table[s, rng.choice(v, 30, replace=False)] = 0x8000
        gen = rng.choice(v, 20, replace=False)
        table[s, gen] |= rng.integers(1, 6, 20).astype(np.uint16)
    slots = rng.permutation(b + 2)[:b].astype(np.int64)
    slots[::5] = -1
    T = rng.choice([0.0, 0.7, 1.0, 1.3], b).astype(np.float32)
    K = rng.choice([0, 0, 5, 40], b).astype(np.int32)
    P = rng.choice([1.0, 0.9, 0.5], b).astype(np.float32)
    keys = np.stack([rng.integers(0, 2 ** 63, b), np.arange(b)], 1).astype(np.int64)
    ctr = rng.integers(0, 2 ** 40, b).astype(np.int64)
    opts = dict(min_p=rng.choice([0.0, 0.05, 0.3], b).astype(np.float32),
                repetition_penalty=rng.choice([0.8, 1.0, 1.3], b).astype(np.float32),
                frequency_penalty=rng.choice([0.0, 0.4, -0.2], b).astype(np.float32),
                presence_penalty=rng.choice([0.0, 0.6, -0.5], b).astype(np.float32), slots=slots)
    return l, T, K, P, keys, ctr, table, opts


def _run(seed, faults=(), n=5):
    l, T, K, P, keys, ctr, table, opts = _setup(seed)
    before = table.copy()
    tok, lp, ids, lps = R.sample_np(l, T, K, P, keys, ctr, faults, penalty_table=table, logprobs=n, **opts)
    R.check_tokens(l, T, K, P, keys, ctr, tok, penalty_table=before, logprob=lp, top_ids=ids, top_logprobs=lps, **opts)
    return l, tok, before, table, opts


def test_penalised_logits_follow_the_rule_bit_for_bit():
    rng = np.random.default_rng(1)
    v = 4000
    row = (rng.standard_normal(v) * 20).astype(np.float16)
    row[:40] = [-np.inf, np.inf, 65504, -65504, 0.0, -0.0] * 6 + [1.0, -1.0, 0.5, -0.5]
    ent = rng.integers(0, 1 << 16, v).astype(np.uint16)
    ent[::7] = 0
    for r, f, q in [(1.3, 0.4, 0.6), (0.7, -0.3, -1.0), (1e-30, 1e30, 0.0), (1e30, 0.0, 3e38)]:
        got = R.penalise(row, ent, r, f, q)
        l = row.astype(np.float64)
        c = (ent & 0x7FFF).astype(np.float64)
        hit = ((ent & 0x8000) != 0) | (c > 0)
        f32 = lambda x: np.float32(x).astype(np.float64)          # noqa: E731
        want = np.empty(v, np.float16)
        for i in range(v):
            x = l[i]
            if x == -np.inf:
                want[i] = -np.inf
                continue
            if hit[i]:
                x = f32(x / f32(r)) if x > 0 else f32(x * f32(r))
            with np.errstate(all="ignore"):
                x = f32(x - f32(c[i] * f32(f)))
                if c[i] > 0:
                    x = f32(x - f32(q))
            x = -65504.0 if np.isnan(x) else min(max(x, -65504.0), 65504.0)
            want[i] = np.float16(x)
        assert np.array_equal(got.view(np.uint16), want.view(np.uint16)), (r, f, q)


@pytest.mark.parametrize("seed", range(4))
def test_the_numpy_sampler_passes_and_records_each_token_once(seed):
    l, tok, before, after, opts = _run(seed)
    want = before.copy()
    for s, t in zip(opts["slots"], tok):
        if s >= 0 and t >= 0:
            want[s, t] += 1
    assert np.array_equal(after, want)


def test_neutral_options_and_no_state_are_the_plain_sampler():
    l, T, K, P, keys, ctr, table, opts = _setup(5)
    plain = R.sample_np(l, T, K, P, keys, ctr)
    z = np.zeros_like(table)
    got = R.sample_np(l, T, K, P, keys, ctr, penalty_table=z, slots=np.arange(len(l)))
    assert np.array_equal(plain, got)
    got = R.sample_np(l, T, K, P, keys, ctr, penalty_table=table, slots=np.full(len(l), -1), repetition_penalty=1.7,
                      frequency_penalty=2.0, presence_penalty=3.0)
    assert np.array_equal(plain, got)


def test_counts_saturate():
    l = np.zeros((1, 16), np.float16)
    table = np.full((1, 16), 0x7FFF | 0x8000, np.uint16)
    R.sample_np(l, 0.0, 0, 1.0, [(0, 0)], [0], penalty_table=table, slots=[0])
    assert table[0, 0] == 0xFFFF
    t2 = np.full((1, 16), 0x7FFF, np.uint16)
    R.sample_np(l, 0.0, 0, 1.0, [(0, 0)], [0], ("no_saturate",), penalty_table=t2, slots=[0])
    assert t2[0, 0] == 0x8000                           # the fault: the count wraps into the prompt bit


def _rejects(faults, rule_words, seeds=range(6), n=5):
    for seed in seeds:
        try:
            _run(seed, faults, n)
        except R.SampleMismatch as e:
            assert any(w in str(e) for w in rule_words), str(e)
            return
    raise AssertionError(f"fault {faults} was never rejected")


@pytest.mark.parametrize("fault", ["presence_on_prompt", "rep_divide_all", "order"])
def test_penalty_faults_are_rejected(fault):
    _rejects((fault,), ["rule"])


def test_penalising_minus_infinity_is_rejected():
    # the fault turns -inf into -65504: with 3 finite tokens the top-20 list must be padded, and it is not
    l = np.full((2, 64), -np.inf, np.float16)
    l[:, :3] = [1.0, 2.0, 3.0]
    args = (l, 1.0, 0, 1.0, np.zeros((2, 2), np.int64), np.arange(2))
    opts = dict(slots=[0, 1], repetition_penalty=1.2, frequency_penalty=0.1)
    for faults, ok in [((), True), (("neginf_penalised",), False)]:
        table = np.full((2, 64), 0x8001, np.uint16)
        before = table.copy()
        tok, lp, ids, lps = R.sample_np(*args, faults, penalty_table=table, logprobs=20, **opts)
        check = lambda: R.check_tokens(*args, tok, penalty_table=before, logprob=lp, top_ids=ids, top_logprobs=lps, **opts)  # noqa
        if ok:
            check()
        else:
            with pytest.raises(R.SampleMismatch, match="top-n"):
                check()


@pytest.mark.parametrize("fault", ["minp_short", "minp_long"])
def test_min_p_one_token_off_is_rejected(fault):
    _rejects((fault,), ["min-p", "draw", "top-p"])


def test_logprob_beyond_its_bound_is_rejected():
    _rejects(("logprob_off",), ["logprob"])


def test_top_n_ties_toward_the_higher_index_are_rejected():
    rng = np.random.default_rng(3)
    l = rng.integers(-3, 3, (4, 200)).astype(np.float16)
    args = (l, 1.0, 0, 1.0, np.zeros((4, 2), np.int64), np.arange(4))
    tok, lp, ids, lps = R.sample_np(*args, logprobs=20)
    R.check_tokens(*args, tok, logprob=lp, top_ids=ids, top_logprobs=lps)
    tok, lp, ids, lps = R.sample_np(*args, ("topn_tie_high",), logprobs=20)
    with pytest.raises(R.SampleMismatch, match="top-n"):
        R.check_tokens(*args, tok, logprob=lp, top_ids=ids, top_logprobs=lps)


def test_invalid_rows_and_parameters():
    l = np.zeros((4, 50), np.float16)
    l[1] = -np.inf
    l[2, 3] = np.nan
    opts = dict(min_p=[0.0, 0.0, 0.0, 1.5], logprobs=3)
    tok, lp, ids, lps = R.sample_np(l, 1.0, 0, 1.0, np.zeros((4, 2), np.int64), np.arange(4), **opts)
    assert tok.tolist() == [tok[0], -1, -1, -1] and tok[0] >= 0
    assert np.isnan(lp[1:]).all() and (ids[1:] == -1).all() and np.isnan(lps[1:]).all()
    R.check_tokens(l, 1.0, 0, 1.0, np.zeros((4, 2), np.int64), np.arange(4), tok, min_p=opts["min_p"], logprob=lp, top_ids=ids,
                   top_logprobs=lps)
    for bad in [dict(repetition_penalty=0.0), dict(repetition_penalty=np.inf), dict(frequency_penalty=np.nan),
                dict(presence_penalty=-np.inf)]:
        t = R.sample_np(l[:1], 1.0, 0, 1.0, [(0, 0)], [0], penalty_table=np.zeros((1, 56), np.uint16), slots=[0], **bad)
        assert t.tolist() == [-1]


def test_logprob_bound_is_small_and_positive():
    for d, z, v in [(0.0, 1.0, 128), (-30.0, 5e4, 128256), (-1e4, 1.0, 32000)]:
        b = R.lp_bound(d, d - np.log(z), z, v)
        assert 0 < b < 1e-3 + 2.0 ** -24 * 2 * abs(d)
