"""CPU suite: penalties, min-p, log-probabilities and stop tokens in the serving harness (atom_b200/textgen.py) -- penalty-table
slots allocated, set up with the whole prompt, freed and reused; each request's row ends as its prompt bits plus the histogram
of its tokens; the same tokens and log-probabilities with and without chunked prefill, shared prefixes and the decode runner;
stop ids ending requests early.  The numpy sampler of tests/sample_penalty_ref64.py stands in for the kernel."""
import numpy as np
import pytest
import torch

from atom_b200 import textgen as tg
from atom_b200.kvcache import KvPoolInt4
from tests import sample_penalty_ref64 as R

VOCAB = 97


class _LM:
    """Stand-in model: every row's logits are a fixed smooth function of its input id (so penalties change what is drawn)."""
    config = type("Config", (), {"vocab_size": VOCAB})

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        x = ids.double()[:, None] * 13 + torch.arange(VOCAB, dtype=torch.float64)[None] * 7
        return (torch.sin(x * 0.37) * 3 + torch.cos(x * 0.11)).float(), None


class _SlotLog:
    """slot_init_op: records every (slot, prompt) and the row each slot held just before it was set up again."""

    def __init__(self):
        self.inits, self.rows_before = [], []

    def __call__(self, table, slot, prompt):
        self.rows_before.append((slot, R._table_np(table)[slot].copy()))
        self.inits.append((slot, list(prompt)))
        R.init_penalty_slot_np(table, slot, prompt)


def _run(cfg, rs, use_runner, maxlen=80, block=16, slot_log=None):
    pool = KvPoolInt4(1, 2, 128, tg.pool_capacity(cfg.batch_size, maxlen + cfg.shared_prefix, block) + 8, block, torch.device("cpu"))
    runner = None
    if use_runner:
        runner = tg.DecodeGraphRunner(_LM(), pool, "cpu", max_pages_per_seq=(maxlen + cfg.shared_prefix) // block + 2, capture=False,
                                      sampling=cfg.sampling, sample_op=R.sample_tokens_np)
    slot_log = slot_log or _SlotLog()
    res = tg.run_textgen(_LM(), rs, cfg, pool, torch.device("cpu"), keep_tokens=True, decode_runner=runner,
                         sample_op=R.sample_tokens_np, slot_init_op=slot_log)
    return res, pool, runner


def _prompts(rs, shared):
    rng = np.random.Generator(np.random.PCG64(seed=tg.SEED))
    system = np.random.Generator(np.random.PCG64(seed=tg.SEED + 1)).integers(0, VOCAB, shared).tolist() if shared else []
    return [system + rng.integers(0, VOCAB, int(n)).tolist() for n in rs.prompt_lens]


SP = tg.SamplingParams(0.9, top_k=30, top_p=0.95, seed=11, min_p=0.05, repetition_penalty=1.3, frequency_penalty=0.4,
                       presence_penalty=-0.3, logprobs=5)


@pytest.mark.parametrize("chunk,shared", [(None, 0), (6, 0), (None, 24), (5, 24)])
def test_slots_are_set_up_with_the_whole_prompt_freed_and_reused(chunk, shared):
    rs = tg.generate_request_set(9, 64)
    log = _SlotLog()
    res, pool, _ = _run(tg.TextGenConfig(3, prefill_chunk=chunk, shared_prefix=shared, sampling=SP), rs, True, slot_log=log)
    prompts = _prompts(rs, shared)
    assert [p for _, p in log.inits] == prompts                    # request order, system prompt first
    slots = [s for s, _ in log.inits]
    assert set(slots) <= {0, 1, 2} and len(slots) == len(rs)       # batch_size slots, reused
    # a slot's row when it is set up again is its previous holder's prompt bits + the histogram of that holder's tokens
    reused = 0
    for r, (s, _) in enumerate(log.inits):
        later = [i for i in range(r + 1, len(log.inits)) if log.inits[i][0] == s]
        if later:
            want = np.zeros(VOCAB, np.uint16)
            want[prompts[r]] = 0x8000
            np.add.at(want, res.tokens[r], 1)
            assert np.array_equal(log.rows_before[later[0]][1][:VOCAB], want), r
            reused += 1
    assert reused >= len(rs) - 3
    assert pool.num_free_blocks == pool.capacity


def test_final_table_rows_match_the_histograms():
    rs = tg.generate_request_set(5, 48)
    captured = {}
    log = _SlotLog()

    def sample(logits, *args, **kw):
        captured["table"] = kw.get("penalty_table")
        return R.sample_tokens_np(logits, *args, **kw)
    pool = KvPoolInt4(1, 2, 128, tg.pool_capacity(5, 64, 16) + 8, 16, torch.device("cpu"))
    res = tg.run_textgen(_LM(), rs, tg.TextGenConfig(5, sampling=SP), pool, torch.device("cpu"), keep_tokens=True,
                         sample_op=sample, slot_init_op=log)
    table = R._table_np(captured["table"])
    prompts = _prompts(rs, 0)
    for r, (s, _) in enumerate(log.inits):                         # 5 slots for 5 requests: no reuse
        want = np.zeros(table.shape[1], np.uint16)
        want[prompts[r]] = 0x8000
        np.add.at(want, res.tokens[r], 1)
        assert np.array_equal(table[s], want), r
    assert len(res.logprobs) == len(rs) and all(len(a) == len(t) for a, t in zip(res.logprobs, res.tokens))
    assert all(len(ids) == 5 and len(lps) == 5 for row in res.top_logprobs for ids, lps in row)


def test_tokens_and_logprobs_do_not_depend_on_chunking_shared_prefix_or_the_runner():
    rs = tg.generate_request_set(10, 72)
    # frequency and presence count generated tokens only, so a system prompt does not change what is drawn
    sp = tg.SamplingParams(0.8, top_p=0.9, seed=3, min_p=0.02, frequency_penalty=0.5, presence_penalty=0.7, logprobs=4)
    base, _, _ = _run(tg.TextGenConfig(4, sampling=sp), rs, False)
    for chunk, shared, runner in [(None, 0, True), (7, 0, False), (7, 0, True), (None, 20, True), (6, 20, False)]:
        r, pool, _ = _run(tg.TextGenConfig(4, prefill_chunk=chunk, shared_prefix=shared, sampling=sp), rs, runner)
        assert r.tokens == base.tokens and r.logprobs == base.logprobs and r.top_logprobs == base.top_logprobs, (chunk, shared)
        assert pool.num_free_blocks == pool.capacity
    # the repetition penalty also covers the prompt: same tokens with and without chunking and the runner
    a, _, _ = _run(tg.TextGenConfig(4, sampling=SP), rs, False)
    b, _, runner = _run(tg.TextGenConfig(4, prefill_chunk=5, sampling=SP), rs, True)
    assert a.tokens == b.tokens and a.logprobs == b.logprobs and b.graphed_steps > 0
    plain, _, _ = _run(tg.TextGenConfig(4, sampling=tg.SamplingParams(0.9, top_k=30, top_p=0.95, seed=11)), rs, False)
    assert plain.tokens != a.tokens and plain.logprobs is None


def test_runner_buffer_gains_the_option_block_only_when_used():
    block, maxp = 16, 4
    pool = KvPoolInt4(1, 2, 128, 16, block, torch.device("cpu"))
    seen = {}

    def op(logits, *args, **kw):
        seen["kw"] = kw
        n = logits.size(0)
        out = torch.zeros(n, dtype=torch.int32)
        return (out, torch.zeros(n), torch.zeros(n, 2, dtype=torch.int32), torch.zeros(n, 2)) if "logprobs" in kw else out
    lm = lambda ids, blen, p, kv: (torch.zeros(ids.numel(), 5), None)          # noqa: E731
    plain = tg.DecodeGraphRunner(lm, pool, "cpu", max_pages_per_seq=maxp, capture=False, sampling=tg.SamplingParams(0.7),
                                 sample_op=op)
    sp = tg.SamplingParams(0.7, min_p=0.1, repetition_penalty=1.2, frequency_penalty=0.5, presence_penalty=-0.25, logprobs=2)
    r = tg.DecodeGraphRunner(lambda ids, blen, p, kv: (torch.zeros(ids.numel(), 5), None), pool, "cpu", max_pages_per_seq=maxp,
                             capture=False, sampling=sp, sample_op=op)
    table = torch.zeros(4, 8, dtype=torch.int16)
    r.use_table(table)
    from atom_b200.kvcache import KvCacheInt4
    for b in (1, 3):
        kvs = [KvCacheInt4(pool, 5 + i) for i in range(b)]
        out = r.run([1] * b, kvs, [(i, 0) for i in range(b)], [3 - i for i in range(b)])
        for c in kvs:
            c.release()
        assert isinstance(out, tuple) and len(out) == 4
        o_sl, o_m, o_r, o_f, o_q, total = r._ext_layout(b)
        assert o_sl == plain._sampling_layout(b)[-1] and total == o_sl + 5 * b
        h = r._entries[(b, 0)]["host"].numpy()
        assert h[o_sl:o_m].tolist() == [3 - i for i in range(b)]
        for o, v in ((o_m, 0.1), (o_r, 1.2), (o_f, 0.5), (o_q, -0.25)):
            assert h[o:o + b].view(np.float32).tolist() == [np.float32(v)] * b
        kw = seen["kw"]
        assert kw["penalty_table"] is table and kw["logprobs"] == 2 and kw["slots"].dtype == torch.int32
        assert kw["min_p"].data_ptr() == r._entries[(b, 0)]["dev"].data_ptr() + 4 * o_m
        kvs = [KvCacheInt4(pool, 3) for _ in range(b)]
        plain.run([1] * b, kvs, [(i, 0) for i in range(b)])
        for c in kvs:
            c.release()
        assert plain._entries[(b, 0)]["host"].numel() == plain._sampling_layout(b)[-1] and "ext" not in plain._entries[(b, 0)]


@pytest.mark.parametrize("sampled", [False, True])
def test_stop_ids_end_requests_and_release_everything(sampled):
    rs = tg.generate_request_set(12, 80)
    sp = SP if sampled else None
    full, _, _ = _run(tg.TextGenConfig(4, sampling=sp), rs, False)
    counts = {}
    for t in full.tokens:
        for x in t[:-1]:
            counts[x] = counts.get(x, 0) + 1
    stop = max(counts, key=counts.get)                             # a token that ends several requests early
    for runner in (False, True):
        res, pool, _ = _run(tg.TextGenConfig(4, sampling=sp, stop_token_ids=(stop,)), rs, runner)
        assert pool.num_free_blocks == pool.capacity
        early = 0
        for t, f in zip(res.tokens, full.tokens):
            cut = f.index(stop) + 1 if stop in f else len(f)
            assert t == f[:cut]
            early += cut < len(f)
        assert early >= 2
        assert res.output_lens.tolist() == [len(t) for t in res.tokens]
        rep = tg.report(rs, tg.TextGenConfig(4, sampling=sp, stop_token_ids=(stop,)), res)
        assert rep["total_new_tokens"] == sum(len(t) for t in res.tokens) < int(rs.output_lens.sum())
        assert rep["stop_token_ids"] == [stop]
    plain = tg.report(rs, tg.TextGenConfig(4, sampling=sp), full)
    assert plain["total_new_tokens"] == int(rs.output_lens.sum()) and "stop_token_ids" not in plain


def test_new_sampling_params_are_validated():
    for bad in [dict(min_p=-0.1), dict(min_p=1.5), dict(repetition_penalty=0.0), dict(repetition_penalty=float("inf")),
                dict(frequency_penalty=float("nan")), dict(presence_penalty=float("inf")), dict(logprobs=21), dict(logprobs=-1)]:
        with pytest.raises(ValueError):
            tg.SamplingParams(1.0, **bad)
    assert tg.SamplingParams(1.0).asdict() == {"temperature": 1.0, "top_k": 0, "top_p": 1.0, "seed": 0}
    assert tg.SamplingParams(1.0, logprobs=0).asdict()["logprobs"] == 0
