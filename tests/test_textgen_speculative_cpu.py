"""CPU suite: speculative decoding in the serving harness (atom_b200/textgen.py) -- verify steps in the scheduler and the decode
runner, page accounting around them, the report's "speculative" entry -- with the numpy proposer and draft sampler of
tests/spec_ref.py standing in for the kernels and a stand-in model whose greedy output cycles with a short period."""
import numpy as np
import pytest
import torch

from atom_b200 import textgen as tg
from atom_b200.kvcache import KvPoolInt4
from tests import sample_ref64 as R
from tests import spec_ref as SR

VOCAB = 97
PERIOD = 5


class _CycleLM:
    """Greedy continuation of id t is (t % PERIOD) + 1: after one token the output cycles 1, 2, .., PERIOD.  Sampled runs see
    logits that favour that token without excluding the others."""
    config = type("Config", (), {"vocab_size": VOCAB})

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        assert ids.numel() == blen.doff + blen.decode * blen.decode_len
        nxt = ids.long() % PERIOD + 1
        x = torch.sin(ids.double()[:, None] * 0.3 + torch.arange(VOCAB, dtype=torch.float64)[None])
        return (x + 4 * torch.nn.functional.one_hot(nxt, VOCAB)).float(), None


class _ProposeLog:
    """propose_op: the numpy commit and proposal, recording (emitted, drafts offered) per sequence and step; never_match
    discards every proposal."""

    def __init__(self, never_match=False):
        self.steps, self.never_match = [], never_match

    def __call__(self, tokens, cands, row_indptr, slots, history, lengths, out, k, nmin, nmax):
        c = np.asarray(cands.cpu()).reshape(-1)
        ip = np.asarray(row_indptr.cpu()).reshape(-1)
        SR.commit_propose_np(tokens, cands, row_indptr, slots, history, lengths, out, k, nmin, nmax)
        o = out.numpy()
        self.steps.append([(int(o[i, 0]), int(np.count_nonzero(c[ip[i]:ip[i + 1]] >= 0))) for i in range(len(ip) - 1)])
        if self.never_match:
            o[:, 1] = 0
            o[:, k + 3:] = -1
        return out


def _run(cfg, rs, use_runner, maxlen=96, block=16, pool_pages=None, propose=None, sample_op=None):
    cap = pool_pages or tg.pool_capacity(cfg.batch_size, maxlen + cfg.shared_prefix, block) + 8
    pool = KvPoolInt4(1, 2, 128, cap, block, torch.device("cpu"))
    propose = propose or _ProposeLog()
    runner = None
    if use_runner:
        runner = tg.DecodeGraphRunner(_CycleLM(), pool, "cpu", max_pages_per_seq=(maxlen + cfg.shared_prefix) // block + 2,
                                      capture=False, sampling=cfg.sampling, sample_op=sample_op, speculate=cfg.speculate,
                                      propose_op=propose, draft_sample_op=SR.sample_draft_tokens_np)
    res = tg.run_textgen(_CycleLM(), rs, cfg, pool, torch.device("cpu"), keep_tokens=True, decode_runner=runner,
                         sample_op=sample_op, propose_op=propose, draft_sample_op=SR.sample_draft_tokens_np)
    return res, pool, propose


CASES = [(None, 0, ()), (5, 0, ()), (None, 20, ()), (7, 20, ()), (None, 0, (4,)), (6, 20, (2, 5))]


@pytest.mark.parametrize("chunk,shared,stops", CASES)
@pytest.mark.parametrize("use_runner", [False, True])
def test_greedy_speculation_gives_the_greedy_tokens(chunk, shared, stops, use_runner):
    rs = tg.generate_request_set(12, 64)
    base = tg.TextGenConfig(4, prefill_chunk=chunk, shared_prefix=shared, stop_token_ids=stops)
    ref, _, _ = _run(base, rs, False)
    cfg = tg.TextGenConfig(4, prefill_chunk=chunk, shared_prefix=shared, stop_token_ids=stops,
                           speculate=tg.SpeculativeParams(num_draft=4, ngram_max=3, ngram_min=1))
    res, pool, log = _run(cfg, rs, use_runner)
    assert res.tokens == ref.tokens
    assert pool.num_free_blocks == pool.capacity
    if use_runner:
        assert res.graphed_steps > 0
    verify = [s for s in log.steps if any(d for _, d in s)]
    assert verify, "no verify step ran"
    rep = tg.report(rs, cfg, res)["speculative"]
    assert rep["emitted_tokens"] == int(res.output_lens.sum()) - len(rs)
    assert rep["verify_steps"] > 0 and rep["accepted_tokens"] <= rep["drafted_tokens"]
    if not stops:                                   # (a stop id in the cycle ends every request within a few tokens)
        full = [e == d + 1 for s in verify for e, d in s if d]
        assert any(full) and not all(full), "need both fully accepted and partly rejected drafts"
        assert 1 < rep["tokens_per_sequence_per_verify_step"] <= 5


@pytest.mark.parametrize("shared", [0, 20])
def test_verify_steps_never_wait_for_a_page(shared):
    # a pool that holds about two requests at a time: admission is limited by pages, so the reserve for K + 1 tokens per
    # running request is what keeps every verify step and every commit within the pool
    rs = tg.generate_request_set(10, 64)
    for k in (1, 4, 7):
        cfg = tg.TextGenConfig(4, shared_prefix=shared, speculate=tg.SpeculativeParams(num_draft=k))
        res, pool, _ = _run(cfg, rs, True, block=8, pool_pages=(64 + shared) // 8 * 2 + 6)
        assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
        assert pool.num_free_blocks == pool.capacity


def test_sampled_speculation_without_matches_is_the_plain_sampled_run():
    rs = tg.generate_request_set(9, 64)
    sp = tg.SamplingParams(0.8, top_k=30, top_p=0.95, seed=11)
    ref, _, _ = _run(tg.TextGenConfig(3, sampling=sp), rs, False, sample_op=R.sample_tokens_np)
    for use_runner in (False, True):
        cfg = tg.TextGenConfig(3, sampling=sp, speculate=tg.SpeculativeParams())
        res, pool, log = _run(cfg, rs, use_runner, propose=_ProposeLog(never_match=True), sample_op=R.sample_tokens_np)
        assert res.tokens == ref.tokens
        assert res.speculative["verify_steps"] == 0
        assert pool.num_free_blocks == pool.capacity


def test_sampled_speculation_runs_verify_steps_alike_with_and_without_the_runner():
    rs = tg.generate_request_set(9, 64)
    sp = tg.SamplingParams(0.8, seed=3, min_p=0.01)
    cfg = tg.TextGenConfig(3, prefill_chunk=9, sampling=sp, speculate=tg.SpeculativeParams(num_draft=3))
    a, pa, _ = _run(cfg, rs, False, sample_op=R.sample_tokens_np)
    b, pb, _ = _run(cfg, rs, True, sample_op=R.sample_tokens_np)
    assert a.tokens == b.tokens and a.speculative == b.speculative
    assert a.speculative["verify_steps"] > 0
    assert pa.num_free_blocks == pa.capacity and pb.num_free_blocks == pb.capacity


def test_speculation_off_is_the_plain_harness():
    rs = tg.generate_request_set(8, 64)
    cfg = tg.TextGenConfig(4, prefill_chunk=6)
    res, _, log = _run(cfg, rs, True)
    assert not log.steps and res.speculative is None
    assert "speculative" not in tg.report(rs, cfg, res)


def test_speculation_refuses_penalties_and_bad_parameters():
    rs = tg.generate_request_set(2, 32)
    sp = tg.SamplingParams(0.7, repetition_penalty=1.2)
    with pytest.raises(ValueError):
        _run(tg.TextGenConfig(2, sampling=sp, speculate=tg.SpeculativeParams()), rs, False, sample_op=R.sample_tokens_np)
    for bad in ({"num_draft": 0}, {"num_draft": 8}, {"ngram_min": 0}, {"ngram_min": 3, "ngram_max": 2}):
        with pytest.raises(ValueError):
            tg.SpeculativeParams(**bad)


@pytest.mark.parametrize("shared,chunk", [(0, None), (12, 5)])
def test_a_pool_of_pool_capacity_pages_serves_every_request(shared, chunk):
    # pool_capacity(..., num_draft=K) is the pool speculation needs: every request reaches its full length, verify growth
    # included, with small pages so that verify steps cross page boundaries
    rs = tg.generate_request_set(10, 48)
    for k in (1, 4, 7):
        cfg = tg.TextGenConfig(3, prefill_chunk=chunk, shared_prefix=shared, speculate=tg.SpeculativeParams(num_draft=k))
        pages = tg.pool_capacity(3, 48 + shared, 4, num_draft=k)
        res, pool, _ = _run(cfg, rs, True, maxlen=48, block=4, pool_pages=pages)
        assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
        assert pool.num_free_blocks == pool.capacity
    assert tg.pool_capacity(3, 48, 4) == tg.pool_capacity(3, 48, 4, num_draft=0) == 3 * 13
    assert tg.pool_capacity(3, 48, 4, num_draft=7) == 3 * 15


def test_admission_keeps_room_for_the_first_verify_step():
    # a request admitted while speculating reserves its prompt, its first token and K + 1 more tokens
    rs = tg.RequestSet(np.array([9, 9], np.int32), np.array([5, 5], np.int32))
    pool = KvPoolInt4(1, 2, 128, 64, 4, torch.device("cpu"))
    for k, want in ((0, 3 + 1), (4, 4), (7, 5)):
        sched = tg.TextGenScheduler(rs, 2, pool, "cpu", vocab_size=VOCAB, penalty_slots=True, num_draft=k)
        assert sched._pages_needed(9) == want              # ceil((9 + 1 + k + 1) / 4) pages, or the plain prompt + spare


def test_the_runner_keeps_its_histories_and_graphs_across_request_sets():
    # a warm-up on one request set and a run on another must not drop the runner's graphs when the histories still fit
    big, small = tg.generate_request_set(6, 64), tg.generate_request_set(2, 64)
    cfg = tg.TextGenConfig(2, speculate=tg.SpeculativeParams())
    pool = KvPoolInt4(1, 2, 128, tg.pool_capacity(2, 64, 16, 4) + 8, 16, torch.device("cpu"))
    runner = tg.DecodeGraphRunner(_CycleLM(), pool, "cpu", max_pages_per_seq=64 // 16 + 3, capture=False, speculate=cfg.speculate,
                                  propose_op=_ProposeLog(), draft_sample_op=SR.sample_draft_tokens_np)
    kw = dict(keep_tokens=True, decode_runner=runner, propose_op=_ProposeLog(), draft_sample_op=SR.sample_draft_tokens_np)
    tg.run_textgen(_CycleLM(), big, cfg, pool, torch.device("cpu"), **kw)
    hist, entries = runner.history, dict(runner._entries)
    assert entries
    tg.run_textgen(_CycleLM(), small, cfg, pool, torch.device("cpu"), **kw)
    assert runner.history is hist and all(runner._entries.get(key) is e for key, e in entries.items())
    longer = tg.RequestSet(np.array([60], np.int32), np.array([40], np.int32))
    tg.run_textgen(_CycleLM(), longer, tg.TextGenConfig(2, speculate=cfg.speculate), pool, torch.device("cpu"), **kw)
    assert runner.history is not hist and runner.history[0].size(1) >= 60 + 40 + 4 + 1
