"""CPU suite: beam search in the serving harness (atom_b200/textgen.py) -- the scheduler's beams, deferred page copies and
finished hypotheses, the decode runner's beam step (capture=False) and the report's "beam" entry -- with the numpy beam step and
page copy of tests/beam_ref.py standing in for the kernels and a Markov stand-in model."""
import numpy as np
import pytest
import torch

from atom_b200 import textgen as tg
from atom_b200.kvcache import KvPoolInt4
from tests import beam_ref as BR

VOCAB = 23


def _table():
    x = np.sin(np.arange(VOCAB)[:, None] * 0.37 + np.arange(VOCAB)[None] * 1.3) * 3 + \
        np.cos(np.arange(VOCAB)[:, None] * np.arange(VOCAB)[None] * 0.11)
    return x.astype(np.float16)


class _MarkovLM:
    """The logits row after token t is row t of a fixed FP16 table: greedy and beam search both follow it exactly."""
    config = type("Config", (), {"vocab_size": VOCAB})
    table = torch.from_numpy(_table().astype(np.float32))

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        return self.table[ids.long()], None


def _run(cfg, rs, use_runner, maxlen=40, block=8, exact_pool=False, copy_op=None):
    cap = tg.pool_capacity(cfg.batch_size, maxlen + cfg.shared_prefix, block) + (0 if exact_pool else 8)
    pool = KvPoolInt4(1, 2, 128, cap, block, torch.device("cpu"))
    pool.buf.zero_()
    pool.param.zero_()
    copy_op = copy_op or BR.CopyLog()
    runner = None
    if use_runner and cfg.beam is not None:
        runner = tg.DecodeGraphRunner(_MarkovLM(), pool, "cpu", max_pages_per_seq=(maxlen + cfg.shared_prefix) // block + 2,
                                      capture=False, beam=cfg.beam, stop_token_ids=cfg.stop_token_ids,
                                      beam_select_op=BR.beam_select_tokens_np, copy_op=copy_op)
    elif use_runner:
        runner = tg.DecodeGraphRunner(_MarkovLM(), pool, "cpu", max_pages_per_seq=(maxlen + cfg.shared_prefix) // block + 2,
                                      capture=False)
    res = tg.run_textgen(_MarkovLM(), rs, cfg, pool, torch.device("cpu"), keep_tokens=True, decode_runner=runner,
                         beam_select_op=BR.beam_select_tokens_np, copy_op=copy_op)
    assert pool.num_free_blocks == pool.capacity, "pages leaked"
    return res, copy_op


def _rs(n=7, maxlen=40):
    return tg.generate_request_set(n, maxlen)


def _prompts(rs):
    rng = np.random.Generator(np.random.PCG64(seed=tg.SEED))
    return [rng.integers(0, VOCAB, int(p)).tolist() for p in rs.prompt_lens]


def _expected_copies(table, prompt, width, alpha, n_out, stops, ctx, P):
    """The slots of every page copy the reference's beam search implies for one request: at each step that does not end it, a
    parent with c >= 2 children is forked c - 1 times, and each fork copies the n % P cached tokens of its partly filled page."""
    req = BR.BeamRequest(width, alpha, n_out, stops)
    rows, k, out = [table[prompt[-1]]], 0, []
    while True:
        res = BR.beam_select_np(np.stack(rows), [0, len(rows)], [s for _, s in req.live], width, stops)
        parents = req.step(res[0][0], res[1][0], res[2][0], res[3][0], lambda r: r)
        if req.done:
            return out
        n = ctx + k                                          # tokens the parents hold: the context and k generated ones
        for b in set(parents):
            if parents.count(b) >= 2 and n % P:
                out += [n % P] * (parents.count(b) - 1)
        k += 1
        rows = [table[t[-1]] for t, _ in req.live]


CONFIGS = [dict(), dict(prefill_chunk=5), dict(shared_prefix=11), dict(stop_token_ids=(3, 17)),
           dict(prefill_chunk=6, shared_prefix=9, stop_token_ids=(5,))]


@pytest.mark.parametrize("use_runner", [False, True])
@pytest.mark.parametrize("extra", CONFIGS)
def test_width_one_is_greedy(extra, use_runner):
    rs = _rs()
    greedy, _ = _run(tg.TextGenConfig(batch_size=4, **extra), rs, use_runner)
    beam, copies = _run(tg.TextGenConfig(batch_size=4, beam=tg.BeamSearchParams(1), **extra), rs, use_runner)
    assert beam.tokens == greedy.tokens
    assert beam.output_lens.tolist() == greedy.output_lens.tolist()
    assert not copies.pairs                              # one beam never forks
    if use_runner:
        assert beam.graphed_steps > 0


@pytest.mark.parametrize("width,alpha,stops", [(2, 0.0, ()), (4, 1.0, (3, 17)), (8, 0.6, (5,)), (4, -0.5, (2,))])
@pytest.mark.parametrize("use_runner", [False, True])
def test_matches_reference(width, alpha, stops, use_runner):
    rs = _rs()
    cfg = tg.TextGenConfig(batch_size=2 * width, beam=tg.BeamSearchParams(width, alpha), stop_token_ids=stops, prefill_chunk=7)
    res, copies = _run(cfg, rs, use_runner, exact_pool=True)
    table = _table()
    for i, prompt in enumerate(_prompts(rs)):
        req = BR.beam_search_ref(lambda t: table[t], table[prompt[-1]], width, alpha, int(rs.output_lens[i]), stops)
        tokens, _, score = req.best()
        assert res.tokens[i] == tokens, i
        assert res.beam_scores[i] == score
    # a copy is the partly filled page of a parent with a second child: never a full page, its source still held, and exactly
    # one per further child of every parent the reference forks at a length that is not a whole number of pages
    assert copies.pairs and all(1 <= n < 8 and held >= 1 and dst_held == 1 for _, _, n, held, dst_held in copies.pairs)
    want = []
    for i, prompt in enumerate(_prompts(rs)):
        want += _expected_copies(table, prompt, width, alpha, int(rs.output_lens[i]), stops, len(prompt), 8)
    assert sorted(n for _, _, n, _, _ in copies.pairs) == sorted(want)
    rep = tg.report(rs, cfg, res)["beam"]
    assert rep["width"] == width and rep["page_copies"] == len(copies.pairs)
    assert rep["bytes_copied"] == sum(n for _, _, n, _, _ in copies.pairs) * 1 * 2 * 2 * 68
    assert rep["stop_finished_requests"] == sum(bool(t) and t[-1] in stops for t in res.tokens)


def test_wide_beam_finds_exhaustive_best():
    V = 8
    table = _table()[:V, :V].copy()

    class LM(_MarkovLM):
        config = type("Config", (), {"vocab_size": V})

        def __call__(self, ids, blen, prefill_kv, decode_kv):
            return torch.from_numpy(table.astype(np.float32))[ids.long()], None
    rs = tg.RequestSet(np.array([3, 5, 2], np.int32), np.array([2, 2, 2], np.int32))
    cfg = tg.TextGenConfig(batch_size=8, beam=tg.BeamSearchParams(8))
    pool = KvPoolInt4(1, 2, 128, tg.pool_capacity(8, 16, 4), 4, torch.device("cpu"))
    res = tg.run_textgen(LM(), rs, cfg, pool, torch.device("cpu"), keep_tokens=True, beam_select_op=BR.beam_select_tokens_np,
                         copy_op=BR.CopyLog())
    rng = np.random.Generator(np.random.PCG64(seed=tg.SEED))
    for i in range(3):
        prompt = rng.integers(0, V, int(rs.prompt_lens[i])).tolist()
        score, tokens = BR.exhaustive_best(lambda t: table[t], table[prompt[-1]], 0.0, 2)
        assert res.tokens[i] == tokens and res.beam_scores[i] == pytest.approx(score, abs=1e-6)


def test_incompatible_configs_raise():
    rs = _rs(2)
    pool = KvPoolInt4(1, 2, 128, 64, 8, torch.device("cpu"))
    bad = [tg.TextGenConfig(batch_size=8, beam=tg.BeamSearchParams(2), sampling=tg.SamplingParams(1.0)),
           tg.TextGenConfig(batch_size=8, beam=tg.BeamSearchParams(2), speculate=tg.SpeculativeParams()),
           tg.TextGenConfig(batch_size=3, beam=tg.BeamSearchParams(4))]
    for cfg in bad:
        with pytest.raises(ValueError):
            tg.run_textgen(_MarkovLM(), rs, cfg, pool, torch.device("cpu"), beam_select_op=BR.beam_select_tokens_np,
                           copy_op=BR.CopyLog())
    for w, a in ((0, 0.0), (9, 0.0), (2, float("nan")), (2, float("inf"))):
        with pytest.raises(ValueError):
            tg.BeamSearchParams(w, a)


def test_fork_defers_copy():
    pool = KvPoolInt4(1, 2, 128, 8, 4, torch.device("cpu"))
    pool.buf.copy_(torch.randint(0, 256, pool.buf.shape, dtype=torch.uint8))
    from atom_b200.kvcache import KvCacheInt4
    a = KvCacheInt4(pool, 6)
    before = pool.buf.clone()
    copies = []
    b = a.fork(copies=copies)
    assert copies == [(a.indicies[1], b.indicies[1], 2)] and b.indicies[0] == a.indicies[0]
    assert torch.equal(pool.buf, before)                 # nothing copied yet
    c = a.fork()                                         # the default still copies at once
    assert torch.equal(pool.buf[c.indicies[1]], pool.buf[a.indicies[1]])
    full = KvCacheInt4(pool, 4)
    full.fork(copies=copies)
    assert len(copies) == 1                              # a full last page is shared, not copied


def test_runner_refuses_a_bad_page_copy():
    pool = KvPoolInt4(1, 2, 128, 16, 8, torch.device("cpu"))
    from atom_b200.kvcache import KvCacheInt4
    kv = [KvCacheInt4(pool, 5), KvCacheInt4(pool, 3)]
    runner = tg.DecodeGraphRunner(_MarkovLM(), pool, "cpu", max_pages_per_seq=4, capture=False, beam=tg.BeamSearchParams(2),
                                  beam_select_op=BR.beam_select_tokens_np, copy_op=BR.CopyLog())
    for bad in ((kv[0].indicies[0], kv[0].indicies[0], 3), (kv[0].indicies[0], 16, 3), (kv[0].indicies[0], kv[1].indicies[0], 9)):
        with pytest.raises(RuntimeError):
            runner.run_beam([1, 2], kv, [bad], [0, 2], [0.0, 0.0])
