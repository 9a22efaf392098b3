"""GPU suite (-m gpu): penalties, min-p, log-probabilities and a stop id in the serving harness -- with the small random model of
test_z_textgen_gpu.py, graphed and eager runs bit for bit equal in tokens and log-probabilities, requests ending on the stop id,
and the device table equal to the host histogram at the end; with a device stand-in model whose logits depend on the input id
only, tokens independent of batch size, chunked prefill and (with generated-token penalties) a shared prefix.  (The INT4
model's decode attention picks its KV split from the batch size, so its logits, and a draw near a boundary, may change with
the batch; the sampler's own row independence is tested in test_z_sample_penalty_gpu.py.)"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
VOCAB = 128


def _model():
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM
    dev = torch.device("cuda:0")
    torch.manual_seed(11)
    torch.set_default_dtype(torch.float16)
    try:
        with dev:
            model = LlamaForCausalLM(LlamaConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=4,
                                                 num_hidden_layers=2, vocab_size=VOCAB))
    finally:
        torch.set_default_dtype(torch.float32)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    return model.eval()


class _IdLM:
    """Device stand-in: every row's logits are a fixed function of its input id, so they do not depend on the batch."""
    config = type("Config", (), {"vocab_size": VOCAB})

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        x = ids.double()[:, None] * 13 + torch.arange(VOCAB, dtype=torch.float64, device=ids.device)[None] * 7
        return (torch.sin(x * 0.37) * 3 + torch.cos(x * 0.11)).half(), None


def _run(sp, graphs=False, batch=3, chunk=None, shared=0, stop=(), tables=None, model=None):
    from atom_b200 import ops
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvPoolInt4
    dev = torch.device("cuda:0")
    model = model or _model()
    rs = tg.generate_request_set(8, 72)
    pool = KvPoolInt4(2, 4, 128, tg.pool_capacity(batch, 72 + shared, 16) + 8, 16, dev)
    free0 = pool.num_free_blocks
    runner = tg.DecodeGraphRunner(model, pool, dev, max_pages_per_seq=(72 + shared) // 16 + 2, sampling=sp) if graphs else None

    def sample(logits, *args, **kw):
        if tables is not None and kw.get("penalty_table") is not None:
            tables["table"] = kw["penalty_table"]
        return ops.sample_tokens(logits, *args, **kw)
    res = tg.run_textgen(model, rs, tg.TextGenConfig(batch, prefill_chunk=chunk, shared_prefix=shared, sampling=sp,
                                                     stop_token_ids=stop), pool, dev, sync=torch.cuda.synchronize,
                         keep_tokens=True, decode_runner=runner, sample_op=sample)
    assert (res.graphed_steps > 0) == graphs
    assert pool.num_free_blocks == free0
    assert all(0 <= t < VOCAB for toks in res.tokens for t in toks)
    return res, rs


def _sp(**kw):
    from atom_b200 import textgen as tg
    args = dict(temperature=0.9, top_p=0.95, seed=5, min_p=0.03, repetition_penalty=1.3, frequency_penalty=0.3,
                presence_penalty=0.4, logprobs=5)
    args.update(kw)
    return tg.SamplingParams(**args)


@pytest.mark.timeout(900)
def test_graphed_and_eager_runs_agree_and_stop_ids_end_requests():
    base, rs = _run(_sp())
    g, _ = _run(_sp(), graphs=True)
    assert g.tokens == base.tokens and g.logprobs == base.logprobs and g.top_logprobs == base.top_logprobs
    assert all(np.isfinite(x) and x <= 0 for lps in base.logprobs for x in lps)
    assert all(len(ids) == 5 and ids[0] >= 0 for row in base.top_logprobs for ids, _ in row)
    stop = max({t for toks in base.tokens for t in toks[:-1]}, key=lambda t: sum(toks[:-1].count(t) for toks in base.tokens))
    a, _ = _run(_sp(), stop=(stop,))
    b, _ = _run(_sp(), graphs=True, stop=(stop,))
    assert a.tokens == b.tokens and a.logprobs == b.logprobs and a.top_logprobs == b.top_logprobs
    early = 0
    for toks, n in zip(a.tokens, rs.output_lens):
        assert stop not in toks[:-1] and (toks[-1] == stop or len(toks) == n)
        early += len(toks) < n
    assert early >= 1 and a.output_lens.tolist() == [len(t) for t in a.tokens]


@pytest.mark.timeout(900)
def test_tokens_do_not_depend_on_batch_chunking_or_shared_prefix():
    lm = _IdLM()
    a, _ = _run(_sp(), model=lm)
    for kw in (dict(batch=5, graphs=True), dict(chunk=9, graphs=True), dict(batch=2, chunk=4)):
        r, _ = _run(_sp(), model=lm, **kw)
        assert r.tokens == a.tokens and r.logprobs == a.logprobs, kw
    # frequency and presence count generated tokens only: a system prompt leaves them unchanged
    sp = _sp(repetition_penalty=1.0)
    b, _ = _run(sp, model=lm)
    assert b.tokens != a.tokens
    for kw in (dict(shared=24, graphs=True), dict(shared=24, chunk=7, batch=4)):
        assert _run(sp, model=lm, **kw)[0].tokens == b.tokens, kw
    # and a stop id ends each request on its first occurrence of it
    stop = a.tokens[0][0]
    r, _ = _run(_sp(), model=lm, graphs=True, stop=(stop,))
    assert r.tokens == [t[:t.index(stop) + 1] if stop in t else t for t in a.tokens]


@pytest.mark.timeout(900)
def test_device_table_matches_the_host_histogram():
    from atom_b200 import textgen as tg
    tables = {}
    res, rs = _run(_sp(), graphs=True, batch=8, tables=tables)                # 8 slots for 8 requests: each keeps its slot
    t = tables["table"].cpu().numpy().view(np.uint16)
    rng = np.random.Generator(np.random.PCG64(seed=tg.SEED))
    rows = set()
    for r, n in enumerate(rs.prompt_lens):
        prompt = rng.integers(0, VOCAB, int(n))
        want = np.zeros(t.shape[1], np.uint16)
        want[prompt] = 0x8000
        np.add.at(want, res.tokens[r], 1)
        hits = [s for s in range(t.shape[0]) if np.array_equal(t[s], want)]
        assert hits, r
        rows.update(hits)
    assert len(rows) == len(rs)
