"""GPU suite (-m gpu), sorted last: the continuous-batching harness with a shared system prompt end to end on the kernels with a
small random model -- the system prompt prefilled once as a root sequence, every request forked from it and continued with its
own prompt, eager and graphed decode steps, the pool back to full at the end.  Tokens are compared between runs of the shared
harness only: a prompt prefilled as a continuation can store different K/V codes than a one-shot prefill (DESIGN.md 5.3)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(seed_pages, graphs=False, shared=40, chunk=None):
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvPoolInt4
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM
    dev = torch.device("cuda:0")
    torch.manual_seed(11)
    torch.set_default_dtype(torch.float16)
    try:
        with dev:
            model = LlamaForCausalLM(LlamaConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=4,
                                                 num_hidden_layers=2, vocab_size=128))
    finally:
        torch.set_default_dtype(torch.float32)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    rs = tg.generate_request_set(7, 72)
    shared_pages = -(-shared // 16)
    pool = KvPoolInt4(2, 4, 128, tg.pool_capacity(3, 72, 16) + shared_pages + 3 + seed_pages, 16, dev)
    for _ in range(seed_pages):            # shift the page ids the requests will get
        pool.alloc_block()
    free0 = pool.num_free_blocks
    runner = tg.DecodeGraphRunner(model.eval(), pool, dev, max_pages_per_seq=72 // 16 + 1 + shared_pages) if graphs else None
    res = tg.run_textgen(model.eval(), rs, tg.TextGenConfig(3, prefill_chunk=chunk, shared_prefix=shared), pool, dev,
                         sync=torch.cuda.synchronize, keep_tokens=True, decode_runner=runner)
    assert (res.graphed_steps > 0) == graphs
    assert pool.num_free_blocks == free0
    assert res.peak_pages > 0
    assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
    assert all(0 <= t < 128 for toks in res.tokens for t in toks)
    return res.tokens


@pytest.mark.timeout(300)
def test_shared_prefix_harness_end_to_end_with_and_without_graphs_and_page_placement_independent():
    a = _run(0)
    assert _run(5) == a                    # same requests on other physical pages
    assert _run(0, graphs=True) == a       # decode-only steps replayed from CUDA graphs


@pytest.mark.timeout(300)
def test_shared_prefix_harness_with_chunked_prefill():
    a = _run(0, shared=70, chunk=24)
    assert _run(3, shared=70, chunk=24, graphs=True) == a


def _run_gqa(monkeypatch, seed_pages, graphs):
    """8 requests at batch 8 behind a 3072-token system prompt, 8 query heads over 2 KV heads: every decode batch is one group of
    8 forks with 96 shared pages, which ops.decode_cascade sends through the cascade, eagerly and in the decode graphs."""
    from atom_b200 import ops
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvPoolInt4
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM
    dev = torch.device("cuda:0")
    torch.manual_seed(11)
    torch.set_default_dtype(torch.float16)
    try:
        with dev:
            model = LlamaForCausalLM(LlamaConfig(hidden_size=1024, intermediate_size=1024, num_attention_heads=8,
                                                 num_key_value_heads=2, num_hidden_layers=2, vocab_size=128, rope_theta=5e5))
    finally:
        torch.set_default_dtype(torch.float32)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    calls = []
    real = ops._batch_decode_shared
    monkeypatch.setattr(ops, "_batch_decode_shared", lambda *a, **k: calls.append(1) or real(*a, **k))
    rs = tg.generate_request_set(8, 40)
    shared, P = 3072, 32
    pool = KvPoolInt4(2, 2, 128, 96 + 8 * 4 + seed_pages + 4, P, dev)
    for _ in range(seed_pages):
        pool.alloc_block()
    free0 = pool.num_free_blocks
    runner = tg.DecodeGraphRunner(model.eval(), pool, dev, max_pages_per_seq=96 + 4) if graphs else None
    res = tg.run_textgen(model.eval(), rs, tg.TextGenConfig(8, shared_prefix=shared), pool, dev, sync=torch.cuda.synchronize,
                         keep_tokens=True, decode_runner=runner)
    assert (res.graphed_steps > 0) == graphs
    assert calls, "no decode step ran the cascade"
    assert pool.num_free_blocks == free0
    assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
    return res.tokens


@pytest.mark.timeout(600)
def test_shared_prefix_harness_runs_the_cascade_eagerly_and_from_graphs(monkeypatch):
    a = _run_gqa(monkeypatch, 0, False)
    assert _run_gqa(monkeypatch, 7, False) == a           # other physical pages
    assert _run_gqa(monkeypatch, 0, True) == a            # decode-only steps replayed from graphs keyed on (8 rows, 1 group)
