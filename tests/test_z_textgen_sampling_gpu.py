"""GPU suite (-m gpu): sampled decoding in the serving harness with the small random model of test_z_textgen_gpu.py --
tokens independent of CUDA graphs and page placement, top_k = 1 equal to the greedy run, seeds that agree and differ, and
the kernel's tokens on real lm_head rows accepted by the float64 reference."""
import numpy as np
import pytest
import torch

from tests import sample_ref64 as R

pytestmark = pytest.mark.gpu


def _run(seed_pages, graphs=False, sampling=None, sample_op=None, shared=0):
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
    pool = KvPoolInt4(2, 4, 128, tg.pool_capacity(3, 72, 16) + seed_pages + 8, 16, dev)
    for _ in range(seed_pages):
        pool.alloc_block()
    free0 = pool.num_free_blocks
    runner = tg.DecodeGraphRunner(model.eval(), pool, dev, max_pages_per_seq=(72 + shared) // 16 + 2,
                                  sampling=sampling) if graphs else None
    res = tg.run_textgen(model.eval(), rs, tg.TextGenConfig(3, shared_prefix=shared, sampling=sampling), pool, dev,
                         sync=torch.cuda.synchronize, keep_tokens=True, decode_runner=runner, sample_op=sample_op)
    assert (res.graphed_steps > 0) == graphs
    assert pool.num_free_blocks == free0
    assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
    assert all(0 <= t < 128 for toks in res.tokens for t in toks)
    return res.tokens


def _sp(**kw):
    from atom_b200 import textgen as tg
    args = dict(temperature=0.8, top_p=0.9, seed=5)
    args.update(kw)
    return tg.SamplingParams(**args)


@pytest.mark.timeout(600)
def test_sampled_tokens_do_not_depend_on_graphs_or_page_placement():
    a = _run(0, sampling=_sp())
    assert _run(5, sampling=_sp()) == a
    assert _run(0, graphs=True, sampling=_sp()) == a
    assert _run(3, graphs=True, sampling=_sp(), shared=24) == _run(0, sampling=_sp(), shared=24)


@pytest.mark.timeout(600)
def test_top1_reproduces_greedy_and_seeds_agree_or_differ():
    greedy = _run(0)
    assert _run(0, graphs=True, sampling=_sp(top_k=1)) == greedy
    a = _run(0, graphs=True, sampling=_sp(seed=1))
    assert _run(0, graphs=True, sampling=_sp(seed=1)) == a
    assert _run(0, graphs=True, sampling=_sp(seed=2)) != a
    assert a != greedy


@pytest.mark.timeout(600)
def test_kernel_tokens_on_real_lm_head_rows_pass_the_reference():
    from atom_b200 import ops
    seen = []

    def op(logits, *args):
        tok = ops.sample_tokens(logits, *args)
        seen.append((logits.float().cpu().numpy(), [a.cpu().numpy() if hasattr(a, "cpu") else a for a in args], tok.cpu().numpy()))
        return tok

    for kw in (dict(), dict(top_k=20), dict(temperature=1.3, top_k=50, top_p=0.7)):
        _run(0, sampling=_sp(**kw), sample_op=op)
    rows = amb = 0
    for l, (T, K, P, keys, ctr), tok in seen:
        amb += R.check_tokens(l, T, K, P, keys, ctr, tok)
        rows += len(tok)
    print(f"{rows} lm_head rows checked, {amb} ambiguous")
    assert rows > 100
