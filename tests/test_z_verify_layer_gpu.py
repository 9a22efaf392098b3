"""GPU suite (-m gpu): a decoder layer's verify step (BatchLenInfo(decode_len=S)), Llama and Mixtral.  Every sequence carries S
tokens; the step must write their K/V into the pages exactly as a chunked-prefill step of the same rows does (same projections,
same init_kv_i4), its attention must stay within tests/attn_verify_ref64.verify_bound over the pool the step left, and with the
verify attention's output put in place of the chunked prefill's attention the two layer outputs must be bit-identical (the rows
reach o_proj and the MLP in the same order and layout).  A CUDA graph of a verify step sized by BatchLenInfo.max_len replays bit
for bit against the eager step as the lengths grow past several RoPE table sizes."""
import numpy as np
import pytest
import torch

from tests import attn_verify_ref64 as V
from tests.test_z_attention_accuracy_gpu import _check

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _llama(heads, kv_heads, theta):
    from atom_b200.llama import LlamaConfig, LlamaDecoderLayer
    torch.manual_seed(3)
    cfg = LlamaConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=heads, num_key_value_heads=kv_heads,
                      num_hidden_layers=2, rope_theta=theta)
    return LlamaDecoderLayer(cfg, 1).to(DEV).init_random(3).eval()


def _mixtral(heads, kv_heads, theta):
    from atom_b200.mixtral import MixtralConfig, MixtralDecoderLayer
    torch.manual_seed(4)
    cfg = MixtralConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=heads, num_key_value_heads=kv_heads,
                        num_hidden_layers=2, rope_theta=theta)
    return MixtralDecoderLayer(cfg, 1).to(DEV).init_random(4).eval()


@pytest.mark.parametrize("make,heads,kv_heads,theta,S", [(_llama, 4, 2, 1e4, 4), (_llama, 4, 1, 5e5, 8), (_llama, 4, 4, 1e4, 2),
                                                         (_mixtral, 4, 2, 1e6, 3)])
def test_verify_step_writes_the_chunk_kv_and_attends_within_bound(monkeypatch, make, heads, kv_heads, theta, S):
    from atom_b200 import ops
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    layer = make(heads, kv_heads, theta)
    P, prompts = 16, [5, 30, 47]
    pools = []
    for _ in range(2):                       # one pool for the verify step, one for the chunked-prefill step of the same rows
        pool = KvPoolInt4(2, kv_heads, 128, 16, P, DEV)
        pool.buf.fill_(0xFF)
        pool.param.fill_(float("nan"))
        pools.append(pool)
    gen = torch.Generator(device=DEV).manual_seed(9)
    x0 = (torch.randn(sum(prompts), 512, device=DEV, generator=gen) * 0.5).half()
    x1 = (torch.randn(len(prompts) * S, 512, device=DEV, generator=gen) * 0.5).half()
    seen = {}
    verify = ops.batch_verify_i4

    def spy(q, kv, layer_idx, tokens_per_seq, **kw):
        o = verify(q, kv, layer_idx, tokens_per_seq, **kw)
        seen.update(q=q.cpu().numpy(), o=o.cpu().numpy(), S=tokens_per_seq, layer=layer_idx)
        return o
    monkeypatch.setattr(ops, "batch_verify_i4", spy)
    outs, tables = [], []
    with torch.inference_mode():
        for i, pool in enumerate(pools):
            seqs = [KvCacheInt4(pool, n) for n in prompts]
            layer(x0, BatchLenInfo(prompts, 0, DEV), BatchedKvCacheInt4(seqs), None)
            for c in seqs:
                c.acquire(S)
            kv = BatchedKvCacheInt4(seqs)
            tables.append((seqs, kv))
            if i == 0:
                outs.append(layer(x1, BatchLenInfo([], len(seqs), DEV, decode_len=S), None, kv))
            else:
                attn = torch.from_numpy(seen["o"]).to(DEV).view(len(seqs) * S, heads * 128)
                monkeypatch.setattr(ops, "prefill_attention_i4", lambda *a, **kw: attn)
                outs.append(layer(x1, BatchLenInfo([S] * len(seqs), 0, DEV), kv, None))
        torch.cuda.synchronize()
    assert seen and seen["S"] == S and seen["layer"] == 1
    seqs, kv = tables[0]
    assert [c.indicies for c in seqs] == [c.indicies for c in tables[1][0]]
    live = sum((c.indicies for c in seqs), [])
    a, b = (p.buf[live].cpu().numpy() for p in pools)
    assert np.array_equal(a, b), "the verify step wrote other K/V bytes than the chunked prefill"
    a, b = (p.param[live].cpu().numpy().view(np.uint16) for p in pools)
    assert np.array_equal(a, b)
    pool = pools[0]
    data, param = pool.buf.cpu().numpy(), pool.param.cpu().numpy()
    ref, bnd = V.verify_bound(seen["q"], data, param, kv.indptr.cpu().numpy(), kv.indicies.cpu().numpy(),
                              kv.last_page_offset.cpu().numpy(), 1, heads, theta, S)
    _check(seen["o"], ref, bnd, f"{make.__name__} verify step S={S}")
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), "the verify step's rows reach o_proj differently"


class _KV:
    """A page table without host lengths, as a CUDA-graph runner keeps it in static buffers."""

    def __init__(self, pool, indptr, indices, last):
        self.data, self.param = pool.buf, pool.param
        self.indptr, self.indicies, self.last_page_offset = (torch.tensor(a, dtype=torch.int32, device=DEV) for a in (indptr, indices, last))


def test_graph_of_a_verify_step_replays_as_lengths_grow_within_the_stated_bound():
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import KvPoolInt4
    S, P, bound = 4, 16, 600
    layer = _llama(4, 2, 5e5)
    pages = -(-bound // P)
    pool = KvPoolInt4(2, 2, 128, 2 * pages, P, DEV)
    gen = torch.Generator(device=DEV).manual_seed(2)
    pool.buf.random_(0, 256, generator=gen)
    pool.param[..., 0].uniform_(0.01, 0.05, generator=gen)
    pool.param[..., 1].uniform_(0.0, 0.4, generator=gen)
    own = [list(range(pages)), list(range(2 * pages - 1, pages - 1, -1))]
    kv = _KV(pool, [0, pages, 2 * pages], own[0] + own[1], [P, P])
    x = (torch.randn(2 * S, 512, device=DEV, generator=gen) * 0.5).half()

    def set_lens(lens):
        n = [-(-L // P) for L in lens]
        kv.indptr.copy_(torch.tensor([0, n[0], n[0] + n[1]], dtype=torch.int32, device=DEV))
        kv.indicies[:n[0] + n[1]].copy_(torch.tensor(own[0][:n[0]] + own[1][:n[1]], dtype=torch.int32, device=DEV))
        kv.last_page_offset.copy_(torch.tensor([(L - 1) % P + 1 for L in lens], dtype=torch.int32, device=DEV))

    blen = BatchLenInfo([], 2, DEV, decode_len=S, max_len=bound)
    with torch.inference_mode():
        with pytest.raises(RuntimeError):          # without a bound or host lengths the step cannot size its table
            layer(x, BatchLenInfo([], 2, DEV, decode_len=S), None, kv)
        set_lens([100, 40])
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            layer(x, blen, None, kv)
        torch.cuda.current_stream().wait_stream(st)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = layer(x, blen, None, kv)
        for lens in ([100, 40], [257, 130], [300, 513], [600, 577]):
            set_lens(lens)
            g.replay()
            eager = layer(x, blen, None, kv)
            torch.cuda.synchronize()
            assert torch.isfinite(eager).all()
            assert torch.equal(out.view(torch.int16), eager.view(torch.int16)), f"replay differs at lengths {lens}"
