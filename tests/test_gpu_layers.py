"""GPU suite (-m gpu): the operator surfaces built on the kernels -- QLinearLayer.pack() + real-INT4 forward, the
LlamaDecoderLayer mirror (prefill writes the cache that decode reads), and the CUDA-graph capturability of a decode step."""
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _args():
    return types.SimpleNamespace(keep_fp_for_export=True, wbits=4, abits=4, w_sym=True, a_sym=True, weight_group_size=128, act_group_size=128,
                                 weight_channel_group=2, w_clip_ratio=0.85, a_clip_ratio=0.9, keeper=128, keeper_precision=3,
                                 exponential=False, tiling=0, quant_type="int", static=False, kv_clip_ratio=1.0, reorder=True)


def test_qlinear_pack_forward_matches_oracle_and_fakequant():
    from atom_b200.qlinear import QLinearLayer
    from oracle import oracle as O
    torch.manual_seed(0)
    lin = torch.nn.Linear(1024, 256, bias=False)
    q = QLinearLayer(lin, _args())
    q.quant()
    wq = q.weight.clone()
    q.pack(device="cuda:0")
    x = torch.randn(9, 1024)
    x[:, -128:] *= 8            # outlier channels, already "reordered" to the end
    y = q(x.cuda().half()).float().cpu()
    # (1) exact vs the oracle on the very same quantised operands
    o8, o4, s8, s4 = O.reorder_fp16_i4(x.half().numpy(), np.arange(1024, dtype=np.int16))
    ref = O.gemm_i4_o16(o4, q.weight_int4.cpu().numpy(), s4, q.scale_int4.cpu().numpy(), o8, q.weight_int8.cpu().numpy(), s8,
                        q.scale_int8.cpu().numpy())
    assert np.array_equal(y.half().numpy().view(np.uint16), ref.view(np.uint16))
    # (2) close to the simulator's F.linear on fake-quantised weights (activation quantisation differs: the kernels do
    #     not clip, the simulator clips at 0.9) -- a few percent of the output scale
    y_sim = torch.nn.functional.linear(x, wq)
    assert (y - y_sim).abs().max() < 0.08 * y_sim.abs().max()


def _small_cfg():
    from atom_b200.llama import LlamaConfig
    return LlamaConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_hidden_layers=1, vocab_size=128)


def test_decoder_layer_prefill_then_decode_consistent():
    """Prefill L tokens (SDPA on the dequantised K/V it just wrote), then decode token L+1 with the INT4-KV kernel:
    the decode kernel must see exactly the cache the prefill wrote (positions, RoPE convention, page table)."""
    from atom_b200 import ops
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    from atom_b200.llama import LlamaDecoderLayer, _dequant_o4, rotary_pos_emb
    dev = torch.device("cuda:0")
    cfg = _small_cfg()
    torch.manual_seed(1)
    layer = LlamaDecoderLayer(cfg, 0).to(dev).init_random(3)
    pool = KvPoolInt4(1, 4, 128, capacity=16, block_len=16, device=dev)
    L = 21
    cache = KvCacheInt4(pool, L)
    x = torch.randn(L, 512, device=dev, dtype=torch.float16)
    out_p = layer(x, BatchLenInfo([L], 0, dev), BatchedKvCacheInt4([cache]), None)
    assert torch.isfinite(out_p).all() and out_p.shape == (L, 512)
    cache.acquire_one()
    xd = torch.randn(1, 512, device=dev, dtype=torch.float16)
    kv = BatchedKvCacheInt4([cache])
    out_d = layer(xd, BatchLenInfo([], 1, dev), None, kv)
    assert torch.isfinite(out_d).all() and out_d.shape == (1, 512)
    # reference for the decode attention: dequantise the whole cache and run causal SDPA for the last position
    h = layer.input_layernorm(xd)
    q = layer.self_attn.q_proj(h).view(1, 4, 128)
    data, param = pool.buf, pool.param
    idx = torch.tensor(cache.indicies, device=dev)
    kd = data[idx, 0, 0].permute(1, 0, 2, 3).reshape(4, -1, 64)[:, :L + 1]
    vd = data[idx, 0, 1].permute(1, 0, 2, 3).reshape(4, -1, 64)[:, :L + 1]
    kp = param[idx, 0, 0].permute(1, 0, 2, 3).reshape(4, -1, 2)[:, :L + 1].float()
    vp = param[idx, 0, 1].permute(1, 0, 2, 3).reshape(4, -1, 2)[:, :L + 1].float()
    un = lambda d: torch.stack(((d & 0xF).float(), (d >> 4).float()), -1).reshape(4, L + 1, 128)
    K = un(kd) * kp[..., :1] - kp[..., 1:]
    V = un(vd) * vp[..., :1] - vp[..., 1:]
    qq, _ = rotary_pos_emb(q.transpose(0, 1)[None].float(), q.transpose(0, 1)[None].float(), L)
    _, KK = rotary_pos_emb(K[None], K[None], 0)
    s = (qq[0] @ KK[0].transpose(1, 2)) / np.sqrt(128.0)
    ref = (torch.softmax(s, -1) @ V)[:, 0]                       # [heads, 128]
    got = ops.batch_decode_i4(q.contiguous(), kv, 0)[0].float()
    assert torch.allclose(got, ref, rtol=2e-3, atol=2e-3)


def test_decode_step_is_cuda_graph_capturable():
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    from atom_b200.llama import LlamaDecoderLayer
    dev = torch.device("cuda:0")
    cfg = _small_cfg()
    layer = LlamaDecoderLayer(cfg, 0).to(dev).init_random(5)
    pool = KvPoolInt4(1, 4, 128, capacity=32, block_len=16, device=dev)
    pool.buf.random_(0, 256); pool.param.uniform_(0.01, 0.05)
    caches = [KvCacheInt4(pool, n) for n in (33, 7, 100)]
    for c in caches:
        c.acquire_one()
    kv = BatchedKvCacheInt4(caches)
    blen = BatchLenInfo([], 3, dev)
    x = torch.randn(3, 512, device=dev, dtype=torch.float16)
    eager = layer(x, blen, None, kv).clone()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        layer(x, blen, None, kv)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            y = layer(x, blen, None, kv)
        g.replay(); st.synchronize()
    assert torch.equal(y, eager)


@pytest.mark.parametrize("lens,heads", [([5], 2), ([64, 1, 130], 4), ([300, 77], 3), ([2048], 2)])
def test_prefill_attention_matches_the_eager_dequant_rope_sdpa_path(lens, heads):
    """EXTENSION op (SURVEY.md 8 f3): one-launch causal prefill attention over the just-quantised K/V vs the eager pipeline
    round 1 shipped (torch dequantisation, rotary_pos_emb of llama.py:18-32, scaled_dot_product_attention per prompt)."""
    from atom_b200 import ops
    from atom_b200.llama import _dequant_o4, rotary_pos_emb
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(sum(lens) + heads)
    t = sum(lens)
    q = (torch.randn(t, heads * 128, generator=g) * 1.5).half().to(dev)
    k4 = torch.randint(0, 256, (t, heads * 64), dtype=torch.uint8, generator=g).to(dev)
    v4 = torch.randint(0, 256, (t, heads * 64), dtype=torch.uint8, generator=g).to(dev)
    kp = torch.stack((torch.rand(t, heads, generator=g) * 0.2 + 0.05, torch.rand(t, heads, generator=g) * 1.5), -1).half().to(dev).view(t, heads * 2)
    vp = torch.stack((torch.rand(t, heads, generator=g) * 0.2 + 0.05, torch.rand(t, heads, generator=g) * 1.5), -1).half().to(dev).view(t, heads * 2)
    indptr = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=dev)
    got = ops.prefill_attention_i4(q, k4, kp, v4, vp, indptr, seqlens=lens)
    # the multi-head C entry point, called directly, gives the operator's bits
    from atom_b200 import _lib
    pos = torch.cat([torch.arange(n, dtype=torch.int32) for n in lens]).to(dev)
    table = ops.rope_table(max(lens), dev)
    kf, vf, direct = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
    _lib.check(_lib.lib().atom_prefill_attention_i4(q.data_ptr(), k4.data_ptr(), kp.data_ptr(), v4.data_ptr(), vp.data_ptr(),
                                                    indptr.data_ptr(), pos.data_ptr(), table.data_ptr(), kf.data_ptr(), vf.data_ptr(),
                                                    direct.data_ptr(), t, len(lens), max(lens), heads,
                                                    torch.cuda.current_stream().cuda_stream), "prefill_attention_i4")
    assert torch.equal(direct, got)
    kd, vd = _dequant_o4(k4, kp, heads), _dequant_o4(v4, vp, heads)
    ref, off = [], 0
    for n in lens:
        qq = q[off:off + n].view(1, n, heads, 128).transpose(1, 2)
        kk = kd[off:off + n].view(1, n, heads, 128).transpose(1, 2)
        vv = vd[off:off + n].view(1, n, heads, 128).transpose(1, 2)
        qq, kk = rotary_pos_emb(qq, kk, 0)
        o = torch.nn.functional.scaled_dot_product_attention(qq.float(), kk.float(), vv.float(), is_causal=True)
        ref.append(o.squeeze(0).transpose(0, 1).reshape(n, heads * 128))
        off += n
    ref = torch.cat(ref, 0)
    err = (got.float() - ref).abs() - 5e-3 * ref.abs()
    assert err.max().item() <= 5e-3, f"worst excess over rtol*|ref| = {err.max().item():.2e}"
