"""GPU suite (-m gpu): grouped-query attention on the INT4 paged-KV path -- the GQA decode kernel against the CPU oracle and
against the multi-head kernel on a head-repeated cache, the fused q/k/v GEMM with unequal parts, GQA prefill attention, the
layers built on them (prefill -> decode consistency, an exported toy GQA layer), CUDA-graph capture and the error paths."""
import types

import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import gqa_oracle as GO

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


class _KV:
    def __init__(self, data, param, indptr, indices, last):
        self.data, self.param, self.indptr, self.indicies, self.last_page_offset = T(data), T(param), T(indptr), T(indices), T(last)


def _kv_fixture(rng, hkv, P, L, lens):
    pages = sum((l + P - 1) // P for l in lens) + 3
    data = rng.integers(0, 256, (pages, L, 2, hkv, P, 64), dtype=np.uint8)
    param = np.stack([rng.uniform(0.01, 0.05, (pages, L, 2, hkv, P)), rng.uniform(0, 0.4, (pages, L, 2, hkv, P))], -1).astype(np.float16)
    perm = rng.permutation(pages)
    indptr, indices, last, c = [0], [], [], 0
    for l in lens:
        npg = (l + P - 1) // P
        indices += list(perm[c:c + npg]); c += npg
        indptr.append(len(indices)); last.append((l - 1) % P + 1)
    return data, param, np.array(indptr, np.int32), np.array(indices, np.int32), np.array(last, np.int32)


def _excess(o, ref, tol=5e-4):
    o, ref = np.asarray(o, np.float32), np.asarray(ref, np.float32)
    return float((np.abs(o - ref) - tol * np.abs(ref)).max())


def _lens(P):
    # 1 token, exactly a page, one more, one short of a page, fewer pages than stripes, many pages
    return [1, P, P + 1, 2 * P - 1, 3 * P, 2048, 777]


# ------------------------------------------------------------------------------------------------ 1. decode vs the oracle
@pytest.mark.parametrize("theta", [1e4, 5e5, 1e6])
@pytest.mark.parametrize("P", [8, 16, 24, 32, 64])
@pytest.mark.parametrize("hq,hkv", [(4, 2), (8, 2), (8, 1), (64, 8)])
def test_gqa_decode_matches_oracle(hq, hkv, P, theta):
    from atom_b200 import ops
    rng = np.random.default_rng(hq * 1000 + hkv * 100 + P)
    lens = _lens(P) if hq < 64 else [1, P + 1, 2048 if P == 32 else 300]
    L, layer = 2, 1
    data, param, indptr, indices, last = _kv_fixture(rng, hkv, P, L, lens)
    q = rng.standard_normal((len(lens), hq, 128)).astype(np.float16)
    kv = _KV(data, param, indptr, indices, last)
    o = ops.batch_decode_i4(T(q), kv, layer, rope_theta=theta).cpu().numpy()
    ref = GO.batch_decode_gqa_i4(q, data, param, indptr, indices, last, layer, theta=theta)
    e = _excess(o, ref)
    assert e <= 5e-4, f"worst excess over rtol*|ref| = {e:.2e} (atol 5e-4)"


# ------------------------------------------------------------------------------------------------ 2. decode vs the MHA kernel
@pytest.mark.parametrize("hq,hkv,P", [(8, 2, 16), (8, 1, 32), (64, 8, 32), (4, 2, 8)])
def test_gqa_decode_agrees_with_mha_kernel_on_head_repeated_cache(hq, hkv, P):
    from atom_b200 import ops
    rng = np.random.default_rng(hq + hkv + P)
    lens = [1, P + 1, 500, 3 * P, 1000]
    data, param, indptr, indices, last = _kv_fixture(rng, hkv, P, 1, lens)
    q = rng.standard_normal((len(lens), hq, 128)).astype(np.float16)
    gqa = ops.batch_decode_i4(T(q), _KV(data, param, indptr, indices, last), 0).cpu().numpy()
    rd, rp = GO.repeat_heads(data, param, hq // hkv)
    mha = ops.batch_decode_i4(T(q), _KV(rd, rp, indptr, indices, last), 0).cpu().numpy()
    ref = GO.batch_decode_gqa_i4(q, data, param, indptr, indices, last, 0)
    assert _excess(gqa, mha) <= 5e-4
    assert _excess(gqa, ref) <= 5e-4 and _excess(mha, ref) <= 5e-4


# ------------------------------------------------------------------------------------------------ 3. G = 1 through the new entry
def test_gqa_entry_with_one_head_per_group_is_the_mha_kernel_bit_for_bit():
    from atom_b200 import _lib, ops
    rng = np.random.default_rng(3)
    H, P, lens = 4, 16, [1, 17, 333, 64]
    data, param, indptr, indices, last = _kv_fixture(rng, H, P, 2, lens)
    kv = _KV(data, param, indptr, indices, last)
    q = T(rng.standard_normal((len(lens), H, 128)).astype(np.float16))
    ref = ops.batch_decode_i4(q, kv, 1)
    o = torch.zeros_like(q)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.lib().atom_batch_decode_gqa_i4(o.data_ptr(), q.data_ptr(), kv.data.data_ptr(), kv.param.data_ptr(), kv.indptr.data_ptr(),
                                                   kv.indicies.data_ptr(), kv.last_page_offset.data_ptr(), 2, 1, H, H, P, len(lens), 10000.0,
                                                   st), "batch_decode_gqa_i4")
    assert torch.equal(o, ref)
    # one head per group with another base runs the eight-stripe instantiation: inside the oracle bound
    o5 = ops.batch_decode_i4(q, kv, 1, rope_theta=5e5).cpu().numpy()
    assert _excess(o5, GO.batch_decode_gqa_i4(q.cpu().numpy(), data, param, indptr, indices, last, 1, theta=5e5)) <= 5e-4


# ------------------------------------------------------------------------------------------------ 4. fused q/k/v GEMM
def _qkv_operands(m, hq, hkv, k):
    t = [O.make_gemm_inputs(m, n, k, seed=m + n + k + i) for i, n in enumerate((hq, hkv, hkv))]
    act = [T(t[0][i]) for i in (0, 2, 4, 6)]
    ws = [(x[1], x[3], x[5], x[7]) for x in t]
    cat = [np.concatenate([w[j] for w in ws], 1 if j == 1 else 0) for j in range(4)]
    return act, ws, [T(c) for c in cat]


def _three_calls(act, ws):
    from atom_b200 import ops
    q = ops.dense_layer_gemm_i4_fp16(act[0], T(ws[0][0]), act[1], T(ws[0][1]), act[2], T(ws[0][2]), act[3], T(ws[0][3]), flags=1)
    k = ops.dense_layer_gemm_i4_o4(act[0], T(ws[1][0]), act[1], T(ws[1][1]), act[2], T(ws[1][2]), act[3], T(ws[1][3]))
    v = ops.dense_layer_gemm_i4_o4(act[0], T(ws[2][0]), act[1], T(ws[2][1]), act[2], T(ws[2][2]), act[3], T(ws[2][3]))
    return q, k, v


@pytest.mark.parametrize("m", [7, 16, 48, 100])
@pytest.mark.parametrize("hq,hkv,k", [(512, 128, 512), (1024, 256, 1024), (4096, 1024, 4096), (384, 128, 512)])
def test_fused_gqa_qkv_equals_three_projections(m, hq, hkv, k):
    from atom_b200 import ops
    act, ws, (b, bs, bk, bks) = _qkv_operands(m, hq, hkv, k)
    q_ref, k_ref, v_ref = _three_calls(act, ws)
    q, (kk, ks), (vv, vs) = ops.dense_layer_gemm_i4_qkv(act[0], b, act[1], bs, act[2], bk, act[3], bks, kv_rows=hkv)
    assert q.shape == (m, hq) and kk.shape == (m, hkv // 2) and ks.shape == (m, hkv // 128 * 2)
    assert torch.equal(q, q_ref)
    assert torch.equal(kk, k_ref[0]) and torch.equal(ks, k_ref[1])
    assert torch.equal(vv, v_ref[0]) and torch.equal(vs, v_ref[1])


@pytest.mark.parametrize("m,h,k", [(16, 256, 512), (100, 512, 1024)])
def test_fused_mha_qkv_unchanged_and_equal_through_both_entries(m, h, k):
    from atom_b200 import ops
    act, ws, (b, bs, bk, bks) = _qkv_operands(m, h, h, k)
    q_ref, k_ref, v_ref = _three_calls(act, ws)
    for kv_rows in (None, h):                  # atom_gemm_i4_qkv, then atom_gemm_i4_qkv_gqa with equal parts
        q, (kk, ks), (vv, vs) = ops.dense_layer_gemm_i4_qkv(act[0], b, act[1], bs, act[2], bk, act[3], bks, kv_rows=kv_rows)
        assert torch.equal(q, q_ref) and torch.equal(kk, k_ref[0]) and torch.equal(ks, k_ref[1])
        assert torch.equal(vv, v_ref[0]) and torch.equal(vs, v_ref[1])


# ------------------------------------------------------------------------------------------------ 5. prefill
@pytest.mark.parametrize("theta", [1e4, 5e5])
@pytest.mark.parametrize("lens,hq,hkv", [([5], 4, 2), ([64, 1, 130], 8, 2), ([300, 77], 8, 1), ([2048], 4, 1)])
def test_gqa_prefill_attention_matches_the_eager_pipeline(lens, hq, hkv, theta):
    from atom_b200 import ops
    from atom_b200.llama import _dequant_o4, rotary_pos_emb
    g = torch.Generator(device="cpu").manual_seed(sum(lens) + hq + hkv)
    t = sum(lens)
    q = (torch.randn(t, hq * 128, generator=g) * 1.5).half().to(DEV)
    k4 = torch.randint(0, 256, (t, hkv * 64), dtype=torch.uint8, generator=g).to(DEV)
    v4 = torch.randint(0, 256, (t, hkv * 64), dtype=torch.uint8, generator=g).to(DEV)
    par = lambda: torch.stack((torch.rand(t, hkv, generator=g) * 0.2 + 0.05, torch.rand(t, hkv, generator=g) * 1.5), -1).half().to(DEV).view(t, hkv * 2)
    kp, vp = par(), par()
    indptr = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)
    got = ops.prefill_attention_i4(q, k4, kp, v4, vp, indptr, seqlens=lens, rope_theta=theta)
    kd, vd = _dequant_o4(k4, kp, hkv), _dequant_o4(v4, vp, hkv)
    ref, off = [], 0
    for n in lens:
        qq = q[off:off + n].view(1, n, hq, 128).transpose(1, 2)
        kk = kd[off:off + n].view(1, n, hkv, 128).transpose(1, 2).repeat_interleave(hq // hkv, dim=1)
        vv = vd[off:off + n].view(1, n, hkv, 128).transpose(1, 2).repeat_interleave(hq // hkv, dim=1)
        qq, kk = rotary_pos_emb(qq, kk, 0, theta=theta)
        o = torch.nn.functional.scaled_dot_product_attention(qq.float(), kk.float(), vv.float(), is_causal=True)
        ref.append(o.squeeze(0).transpose(0, 1).reshape(n, hq * 128))
        off += n
    ref = torch.cat(ref, 0)
    err = (got.float() - ref).abs() - 5e-3 * ref.abs()
    assert err.max().item() <= 5e-3, f"worst excess over rtol*|ref| = {err.max().item():.2e}"


# ------------------------------------------------------------------------------------------------ 6. layers
@pytest.mark.parametrize("hkv,theta", [(1, 1e4), (2, 5e5)])
def test_gqa_decoder_layer_decode_step_agrees_with_prefill_of_one_more_token(hkv, theta):
    """Prefill t tokens, decode token t+1 over the cache the prefill wrote: its attention is the last row of a prefill of all
    t+1 tokens (prefill attends the dequantised K/V it has just quantised -- the very values the decode kernel reads)."""
    from atom_b200 import ops
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    from atom_b200.llama import LlamaConfig, LlamaDecoderLayer
    dev = torch.device(DEV)
    cfg = LlamaConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_hidden_layers=1, vocab_size=128,
                      num_key_value_heads=hkv, rope_theta=theta)
    torch.manual_seed(1)
    layer = LlamaDecoderLayer(cfg, 0).to(dev).init_random(3)
    assert layer.self_attn.k_proj.out_features == hkv * 128
    t, P = 37, 16
    x = torch.randn(t + 1, 512, device=dev, dtype=torch.float16)
    pool = KvPoolInt4(1, hkv, 128, capacity=16, block_len=P, device=dev)
    cache = KvCacheInt4(pool, t)
    out_p = layer(x[:t], BatchLenInfo([t], 0, dev), BatchedKvCacheInt4([cache]), None)
    cache.acquire_one()
    kv = BatchedKvCacheInt4([cache])
    out_d = layer(x[t:], BatchLenInfo([], 1, dev), None, kv)
    assert torch.isfinite(out_p).all() and torch.isfinite(out_d).all() and out_d.shape == (1, 512)
    # the attention of token t+1, twice: the decode kernel over the cache (t prefilled tokens + the appended one) and the prefill
    # kernel over the q/k/v of all t+1 tokens.  Same quantised K/V, same RoPE base and head mapping; the prefill kernel rounds the
    # rotated K and the softmax weights to FP16 for its tensor-core products, hence its 5e-3 bound.
    at = layer.self_attn
    h = layer.input_layernorm(x)
    w4, s4, w8, s8 = at._qkv
    q, (kk, ks), (vv, vs) = ops.dense_layer_gemm_i4_qkv(h[1], w4, h[3], s4, h[0], w8, h[2], s8, kv_rows=hkv * 128)
    ip = torch.tensor([0, t + 1], dtype=torch.int32, device=dev)
    pre = ops.prefill_attention_i4(q, kk, ks, vv, vs, ip, seqlens=[t + 1], rope_theta=theta)[t].float()
    dec = ops.batch_decode_i4(q[t:].view(1, 4, 128).contiguous(), kv, 0, rope_theta=theta).view(-1).float()
    err = (dec - pre).abs() - 5e-3 * pre.abs()
    assert err.max().item() <= 5e-3, err.max().item()
    # and the cache row of token t+1 is the k the projection gave
    assert torch.equal(pool.buf[cache.indicies[t // P], 0, 0, :, t % P].reshape(-1), kk[t])


def _sim_args():
    return types.SimpleNamespace(keep_fp_for_export=True, wbits=4, abits=4, w_sym=True, a_sym=True, weight_group_size=128, act_group_size=128,
                                 weight_channel_group=2, w_clip_ratio=0.85, a_clip_ratio=1.0, keeper=128, keeper_precision=3,
                                 exponential=False, tiling=0, quant_type="int", static=False, kv_clip_ratio=1.0, reorder=False,
                                 kv_cache=True)


@pytest.mark.parametrize("hkv", [1, 2])
def test_exported_toy_gqa_layer_runs_on_the_kernels(hkv):
    """QLlamaDecoderLayer (hidden 512, 4 query heads, 1 or 2 KV heads) -> to_int4(): (a) the fused q/k/v launch on the exported
    operands gives the oracle GEMMs' bits; (b) a decode step over the cache its own prefill filled gives what the CPU oracle
    computes from that cache and that q."""
    from atom_b200 import modelutils, ops
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    from atom_b200.qllama import ToyLlamaDecoderLayer
    torch.manual_seed(hkv)
    theta = 5e5
    toy = ToyLlamaDecoderLayer(512, 1024, 4, kv_heads=hkv)
    toy.self_attn.rope_theta = theta
    layers, a = [toy], _sim_args()
    modelutils.quantize_model_llama(layers, a)
    modelutils.add_act_quant_wrapper_llama(layers, a)
    real = layers[0].to_int4(DEV)
    at = real.self_attn
    assert (at.num_heads, at.num_kv_heads, at.rope_theta) == (4, hkv, theta)
    dev = torch.device(DEV)
    t = 21
    x = (torch.randn(t + 1, 512) * 0.5).half().to(dev)
    # (a) q/k/v on the kernels vs the oracle GEMMs on the same quantised activation bytes
    h = real.input_layernorm(x)
    w4, s4, w8, s8 = at.fuse()._qkv
    q, (kk, ks), (vv, vs) = ops.dense_layer_gemm_i4_qkv(h[1], w4, h[3], s4, h[0], w8, h[2], s8, kv_rows=hkv * 128)
    hn = [h[1].cpu().numpy().view(np.uint8), np.nan_to_num(h[3].cpu().numpy()), h[0].cpu().numpy(), np.nan_to_num(h[2].cpu().numpy())]

    def oracle(lin, f):
        g, n = lin.in_features // 128 - 1, lin.out_features
        bsc = lin.scale_int4.detach().cpu().numpy().reshape(-1)[: g * n].reshape(g, n)
        return f(hn[0], lin.weight_int4.detach().cpu().numpy(), hn[1], bsc, hn[2], lin.weight_int8.detach().cpu().numpy(), hn[3],
                 lin.scale_int8.detach().cpu().numpy()[:n])
    assert np.array_equal(q.cpu().numpy().view(np.uint16), oracle(at.q_proj, O.gemm_i4_o16).view(np.uint16))
    for (d, s), lin in (((kk, ks), at.k_proj), ((vv, vs), at.v_proj)):
        rd, rs = oracle(lin, O.gemm_i4_o4)
        assert np.array_equal(d.cpu().numpy(), rd) and np.array_equal(s.cpu().numpy().view(np.uint16), rs.view(np.uint16))
    # (b) prefill t tokens through the exported layer, then one decode step
    pool = KvPoolInt4(1, hkv, 128, capacity=8, block_len=16, device=dev)
    cache = KvCacheInt4(pool, t)
    real(x[:t], BatchLenInfo([t], 0, dev), BatchedKvCacheInt4([cache]), None)
    cache.acquire_one()
    kv = BatchedKvCacheInt4([cache])
    out = real(x[t:], BatchLenInfo([], 1, dev), None, kv)
    assert torch.isfinite(out).all()
    qd = q[t:].view(1, 4, 128).contiguous()
    got = ops.batch_decode_i4(qd, kv, 0, rope_theta=theta).cpu().numpy()
    ref = GO.batch_decode_gqa_i4(qd.cpu().numpy(), pool.buf.cpu().numpy(), pool.param.cpu().numpy(), kv.indptr.cpu().numpy(),
                                 kv.indicies.cpu().numpy(), kv.last_page_offset.cpu().numpy(), 0, theta=theta)
    assert _excess(got, ref) <= 5e-4
    # the cache row of the decoded token is the k the fused launch produced for it
    page, entry = cache.indicies[t // 16], t % 16
    assert torch.equal(pool.buf[page, 0, 0, :, entry].reshape(-1), kk[t])


# ------------------------------------------------------------------------------------------------ 7. CUDA graphs
def test_gqa_entry_points_are_graph_capturable():
    from atom_b200 import _lib, ops
    rng = np.random.default_rng(11)
    hq, hkv, P, lens = 8, 2, 16, [33, 7, 100]
    data, param, indptr, indices, last = _kv_fixture(rng, hkv, P, 1, lens)
    kv = _KV(data, param, indptr, indices, last)
    q = T(rng.standard_normal((3, hq, 128)).astype(np.float16))
    act, ws, (b, bs, bk, bks) = _qkv_operands(16, hq * 128, hkv * 128, 512)
    g = torch.Generator(device="cpu").manual_seed(0)
    t, pl = 70, [50, 20]
    pq = torch.randn(t, hq * 128, generator=g).half().to(DEV)
    k4 = torch.randint(0, 256, (t, hkv * 64), dtype=torch.uint8, generator=g).to(DEV)
    kp = (torch.rand(t, hkv * 2, generator=g) * 0.2 + 0.05).half().to(DEV)
    ip = torch.tensor([0, 50, 70], dtype=torch.int32, device=DEV)

    # the Python wrapper of the prefill attention builds its position vector on the host, so the C entry point is captured directly
    vp = (torch.rand(t, hkv * 2, generator=g) * 0.2 + 0.05).half().to(DEV)
    v4 = torch.randint(0, 256, (t, hkv * 64), dtype=torch.uint8, generator=g).to(DEV)
    pos = torch.cat([torch.arange(n, dtype=torch.int32) for n in pl]).to(DEV)
    table = ops.rope_table(max(pl), torch.device(DEV), 1e6)
    kf, vf = torch.empty(t, hkv * 128, dtype=torch.float16, device=DEV), torch.empty(t, hkv * 128, dtype=torch.float16, device=DEV)
    p_ref = ops.prefill_attention_i4(pq, k4, kp, v4, vp, ip, seqlens=pl, rope_theta=1e6)

    def run():
        d = ops.batch_decode_i4(q, kv, 0, rope_theta=1e6)
        qq, (kk, ks), (vv, vs) = ops.dense_layer_gemm_i4_qkv(act[0], b, act[1], bs, act[2], bk, act[3], bks, kv_rows=hkv * 128)
        p = torch.empty_like(pq)
        _lib.check(_lib.lib().atom_prefill_attention_gqa_i4(pq.data_ptr(), k4.data_ptr(), kp.data_ptr(), v4.data_ptr(), vp.data_ptr(),
                                                            ip.data_ptr(), pos.data_ptr(), table.data_ptr(), kf.data_ptr(), vf.data_ptr(),
                                                            p.data_ptr(), t, len(pl), max(pl), hq, hkv,
                                                            torch.cuda.current_stream().cuda_stream), "prefill_attention_gqa_i4")
        return d, qq, kk, ks, vv, vs, p
    eager = [x.clone() for x in run()]
    assert torch.equal(eager[-1], p_ref)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        run()
        st.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=st):
            outs = run()
        gr.replay(); st.synchronize()
    for a, e in zip(outs, eager):
        assert torch.equal(a, e)


def test_textgen_cli_serves_llama3_8b_shape_with_graphed_decode_steps():
    """tools/bench_textgen.py on the llama3-8b configuration (32 query / 8 KV heads, base 5e5), two layers: the pool holds KV
    heads and decode-only steps replay from CUDA graphs."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "tools", "bench_textgen.py"), "--model", "llama3-8b", "--layers", "2",
                          "--batch-size", "4", "--num-batches", "2", "--maxlen", "96", "--warmup-batches", "0"],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    rep = json.loads(out.stdout.strip().splitlines()[-1])
    assert rep["model"] == "llama3-8b" and rep["num_requests"] == 8 and rep["graphed_decode_steps"] > 0
    assert rep["total_new_tokens"] > 0 and rep["throughput_tokens_per_s"] > 0


# ------------------------------------------------------------------------------------------------ 8. errors
def test_gqa_errors_are_loud():
    from atom_b200 import ops
    rng = np.random.default_rng(0)
    data, param, indptr, indices, last = _kv_fixture(rng, 2, 16, 1, [5])
    kv = _KV(data, param, indptr, indices, last)
    with pytest.raises(RuntimeError, match="multiple of num_kv_heads"):
        ops.batch_decode_i4(torch.zeros(1, 5, 128, dtype=torch.float16, device=DEV), kv, 0)
    with pytest.raises(RuntimeError, match="supported group sizes are 1, 2, 4 and 8"):
        ops.batch_decode_i4(torch.zeros(1, 6, 128, dtype=torch.float16, device=DEV), kv, 0)
    with pytest.raises(RuntimeError, match="rope_theta"):
        ops.batch_decode_i4(torch.zeros(1, 4, 128, dtype=torch.float16, device=DEV), kv, 0, rope_theta=0.5)
    t = 4
    q = torch.zeros(t, 4 * 128, dtype=torch.float16, device=DEV)
    k3 = torch.zeros(t, 3 * 64, dtype=torch.uint8, device=DEV)
    p3 = torch.zeros(t, 3 * 2, dtype=torch.float16, device=DEV)
    ip = torch.tensor([0, t], dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="multiple of num_kv_heads"):          # 4 query heads over 3 KV heads
        ops.prefill_attention_i4(q, k3, p3, k3, p3, ip, seqlens=[t])
    k2 = torch.zeros(t, 2 * 64, dtype=torch.uint8, device=DEV)
    with pytest.raises(RuntimeError, match="shape mismatch"):                    # v has another head count than k
        ops.prefill_attention_i4(q, k2, p3[:, :4].contiguous(), k3, p3, ip, seqlens=[t])
    act, ws, (b, bs, bk, bks) = _qkv_operands(8, 512, 128, 512)
    with pytest.raises(RuntimeError, match="multiples of 128"):
        ops.dense_layer_gemm_i4_qkv(act[0], b, act[1], bs, act[2], bk, act[3], bks, kv_rows=64)
    act, ws, (b, bs, bk, bks) = _qkv_operands(8, 384, 256, 512)                  # 3 query heads over 2 KV heads
    with pytest.raises(RuntimeError, match="whole query heads per KV head"):
        ops.dense_layer_gemm_i4_qkv(act[0], b, act[1], bs, act[2], bk, act[3], bks, kv_rows=256)
