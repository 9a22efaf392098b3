"""CPU suite for the Mixtral MoE path: the routing plan's numpy restatement, the export of a calibrated toy Mixtral layer into
stacked expert operands, and the MoE block through the oracle's restatement of the kernels against the simulator's
QMixtralSparseMoeBlock, stage by stage (the method of test_export_cpu.py)."""
import types

import numpy as np
import pytest
import torch

from atom_b200 import modelutils, ops
from atom_b200.qmixtral import ToyMixtralDecoderLayer
from oracle import oracle as O
from tests import moe_ref as R
from tests.test_export_cpu import _args, _check_gemm_stage, _check_quant_stage, _np, _outlier_last, _input, OUTLIERS


@pytest.mark.parametrize("t,e,k", [(1, 8, 2), (7, 4, 1), (64, 8, 2), (1000, 64, 4), (300, 8, 2), (33, 4, 4)])
def test_plan_restatement(t, e, k):
    rng = np.random.default_rng(t * 100 + e + k)
    ids = np.stack([rng.permutation(e)[:k] for _ in range(t)])
    bn = R.token_tile(t, e, k)
    assert (bn, R.tiles_max(t, e, k, bn), R.tiles_max(t, e, k, bn) * bn) == ops.moe_tiles(t, e, k)
    tmax = R.tiles_max(t, e, k, bn)
    dest, tiles = R.plan(ids, e, bn, tmax)
    flat, d = ids.reshape(-1), dest.reshape(-1)
    assert len(set(d.tolist())) == t * k and d.max() < tmax * bn              # distinct rows inside the workspace
    for x in range(e):
        rows = d[flat == x]
        assert (np.diff(rows) == 1).all()                                     # stable, contiguous per expert
        if len(rows):
            assert rows[0] % bn == 0                                          # segments start on a token tile
    live = tiles[tiles[:, 2] > 0]
    assert live[:, 2].sum() == t * k and (live[:, 1] % bn == 0).all() and (tiles[len(live):] == 0).all()
    for x, first, n, _ in live:
        assert (flat[(d >= first) & (d < first + n)] == x).all()


def test_plan_extremes():
    """Empty experts, every token on one expert (several tiles), a single token."""
    ids = np.zeros((200, 1), np.int64)
    bn = R.token_tile(200, 8, 1)
    dest, tiles = R.plan(ids, 8, bn, R.tiles_max(200, 8, 1, bn))
    assert bn == 32 and dest.reshape(-1).tolist() == list(range(200))
    assert tiles[:7, 0].tolist() == [0] * 7 and tiles[:7, 2].tolist() == [32] * 6 + [8] and (tiles[7:] == 0).all()
    dest, tiles = R.plan(np.array([[5, 2]]), 8, 16, R.tiles_max(1, 8, 2, 16))
    assert dest.tolist() == [[16, 0]] and tiles.tolist() == [[2, 0, 1, 0], [5, 16, 1, 0]]


def _build_mixtral(hidden=256, inter=256, experts=4, top_k=2, seed=0):
    torch.manual_seed(seed)
    gen = torch.Generator().manual_seed(seed)
    a = _args()
    layers = [ToyMixtralDecoderLayer(hidden, inter, heads=2, kv_heads=1, experts=experts, top_k=top_k)]
    w1_in = _outlier_last(hidden, OUTLIERS, gen)
    idx = {"layers.0.self_attn.k_proj.input": _outlier_last(hidden, OUTLIERS, gen),
           "layers.0.self_attn.o_proj.input": torch.randperm(hidden, generator=gen),
           "layers.0.block_sparse_moe.experts.0.w1.input": w1_in,
           "layers.0.block_sparse_moe.experts.0.w2.input": torch.randperm(inter, generator=gen)}
    modelutils.reorder_model_mixtral(layers, a, idx)
    modelutils.quantize_model_mixtral(layers, a)
    modelutils.add_act_quant_wrapper_mixtral(layers, a)
    return layers[0], a


def _lin(w4, w8, s4, s8, in_f):
    """A LinearInt4-shaped view of one expert's slice of the stacked operands (for the stage checks)."""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    return types.SimpleNamespace(in_features=in_f, out_features=w4.shape[0], weight_int4=t(w4), weight_int8=t(w8),
                                 scale_int4=t(s4).reshape(-1), scale_int8=t(s8), out_dtype="fp16")


def test_export_stacks_every_expert():
    from atom_b200.export import int4_mixtral_decoder_layer
    from atom_b200.mixtral import MixtralDecoderLayer
    q, _ = _build_mixtral(seed=1)
    real = int4_mixtral_decoder_layer(q, device=None, layer_idx=3)
    assert isinstance(real, MixtralDecoderLayer) and real.self_attn.layer_idx == 3
    m, moe = real.block_sparse_moe, q.block_sparse_moe
    e, i, h = 4, 256, 256
    assert m.num_experts == e and m.top_k == 2 and real.self_attn.num_kv_heads == 1 and real.self_attn.rope_theta == 1e6
    shapes = {"w13_int4": ((e, 2 * i, (h - 128) // 2), torch.uint8), "w13_int8": ((e, 2 * i, 128), torch.int8),
              "w13_scale": ((e, h // 128 - 1, 2 * i), torch.float16), "w13_keeper_scale": ((e, 2 * i), torch.float16),
              "w2_int4": ((e, h, (i - 128) // 2), torch.uint8), "w2_int8": ((e, h, 128), torch.int8),
              "w2_scale": ((e, i // 128 - 1, h), torch.float16), "w2_keeper_scale": ((e, h), torch.float16),
              "router_weight": ((e, h), torch.float16)}
    for name, (shape, dt) in shapes.items():
        t = getattr(m, name)
        assert tuple(t.shape) == shape and t.dtype == dt, name
    for x, ex in enumerate(moe.experts):
        o1, o3, o2 = ex.w1.int4_operands(), ex.w3.int4_operands(), ex.w2.int4_operands()
        for key, dst, axis in (("weight_int4", m.w13_int4, 0), ("weight_int8", m.w13_int8, 0), ("scale_int4", m.w13_scale, 1),
                               ("scale_int8", m.w13_keeper_scale, 0)):
            assert torch.equal(dst[x].narrow(axis, 0, i), o1[key]) and torch.equal(dst[x].narrow(axis, i, i), o3[key]), (x, key)
        for key, dst in (("weight_int4", m.w2_int4), ("weight_int8", m.w2_int8), ("scale_int4", m.w2_scale), ("scale_int8", m.w2_keeper_scale)):
            assert torch.equal(dst[x], o2[key]), (x, key)
    assert torch.equal(m.router_weight, moe.gate.weight.half())
    assert torch.equal(real.post_attention_layernorm.reorder_index, q.post_attention_layernorm.reorder_index.to(torch.int16))
    assert torch.equal(real.input_layernorm.reorder_index, q.input_layernorm.reorder_index.to(torch.int16))
    assert torch.equal(real.self_attn.reorder_index, q.self_attn.reorder_index.to(torch.int16))
    assert m.norm is real.post_attention_layernorm
    assert "block_sparse_moe.norm.weight" not in real.state_dict()


def normed_row_f16(x, w, idx, eps):
    """numpy restatement of the FP16 normalised row (1/sqrt in place of the GPU's rsqrtf, so within 1 FP16 ulp of it)."""
    xf = x.astype(np.float32)
    ss = (xf.astype(np.float64) ** 2).sum(-1, keepdims=True)
    rstd = (1.0 / np.sqrt(ss / x.shape[-1] + eps)).astype(np.float32)
    return ((xf[:, idx] * w.astype(np.float32)[idx]) * rstd).astype(np.float16)


def test_moe_block_oracle_chain_matches_simulator():
    q, _ = _build_mixtral(seed=2)
    real = q.to_int4(device=None)
    m, moe = real.block_sparse_moe, q.block_sparse_moe
    n = real.post_attention_layernorm
    t, e, k = 12, 4, 2
    x = _input(t, 256, 5)
    h = O.rmsnorm_fp16_i4(_np(x), _np(n.weight), _np(n.reorder_index), n.variance_epsilon)
    sim_in = q.post_attention_layernorm(x.float()[None])
    _check_quant_stage(h, _np(moe.act_quant(sim_in[0].clone())), "rmsnorm+quant")
    sim_out, sim_logits = moe(sim_in.clone())          # the simulator quantises its input in place
    sim_out = _np(sim_out[0])
    # routing: float64 logits of the FP16 normalised row; a token is kept when its k-th / (k+1)-th gap clears twice the bound
    # of the FP32 logit error plus the effect of one FP16 ulp on every y_j (this row is not the kernel's bit for bit)
    y = normed_row_f16(_np(x), _np(n.weight), _np(n.reorder_index), n.variance_epsilon)
    wr = _np(m.router_weight).astype(np.float64)
    lg = y.astype(np.float64) @ wr.T
    bound = np.stack([R.logit_error_bound(y[r], wr) + 2.0 ** -10 * (np.abs(wr) @ np.abs(y[r].astype(np.float64))) for r in range(t)])
    srt = -np.sort(-lg, axis=1)
    keep = (srt[:, k - 1] - srt[:, k]) > 2 * bound.max(1)
    assert keep.sum() >= t // 2
    np.testing.assert_allclose(lg, _np(sim_logits).astype(np.float64), atol=0.02 * np.abs(lg).max())
    out = np.zeros((t, 256), np.float16)
    g = 256 // 128 - 1
    for r in range(t):
        ids, wts = R.topk_f64(lg[r], k)
        assert not keep[r] or sorted(ids.tolist()) == sorted(torch.topk(sim_logits[r], k).indices.tolist())
        for x_id in sorted(ids.tolist()):
            w = np.float16(wts[ids.tolist().index(x_id)])
            hr = O.rmsnorm_fp16_i4(_np(x)[r:r + 1], _np(n.weight), _np(n.reorder_index), n.variance_epsilon)
            gate = O.gemm_i4_o16(hr[1], _np(m.w13_int4[x_id, :256]), hr[3], _np(m.w13_scale[x_id, :, :256]), hr[0],
                                 _np(m.w13_int8[x_id, :256]), hr[2], _np(m.w13_keeper_scale[x_id, :256]))
            up = O.gemm_i4_o16(hr[1], _np(m.w13_int4[x_id, 256:]), hr[3], _np(m.w13_scale[x_id, :, 256:]), hr[0],
                               _np(m.w13_int8[x_id, 256:]), hr[2], _np(m.w13_keeper_scale[x_id, 256:]))
            act = O.activate_fp16_i4(gate, up)
            ye = O.gemm_i4_o16(act[1], _np(m.w2_int4[x_id]), act[3], _np(m.w2_scale[x_id]).reshape(g, 256), act[0], _np(m.w2_int8[x_id]),
                               act[2], _np(m.w2_keeper_scale[x_id]))
            if r == 0:     # stage checks on the first token's experts
                hdq = _check_quant_stage(hr, _np(moe.act_quant(sim_in[0, :1].clone())), "rmsnorm+quant (row)")
                ex = moe.experts[x_id]
                _check_gemm_stage(gate, hdq, _lin(_np(m.w13_int4[x_id, :256]), _np(m.w13_int8[x_id, :256]), _np(m.w13_scale[x_id, :, :256]),
                                                  _np(m.w13_keeper_scale[x_id, :256]), 256), ex.w1, "w1")
                g32, u32 = torch.from_numpy(gate.astype(np.float32)), torch.from_numpy(up.astype(np.float32))
                adq = _check_quant_stage(act, _np(ex.act_quant(ex.act_fn(g32) * u32)), "silu*up+quant")
                _check_gemm_stage(ye, adq, _lin(_np(m.w2_int4[x_id]), _np(m.w2_int8[x_id]), _np(m.w2_scale[x_id]),
                                                _np(m.w2_keeper_scale[x_id]), 256), ex.w2, "w2")
            out[r] = (out[r] + (ye[0].astype(np.float32) * np.float32(w)).astype(np.float16)).astype(np.float16)
    d = np.abs(out[keep].astype(np.float32) - sim_out[keep]).max() / np.abs(sim_out[keep]).max()
    # quantisation noise compounding through three quantised stages of a 256-channel toy expert: 8.7 % (every stage above is
    # within one grid step of the simulator); the Llama MLP of test_z_export_gpu.py shows the same magnitude
    assert d < 0.10, d
