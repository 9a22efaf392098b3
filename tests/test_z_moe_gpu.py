"""GPU suite (-m gpu) of the Mixtral MoE block (csrc/moe_kernels.cuh and the grouped mode of the GEMM): routing against a float64
top-k inside a bound derived from the kernel's arithmetic, plan and gather against the numpy restatement, the grouped GEMMs and
the whole block bit for bit against the unfused composition of existing operators, CUDA-graph replay with different routings,
and an exported Mixtral layer against the oracle chain and the simulator."""
import math

import numpy as np
import pytest
import torch

from atom_b200 import _lib, ops
from atom_b200.llama import LlamaRMSNormInt4
from atom_b200.mixtral import MixtralConfig, MixtralDecoderLayer, SparseMoeInt4
from tests import moe_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NS = ops.GEMM_NO_SPLITK


def _sidx(rows):
    return torch.tensor([(r // 16) * 64 + (r % 8) * 8 + ((r // 8) % 2) for r in rows], dtype=torch.long, device=DEV)


def _bits(t):
    return t.contiguous().view(torch.int16) if t.dtype == torch.float16 else t.contiguous().view(torch.uint8)


def _rows_equal(tup, rows, ref, what):
    """Rows `rows` of the activation tuple `tup` (layout of its own row count) == rows 0.. of `ref`, scales included."""
    rows = list(rows)
    r = torch.tensor(rows, dtype=torch.long, device=DEV)
    assert torch.equal(_bits(tup[0][r]), _bits(ref[0])), what + " keeper"
    assert torch.equal(_bits(tup[1][r]), _bits(ref[1])), what + " int4"
    src, dst = _sidx(rows), _sidx(range(len(rows)))
    for j in range(4):
        assert torch.equal(_bits(tup[2][src + 2 * j]), _bits(ref[2][dst])), what + " keeper scale"
        assert torch.equal(_bits(tup[3][:, src + 2 * j]), _bits(ref[3][:, dst])), what + " scales"


@torch.no_grad()
def _moe(h, inter, e, k, seed=0):
    norm = LlamaRMSNormInt4(h, eps=1e-5).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    norm.weight.copy_(1 + 0.1 * torch.randn(h, device=DEV, generator=g))
    norm.reorder_index.copy_(torch.randperm(h, device=DEV, generator=g).to(torch.int16))
    cfg = MixtralConfig(hidden_size=h, intermediate_size=inter, num_local_experts=e, num_experts_per_tok=k)
    return SparseMoeInt4(cfg, norm).to(DEV).init_random(seed)


# ------------------------------------------------------------------------------------------------ route
@pytest.mark.parametrize("e", [4, 8, 64])
@pytest.mark.parametrize("k", [1, 2, 4])
@pytest.mark.parametrize("t", [1, 7, 64, 1000])
def test_route_matches_float64_topk(e, k, t):
    h = 512 if t < 1000 else 4096
    g = torch.Generator(device=DEV).manual_seed(e * 1000 + k * 100 + t)
    x = (torch.randn(t, h, device=DEV, generator=g) * 2).half()
    nw = (1 + 0.1 * torch.randn(h, device=DEV, generator=g)).half()
    idx = torch.randperm(h, device=DEV, generator=g).to(torch.int16)
    wr = (torch.randn(e, h, device=DEV, generator=g) / math.sqrt(h)).half()
    ids, w, lg, yn = ops.moe_route_f16(x, nw, idx, 1e-5, wr, k, router_logits=True, normed=True)
    # the normalised row is the one rmsnorm_fp16_i4 quantises: quantising it again (identity order) gives the same tuple
    a, b = ops.rmsnorm_fp16_i4(x, nw, idx, 1e-5), ops.reorder_fp16_i4(yn, torch.arange(h, device=DEV, dtype=torch.int16))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(_bits(a[2][_sidx(range(t))]), _bits(b[2][_sidx(range(t))]))
    y, wrn = yn.double().cpu().numpy(), wr.double().cpu().numpy()
    lg64 = y @ wrn.T
    bound = np.stack([R.logit_error_bound(y[r], wrn) for r in range(t)])
    assert (np.abs(lg.double().cpu().numpy() - lg64) <= bound).all()
    ids, w = ids.cpu().numpy(), w.float().cpu().numpy()
    srt = -np.sort(-lg64, axis=1)
    gap = srt[:, k - 1] - srt[:, k] if k < e else np.full(t, np.inf)
    ok = gap > 2 * bound.max(1)
    assert ok.mean() > 0.9
    for r in np.nonzero(ok)[0]:
        ref_ids, _ = R.topk_f64(lg64[r], k)
        assert sorted(ids[r].tolist()) == sorted(ref_ids.tolist()), r
        p = np.exp(lg64[r] - lg64[r].max())
        w64 = p[ids[r]] / p[ids[r]].sum()
        ulp = 2.0 ** (np.floor(np.log2(np.maximum(w64, 2.0 ** -14))) - 10)
        assert (np.abs(w[r] - w64) <= ulp).all(), (r, w[r], w64)


def test_route_ties_go_to_the_lower_expert():
    h, e, t = 512, 8, 256
    g = torch.Generator(device=DEV).manual_seed(5)
    x = (torch.randn(t, h, device=DEV, generator=g) * 2).half()
    nw = torch.ones(h, device=DEV, dtype=torch.float16)
    idx = torch.arange(h, device=DEV, dtype=torch.int16)
    wr = (torch.randn(e, h, device=DEV, generator=g) / math.sqrt(h)).half()
    wr[2] *= 4
    wr[6] = wr[2]                  # 2 and 6 always tie, and lead for many tokens
    wr[7] = wr[3]
    for k in (1, 2, 3):
        ids, w, lg = ops.moe_route_f16(x, nw, idx, 1e-5, wr, k, router_logits=True)
        assert torch.equal(lg[:, 2], lg[:, 6]) and torch.equal(lg[:, 3], lg[:, 7])
        ids = ids.cpu().tolist()
        hits = 0
        for row in ids:
            for lo, hi in ((2, 6), (3, 7)):
                if hi in row:
                    assert lo in row and row.index(lo) < row.index(hi), row
                    hits += 1
        lead = sum(1 for row in ids if row[0] == 2)
        assert lead > t // 4 and (k == 1 or hits > t // 4)
        if k == 1:
            assert all(row[0] != 6 for row in ids)


# ------------------------------------------------------------------------------------------------ plan + gather
def _ids(kind, t, e, k, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "one":
        return np.zeros((t, 1), np.int32) + 3
    if kind == "empty":                                 # experts 0, 2-5, 7 get nothing
        return np.stack([rng.permutation([1, 6])[:k] for _ in range(t)]).astype(np.int32)
    if kind == "skew":                                  # 70 % of the first choices on expert 0
        out = []
        for _ in range(t):
            first = 0 if rng.random() < 0.7 else int(rng.integers(1, e))
            rest = [x for x in rng.permutation(e) if x != first][:k - 1]
            out.append([first] + rest)
        return np.array(out, np.int32)
    return np.stack([rng.permutation(e)[:k] for _ in range(t)]).astype(np.int32)


@pytest.mark.parametrize("kind,t,e,k", [("random", 300, 8, 2), ("empty", 40, 8, 2), ("one", 150, 8, 1), ("random", 1, 8, 2),
                                        ("random", 1000, 64, 4)])
def test_plan_and_gather(kind, t, e, k):
    h = 512
    ids_np = _ids(kind, t, e, k)
    ids = torch.from_numpy(ids_np).to(DEV)
    bn, tmax, rows_cap = ops.moe_tiles(t, e, k)
    dest, tiles = ops.moe_plan(ids, e)
    rd, rt = R.plan(ids_np, e, bn, tmax)
    assert np.array_equal(dest.cpu().numpy(), rd) and np.array_equal(tiles.cpu().numpy(), rt)
    if kind == "one":
        assert (rt[:, 2] > 0).sum() > 2 and rt[0, 0] == 3
    x = ops.reorder_fp16_i4((torch.randn(t, h, device=DEV) * 3).half(), torch.randperm(h, device=DEV).to(torch.int16))
    ws = ops._quant_outputs(rows_cap, h, DEV)
    for a in ws:
        a.view(torch.uint8).fill_(0xFF)
    xp = ops.moe_gather_i4(x, dest, rows_cap, out=ws)
    slots = rd.reshape(-1)
    tok = np.repeat(np.arange(t), k)
    tt = torch.from_numpy(tok).to(DEV)
    _rows_equal(xp, slots.tolist(), (x[0][tt], x[1][tt], *_scales_of(x, tok.tolist())), kind)
    pad = sorted(set(range(rows_cap)) - set(slots.tolist()))
    if pad:
        p = torch.tensor(pad, device=DEV)
        assert (xp[0][p].view(torch.uint8) == 0xFF).all() and (xp[1][p].view(torch.uint8) == 0xFF).all()


def _scales_of(x, tok):
    """The scales of tokens `tok` of tuple x, re-laid out as a tuple of len(tok) rows (replicated x4)."""
    n = len(tok)
    s8 = torch.zeros(ops.scale_size(n), dtype=torch.float16, device=DEV)
    s4 = torch.zeros((x[3].size(0), ops.scale_size(n)), dtype=torch.float16, device=DEV)
    src, dst = _sidx(list(tok)), _sidx(range(n))
    for j in range(4):
        s8[dst + 2 * j] = x[2][src]
        s4[:, dst + 2 * j] = x[3][:, src]
    return s8, s4


# ------------------------------------------------------------------------------------------------ grouped GEMMs
def _expert_ref(moe, x_e, e):
    """Per-expert operator calls, un-split: gate and up (o16), activate, down."""
    i = moe.intermediate_size
    sl = lambda w4, w8, s4, s8, a, b: (w4[e, a:b], w8[e, a:b], s4[e][:, a:b].contiguous(), s8[e, a:b])  # noqa: E731
    def gemm(x, w4, w8, s4, s8):
        return ops.dense_layer_gemm_i4_fp16(x[1].view(torch.uint8), w4, x[3], s4, x[0], w8, x[2], s8, flags=NS)
    gate = gemm(x_e, *sl(moe.w13_int4, moe.w13_int8, moe.w13_scale, moe.w13_keeper_scale, 0, i))
    up = gemm(x_e, *sl(moe.w13_int4, moe.w13_int8, moe.w13_scale, moe.w13_keeper_scale, i, 2 * i))
    act = ops.activate_fp16_i4(gate, up)
    return act, gemm(act, moe.w2_int4[e], moe.w2_int8[e], moe.w2_scale[e], moe.w2_keeper_scale[e])


_TOY, _MIX = (512, 1024, 4, 2), (4096, 14336, 8, 2)
_moes = {}


def _cached_moe(shape):
    if shape not in _moes:
        _moes.clear()
        _moes[shape] = _moe(*shape, seed=1)
    return _moes[shape]


@pytest.mark.parametrize("shape", [_TOY, _MIX], ids=["toy", "mixtral8x7b"])
@pytest.mark.parametrize("t,kind", [(1, "random"), (5, "random"), (16, "random"), (33, "random"), (64, "random"), (300, "random"),
                                    (2048, "random"), (64, "skew"), (300, "skew")])
def test_grouped_gemms_equal_per_expert_calls(shape, t, kind):
    h, inter, e, k = shape
    moe = _cached_moe(shape)
    ids_np = _ids(kind, t, e, k, seed=t)
    ids = torch.from_numpy(ids_np).to(DEV)
    xr = (torch.randn(t, h, device=DEV) * 2).half()
    idx = moe.norm.reorder_index
    x = ops.reorder_fp16_i4(xr, idx)
    bn, tmax, rows_cap = ops.moe_tiles(t, e, k)
    dest, tiles = ops.moe_plan(ids, e)
    results = []
    for fill in (0x00, 0xFF):          # pad rows of the workspace must not change a single stored bit
        ws = ops._quant_outputs(rows_cap, h, DEV)
        for a in ws:
            a.view(torch.uint8).fill_(fill)
        xp = ops.moe_gather_i4(x, dest, rows_cap, out=ws)
        act = ops.dense_layer_gemm_i4_gateup_act_grouped(xp, moe.w13_int4, moe.w13_scale, moe.w13_int8, moe.w13_keeper_scale, tiles, bn)
        y = ops.dense_layer_gemm_i4_fp16_grouped(act, moe.w2_int4, moe.w2_scale, moe.w2_int8, moe.w2_keeper_scale, tiles, bn)
        results.append((act, y))
    d = dest.cpu().numpy()
    live = sorted(d.reshape(-1).tolist())
    lr = torch.tensor(live, device=DEV)
    (act0, y0), (act1, y1) = results
    assert torch.equal(_bits(y0[lr]), _bits(y1[lr]))
    assert torch.equal(act0[0][lr], act1[0][lr]) and torch.equal(act0[1][lr], act1[1][lr])
    for ex in range(e):
        tok, slot = np.nonzero(ids_np == ex)
        if len(tok) == 0:
            continue
        x_e = ops.reorder_fp16_i4(xr[torch.from_numpy(tok).to(DEV)], idx)
        act_e, y_e = _expert_ref(moe, x_e, ex)
        rows = d[tok, slot].tolist()
        _rows_equal(act0, rows, act_e, f"expert {ex} gate/up+act")
        assert torch.equal(_bits(y0[torch.tensor(rows, device=DEV)]), _bits(y_e)), f"expert {ex} down"


def test_grouped_o16_matches_oracle():
    from oracle import oracle as O
    h, inter, e, k = _TOY
    moe = _cached_moe(_TOY)
    t = 9
    ids_np = _ids("random", t, e, k, seed=3)
    x = ops.reorder_fp16_i4((torch.randn(t, h, device=DEV) * 2).half(), moe.norm.reorder_index)
    bn, tmax, rows_cap = ops.moe_tiles(t, e, k)
    dest, tiles = ops.moe_plan(torch.from_numpy(ids_np).to(DEV), e)
    xp = ops.moe_gather_i4(x, dest, rows_cap)
    y = ops.dense_layer_gemm_i4_fp16_grouped(xp, moe.w13_int4, moe.w13_scale, moe.w13_int8, moe.w13_keeper_scale, tiles, bn)
    n = lambda a: a.cpu().numpy()  # noqa: E731
    d = dest.cpu().numpy()
    for ex in range(e):
        tok, slot = np.nonzero(ids_np == ex)
        if len(tok) == 0:
            continue
        xe = [n(a) for a in x]
        rows = tok.tolist()
        s8, s4 = _scales_of(x, rows)
        ref = O.gemm_i4_o16(xe[1][rows], n(moe.w13_int4[ex]), np.nan_to_num(n(s4)), n(moe.w13_scale[ex]), xe[0][rows],
                            n(moe.w13_int8[ex]), np.nan_to_num(n(s8)), n(moe.w13_keeper_scale[ex]))
        got = n(y[torch.tensor(d[tok, slot].tolist(), device=DEV)])
        assert np.array_equal(got.view(np.uint16), ref.view(np.uint16)), ex


# ------------------------------------------------------------------------------------------------ combine
def test_combine_equals_index_add_loop_with_signed_zeros():
    t, h, e, k = 50, 256, 8, 2
    ids_np = _ids("random", t, e, k, seed=9)
    ids = torch.from_numpy(ids_np).to(DEV)
    bn, tmax, rows_cap = ops.moe_tiles(t, e, k)
    dest, tiles = ops.moe_plan(ids, e)
    y = (torch.randn(rows_cap, h, device=DEV) * 4).half()
    y[:, :16] = -0.0                                  # -0.0 products: the sum from +0.0 stays +0.0
    y[::3, 16:32] = 0.0
    w = torch.rand(t, k, device=DEV).half()
    w[::5, 0] = -0.0
    out = ops.moe_combine_f16(y, ids, w, dest)
    ref = torch.zeros(t, h, device=DEV, dtype=torch.float16)
    d = dest.cpu().numpy()
    for ex in range(e):
        tok, slot = np.nonzero(ids_np == ex)
        if len(tok) == 0:
            continue
        tt, ss = torch.from_numpy(tok).to(DEV), torch.from_numpy(slot).to(DEV)
        ref.index_add_(0, tt, (y[torch.from_numpy(d[tok, slot]).to(DEV)] * w[tt, ss, None]).half())
    assert torch.equal(_bits(out), _bits(ref))
    assert (_bits(out[:, :16]) == 0).all()            # +0.0, not -0.0


# ------------------------------------------------------------------------------------------------ the block
def _unfused(moe, hs):
    """Reference of the expert path: the route kernel's own routing, then existing operators expert by expert."""
    ids, w = moe.route(hs)
    n = moe.norm
    out = torch.zeros_like(hs)
    for ex in range(moe.num_experts):
        tok, slot = torch.where(ids == ex)
        if tok.numel() == 0:
            continue
        x_e = ops.rmsnorm_fp16_i4(hs[tok].contiguous(), n.weight, n.reorder_index, n.variance_epsilon)
        _, y_e = _expert_ref(moe, x_e, ex)
        out.index_add_(0, tok, (y_e * w[tok, slot, None]).half())
    return out


def _block(moe, hs):
    n = moe.norm
    return moe(hs, ops.rmsnorm_fp16_i4(hs, n.weight, n.reorder_index, n.variance_epsilon))


@pytest.mark.parametrize("shape,t", [(_TOY, 1), (_TOY, 33), (_TOY, 300), (_MIX, 1), (_MIX, 32), (_MIX, 512)],
                         ids=["toy-1", "toy-33", "toy-300", "mix-1", "mix-32", "mix-512"])
def test_moe_block_equals_unfused_composition(shape, t):
    moe = _cached_moe(shape)
    hs = (torch.randn(t, shape[0], device=DEV) * 2).half()
    assert torch.equal(_bits(_block(moe, hs)), _bits(_unfused(moe, hs)))


def test_moe_block_with_pdl():
    moe = _cached_moe(_TOY)
    hs = (torch.randn(40, 512, device=DEV) * 2).half()
    ref = _unfused(moe, hs)
    _lib.lib().atom_set_pdl(1)
    try:
        got = _block(moe, hs)
        torch.cuda.synchronize()
    finally:
        _lib.lib().atom_set_pdl(0)
    assert torch.equal(_bits(got), _bits(ref))


def test_moe_block_graph_replays_with_different_routings():
    moe = _cached_moe(_TOY)
    t, h = 32, 512
    g = torch.Generator(device=DEV).manual_seed(11)
    inputs = [(torch.randn(t, h, device=DEV, generator=g) * 2).half(), (torch.randn(t, h, device=DEV, generator=g) * 2).half()]
    inputs.append((torch.randn(1, h, device=DEV, generator=g) * 2).half().repeat(t, 1))     # every token to the same experts
    static = inputs[0].clone()
    _block(moe, static)                                   # descriptors and kernel attributes set up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            out = _block(moe, static)
    torch.cuda.current_stream().wait_stream(s)
    routes = []
    for hs in inputs:
        static.copy_(hs)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(out), _bits(_block(moe, hs)))
        routes.append(moe.route(hs)[0].cpu())
    assert not torch.equal(routes[0], routes[1]) and (routes[2] == routes[2][0]).all()


# ------------------------------------------------------------------------------------------------ layer
def test_exported_mixtral_layer_matches_oracle_chain_and_simulator():
    from oracle import oracle as O
    from tests.test_export_cpu import _input, _np
    from tests.test_moe_cpu import _build_mixtral
    q, _ = _build_mixtral(hidden=256, inter=256, experts=4, top_k=2, seed=7)
    real = q.to_int4(DEV)
    m, n = real.block_sparse_moe, real.post_attention_layernorm
    t = 9
    x = _input(t, 256, 3)
    xs = ops.rmsnorm_fp16_i4(x.to(DEV), n.weight, n.reorder_index, n.variance_epsilon)
    ids, w = m.route(x.to(DEV))
    got = m.experts(xs, ids, w).float().cpu().numpy()
    ids, w = ids.cpu().numpy(), w.cpu().numpy()
    c = lambda a: a.detach().cpu().numpy()  # noqa: E731
    ref = np.zeros((t, 256), np.float16)
    for r in range(t):
        hr = O.rmsnorm_fp16_i4(c(x)[r:r + 1], c(n.weight), c(n.reorder_index), n.variance_epsilon)
        for s in np.argsort(ids[r]):
            ex = int(ids[r, s])
            gate = O.gemm_i4_o16(hr[1], c(m.w13_int4[ex, :256]), hr[3], c(m.w13_scale[ex, :, :256]), hr[0], c(m.w13_int8[ex, :256]), hr[2],
                                 c(m.w13_keeper_scale[ex, :256]))
            up = O.gemm_i4_o16(hr[1], c(m.w13_int4[ex, 256:]), hr[3], c(m.w13_scale[ex, :, 256:]), hr[0], c(m.w13_int8[ex, 256:]), hr[2],
                               c(m.w13_keeper_scale[ex, 256:]))
            act = O.activate_fp16_i4(gate, up)
            ye = O.gemm_i4_o16(act[1], c(m.w2_int4[ex]), act[3], c(m.w2_scale[ex]), act[0], c(m.w2_int8[ex]), act[2], c(m.w2_keeper_scale[ex]))
            ref[r] = (ref[r] + (ye[0].astype(np.float32) * np.float32(w[r, s])).astype(np.float16)).astype(np.float16)
    ref = ref.astype(np.float32)
    assert np.abs(got - ref).max() <= 0.03 * np.abs(ref).max()
    sim, _ = q.block_sparse_moe(q.post_attention_layernorm(x.float()[None]))
    sim = _np(sim[0])
    assert np.abs(got - sim).max() <= 0.20 * np.abs(sim).max()


def test_mixtral_layer_prefill_then_decode_gqa_32_8():
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    cfg = MixtralConfig()
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.rope_theta, cfg.num_local_experts) == (32, 8, 1e6, 8)
    dev = torch.device(DEV)
    layer = MixtralDecoderLayer(cfg, 0).to(dev).init_random(2)
    t = 21
    x = (torch.randn(t + 2, 4096, device=dev) * 0.5).half()
    pool = KvPoolInt4(1, 8, 128, capacity=8, block_len=16, device=dev)
    cache = KvCacheInt4(pool, t)
    out_p = layer(x[:t], BatchLenInfo([t], 0, dev), BatchedKvCacheInt4([cache]), None)
    outs = []
    for i in range(2):
        cache.acquire_one()
        outs.append(layer(x[t + i:t + i + 1], BatchLenInfo([], 1, dev), None, BatchedKvCacheInt4([cache])))
    assert out_p.shape == (t, 4096) and all(o.shape == (1, 4096) for o in outs)
    assert torch.isfinite(out_p).all() and all(torch.isfinite(o).all() for o in outs)
    # the MoE delta is a real contribution, not zeros
    res, delta = layer.forward_residual(x[:4], None, BatchLenInfo([4], 0, dev), BatchedKvCacheInt4([KvCacheInt4(pool, 4)]), None)
    assert delta.abs().max() > 0
