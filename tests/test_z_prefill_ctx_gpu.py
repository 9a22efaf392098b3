"""GPU suite (-m gpu): prefill over a cached prefix -- prefill_attn_kernel<true> reading the context from the INT4 pages.

  * every element of every chunk inside the float64 bound of tests/attn_ctx_ref64.py (prefill_ctx_bound: prefill_bound's terms with
    L = context + chunk), group sizes 1 / 4 / 8, page sizes 8 .. 64, RoPE bases 1e4 and 5e5, sink and moderate score regimes,
    contexts around the 64-token tile, mixed batches with empty contexts, pools whose unowned slots hold 0xFF / NaN, and one
    8192 + 512 case;
  * the FP16 scratch of the chunk at its absolute positions; the empty-context rows of a mixed batch bit for bit the kernel
    without a context; `kv=` with every context empty bit for bit the call without it;
  * a GQA Llama layer and a Mixtral layer prefilling 300 tokens in chunks: chunks that start at a multiple of 16 rows write the
    cache bytes of the one-shot prefill (others do not: see the test), and each chunk's attention lies inside the bound computed
    from the cache it ran on;
  * the text-generation harness with chunked prefill on a small model.
Fixed seeds, no retries."""
import numpy as np
import pytest
import torch

from tests import attn_ctx_ref64 as C
from tests import attn_ref64 as R

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


class _Kv:
    """The attributes ops.prefill_attention_i4 reads of a BatchedKvCacheInt4, on a numpy pool."""

    def __init__(self, data, param, indptr, indices, last):
        self.data, self.param, self.indptr, self.indicies, self.last_page_offset = T(data), T(param), T(indptr), T(indices), T(last)
        self.seqlens = [int((indptr[b + 1] - indptr[b] - 1) * data.shape[4] + last[b]) for b in range(len(last))]


def _check(got, ref, bnd, what):
    got = got.astype(np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output ({np.count_nonzero(~np.isfinite(got))} elements)"
    ratio = np.abs(got - ref) / bnd
    worst = float(ratio.max())
    at = np.unravel_index(int(ratio.argmax()), ratio.shape)
    assert worst <= 1.0, f"{what}: |kernel - ref64| exceeds the bound, worst error/bound = {worst:.3f} at {at} " \
                         f"(kernel {got[at]:.6g}, ref {ref[at]:.6g}, bound {bnd[at]:.3g})"
    print(f"worst error/bound {what}: {worst:.4f}")


def _direct(case, pool, lens, hq, hkv, theta, layer=0):
    """atom_prefill_attention_ctx_gqa_i4 through the C ABI: (out, kf, vf)."""
    from atom_b200 import _lib, ops
    q, k4, kp, v4, vp = case
    kv = _Kv(*pool)
    ctx = [s - n for s, n in zip(kv.seqlens, lens)]
    t = sum(lens)
    args = [T(x) for x in (q, k4, kp, v4, vp)]
    ip = T(np.array([0] + list(np.cumsum(lens)), np.int32))
    pos = T(np.concatenate([np.arange(c, c + n) for c, n in zip(ctx, lens)]).astype(np.int32))
    table = ops.rope_table(max(c + n for c, n in zip(ctx, lens)), torch.device(DEV), theta)
    kf = torch.empty(t, hkv * 128, dtype=torch.float16, device=DEV)
    vf, out = torch.empty_like(kf), torch.empty(t, hq * 128, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().atom_prefill_attention_ctx_gqa_i4(
        *[a.data_ptr() for a in args], ip.data_ptr(), pos.data_ptr(), table.data_ptr(), kf.data_ptr(), vf.data_ptr(), out.data_ptr(),
        t, len(lens), max(lens), hq, hkv, kv.data.data_ptr(), kv.param.data_ptr(), kv.indptr.data_ptr(), kv.indicies.data_ptr(),
        kv.last_page_offset.data_ptr(), pool[0].shape[1], layer, pool[0].shape[4], torch.cuda.current_stream().cuda_stream),
        "prefill_attention_ctx_gqa_i4")
    return out.cpu().numpy(), kf.cpu().numpy(), vf.cpu().numpy(), ctx


def _check_scratch(kf, vf, case, lens, ctx, theta):
    """kf / vf as tests/test_z_attention_accuracy_gpu.py checks them, at the absolute positions ctx_b + i."""
    _, k4, kp, v4, vp = case
    t, hkv = kf.shape[0], kf.shape[1] // 128
    k = R.dequant(R.unpack(k4.reshape(t, hkv, 64)), kp.reshape(t, hkv, 2)).astype(np.float16).astype(np.float64)
    v = R.dequant(R.unpack(v4.reshape(t, hkv, 64)), vp.reshape(t, hkv, 2))
    pos = np.concatenate([np.arange(c, c + n) for c, n in zip(ctx, lens)]).astype(np.float64)
    kr = R.rotate(k.transpose(1, 0, 2), pos, theta).transpose(1, 0, 2).reshape(t, hkv * 128)
    vr = v.reshape(t, hkv * 128)
    zk = np.abs(k[..., :64] + 1j * k[..., 64:])
    ulp = lambda x: np.spacing(np.abs(x).astype(np.float16)).astype(np.float64)
    ang = R.E * (32 * np.multiply.outer(pos, R.freqs(theta)) + 8)[:, None, :] * zk
    tol = ulp(kr) + np.concatenate([ang, ang], -1).reshape(t, hkv * 128) + 2.0 ** -24
    bad = np.abs(kf.astype(np.float64) - kr) > tol
    assert not bad.any(), f"kf: {np.count_nonzero(bad)} elements off, first at {np.argwhere(bad)[0]}"
    bad = np.abs(vf.astype(np.float64) - vr) > ulp(vr) + 2.0 ** -24
    assert not bad.any(), f"vf: {np.count_nonzero(bad)} elements off, first at {np.argwhere(bad)[0]}"


def _plain(case, lens, hq, theta):
    from atom_b200 import ops
    q, k4, kp, v4, vp = [T(x) for x in case]
    ip = T(np.array([0] + list(np.cumsum(lens)), np.int32))
    return ops.prefill_attention_i4(q, k4, kp, v4, vp, ip, seqlens=list(lens), rope_theta=theta).cpu().numpy()


# ------------------------------------------------------------------------------------------------ 1. the kernel in the bound
CTXS = [1, 63, 64, 65, 1000, 0, 64, 0]
LENS = [129, 1, 17, 64, 129, 17, 1, 64]


@pytest.mark.parametrize("regime", ["sink", "moderate"])
@pytest.mark.parametrize("theta", [1e4, 5e5])
@pytest.mark.parametrize("P", [8, 16, 32, 64])
@pytest.mark.parametrize("hq,hkv", [(2, 2), (8, 2), (8, 1)])
def test_chunks_over_cached_context_within_bound(hq, hkv, P, theta, regime):
    rng = np.random.default_rng(hq * 1000 + hkv * 100 + P + (regime == "sink"))
    dirty = P in (16, 64)
    case, pool = C.make_ctx_case(rng, CTXS, LENS, hq, hkv, P, regime, dirty=dirty, L=2, layer=1)
    got, kf, vf, ctx = _direct(case, pool, LENS, hq, hkv, theta, layer=1)
    assert ctx == CTXS
    _check_scratch(kf, vf, case, LENS, ctx, theta)
    ref, bnd = C.prefill_ctx_bound(*case, LENS, hq, theta, *pool, layer=1)
    _check(got, ref, bnd, f"prefill ctx {regime} G={hq // hkv} P={P} theta={theta:g}{' dirty' if dirty else ''}")
    # the empty-context prompts of the batch: bit for bit the kernel without a context
    plain = _plain(case, LENS, hq, theta)
    off = np.concatenate([[0], np.cumsum(LENS)])
    for b, c in enumerate(CTXS):
        if c == 0:
            assert np.array_equal(got[off[b]:off[b + 1]].view(np.uint16), plain[off[b]:off[b + 1]].view(np.uint16)), f"prompt {b}"


def test_ops_path_equals_the_c_abi_and_empty_contexts_take_the_plain_path():
    from atom_b200 import ops
    rng = np.random.default_rng(7)
    hq, hkv, theta, lens = 8, 2, 5e5, [65, 17, 1]
    case, pool = C.make_ctx_case(rng, [200, 0, 64], lens, hq, hkv, 32, "sink", dirty=True)
    got, _, _, _ = _direct(case, pool, lens, hq, hkv, theta)
    q, k4, kp, v4, vp = [T(x) for x in case]
    ip = T(np.array([0] + list(np.cumsum(lens)), np.int32))
    via_ops = ops.prefill_attention_i4(q, k4, kp, v4, vp, ip, seqlens=lens, rope_theta=theta, kv=_Kv(*pool), layer_idx=0).cpu().numpy()
    assert np.array_equal(got.view(np.uint16), via_ops.view(np.uint16))
    case0, pool0 = C.make_ctx_case(rng, [0, 0, 0], lens, hq, hkv, 32, "moderate", dirty=True)
    q, k4, kp, v4, vp = [T(x) for x in case0]
    a = ops.prefill_attention_i4(q, k4, kp, v4, vp, ip, seqlens=lens, rope_theta=theta, kv=_Kv(*pool0), layer_idx=0)
    b = ops.prefill_attention_i4(q, k4, kp, v4, vp, ip, seqlens=lens, rope_theta=theta)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    short = _Kv(*C.make_ctx_case(rng, [0, 0, 0], [65, 16, 1], hq, hkv, 32)[1])
    with pytest.raises(RuntimeError, match="fewer than its prompt"):
        ops.prefill_attention_i4(q, k4, kp, v4, vp, ip, seqlens=lens, kv=short, layer_idx=0)
    with pytest.raises(RuntimeError, match="2 sequences for 3 prompts"):
        ops.prefill_attention_i4(q, k4, kp, v4, vp, ip, seqlens=lens, kv=_Kv(*C.make_ctx_case(rng, [0, 0], [65, 17], hq, hkv, 32)[1]),
                                 layer_idx=0)


def test_group_size_and_page_size_are_checked():
    from atom_b200 import _lib
    rng = np.random.default_rng(8)
    case, pool = C.make_ctx_case(rng, [10], [5], 6, 2, 16)
    with pytest.raises(RuntimeError, match="supported group sizes"):
        _direct(case, pool, [5], 6, 2, 1e4)
    case, pool = C.make_ctx_case(rng, [10], [5], 2, 2, 12)
    with pytest.raises(RuntimeError, match="page_size=12"):
        _direct(case, pool, [5], 2, 2, 1e4)
    assert "atom_prefill_attention_ctx_gqa_i4" in _lib.symbols()


def test_8192_token_context_and_512_token_chunk_within_bound():
    hq, hkv, theta, P = 8, 2, 5e5, 32
    rng = np.random.default_rng(8192)
    case, pool = C.make_ctx_case(rng, [8192], [512], hq, hkv, P, "sink")
    got, kf, vf, ctx = _direct(case, pool, [512], hq, hkv, theta)
    _check_scratch(kf, vf, case, [512], ctx, theta)
    rows = sorted(set(range(16)) | set(range(496, 512)) | {64 * j + d for j in range(1, 8) for d in (-1, 0)}
                  | set(rng.choice(512, 48, replace=False).tolist()))
    ref, bnd = C.prefill_ctx_bound(*case, [512], hq, theta, *pool, rows={0: rows})
    _check(got, ref, bnd, "prefill ctx 8192 + 512 G=4")


# ------------------------------------------------------------------------------------------------ 2. layers, chunked vs one shot
def _llama_layer():
    from atom_b200.llama import LlamaConfig, LlamaDecoderLayer
    torch.manual_seed(5)
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=1024, num_attention_heads=8, num_key_value_heads=2, num_hidden_layers=1,
                      rope_theta=5e5)
    layer = LlamaDecoderLayer(cfg, 0).to(DEV).init_random(5)
    return layer.eval(), cfg


def _mixtral_layer():
    from atom_b200.mixtral import MixtralConfig, MixtralDecoderLayer
    torch.manual_seed(7)
    cfg = MixtralConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=1,
                        num_local_experts=4, num_experts_per_tok=2, rope_theta=1e6)
    layer = MixtralDecoderLayer(cfg, 0).to(DEV).init_random(7)
    return layer.eval(), cfg


@pytest.mark.timeout(600)
@pytest.mark.parametrize("chunks", [[64, 100, 136], [64, 96, 140]], ids=["64-100-136", "64-96-140"])
@pytest.mark.parametrize("make", [_llama_layer, _mixtral_layer], ids=["llama_gqa", "mixtral"])
def test_chunked_layer_prefill_against_one_shot(monkeypatch, make, chunks):
    """A 300-token prompt prefilled in chunks and in one shot.  The cache bytes of every chunk that starts at a multiple of 16
    rows are those of the one-shot prefill, bit for bit.  A chunk that starts elsewhere (164 in 64 + 100 + 136) gets different
    K/V codes for its tokens: the W4A4 projection of a token depends on its row's position modulo 16 in the batch (measured on
    an H100: rows shifted by 4 or 8 modulo 16 differ, the fused q/k/v launch agreeing with the separate projections at every
    M), so the k/v projections are not row-local.  Every chunk's attention lies inside the float64 bound computed from the cache
    it ran on."""
    from atom_b200 import ops
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    layer, cfg = make()
    hq, hkv, theta, P, n = cfg.num_attention_heads, cfg.num_key_value_heads, float(cfg.rope_theta), 16, 300
    x = torch.from_numpy((np.random.default_rng(3).standard_normal((n, cfg.hidden_size)) * 0.5).astype(np.float16)).to(DEV)
    calls = []
    real = ops.prefill_attention_i4

    def spy(*a, **kw):
        out = real(*a, **kw)
        calls.append((a, kw, out))
        return out
    monkeypatch.setattr(ops, "prefill_attention_i4", spy)

    pools = []
    for plan in ([n], chunks):
        pool = KvPoolInt4(1, hkv, 128, 24, P, DEV)
        pool.buf.zero_(); pool.param.zero_()
        cache, a = KvCacheInt4(pool, 0), 0
        with torch.inference_mode():
            for c in plan:
                cache.acquire(c)
                layer(x[a:a + c], BatchLenInfo([c], 0, DEV), BatchedKvCacheInt4([cache]), None)
                a += c
        torch.cuda.synchronize()
        pools.append((pool.buf.cpu().numpy(), pool.param.cpu().numpy(), list(cache.indicies)))
    assert pools[0][2] == pools[1][2]
    pg = pools[0][2]
    tok = lambda a: a[pg, 0].transpose(1, 2, 0, 3, 4).reshape(2, hkv, -1, a.shape[-1])[:, :, :n]
    b0, b1 = tok(pools[0][0]), tok(pools[1][0])
    p0, p1 = tok(pools[0][1]).view(np.uint16), tok(pools[1][1]).view(np.uint16)
    starts = np.cumsum([0] + chunks[:-1])
    aligned = np.concatenate([np.arange(a, a + c) for a, c in zip(starts, chunks) if a % 16 == 0])
    assert np.array_equal(b0[:, :, aligned], b1[:, :, aligned]), "K/V bytes of 16-row-aligned chunks differ from one shot"
    assert np.array_equal(p0[:, :, aligned], p1[:, :, aligned]), "K/V parameters of 16-row-aligned chunks differ from one shot"
    # every chunk's attention (the first call is the one-shot prefill) inside the float64 bound from the chunked cache
    assert len(calls) == 1 + len(chunks) and all(("kv" in kw) == (a > 0) for (_, kw, _), a in zip(calls[1:], starts))
    data, param = pools[1][0], pools[1][1]
    for (args, kw, out), ctx in zip(calls[1:], starts):
        q, k4, kp, v4, vp = [t.cpu().numpy() for t in args[:5]]
        lens = kw["seqlens"]
        if "kv" in kw:
            kv = kw["kv"]
            assert kv.seqlens == [ctx + lens[0]]
            tbl = (data, param, kv.indptr.cpu().numpy(), kv.indicies.cpu().numpy(), kv.last_page_offset.cpu().numpy())
            ref, bnd = C.prefill_ctx_bound(q, k4, kp, v4, vp, lens, hq, theta, *tbl)
        else:
            ref, bnd = R.prefill_bound(q, k4, kp, v4, vp, lens, hq, theta)
        _check(out.cpu().numpy(), ref, bnd, f"{make.__name__} chunk at {ctx} (+{lens[0]})")


# ------------------------------------------------------------------------------------------------ 3. harness
def _textgen(chunk, graphs=False):
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvPoolInt4
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM
    dev = torch.device(DEV)
    torch.manual_seed(11)
    torch.set_default_dtype(torch.float16)
    try:
        with dev:
            model = LlamaForCausalLM(LlamaConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2,
                                                 num_hidden_layers=2, vocab_size=128))
    finally:
        torch.set_default_dtype(torch.float32)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    rs = tg.generate_request_set(7, 72)
    pool = KvPoolInt4(2, 2, 128, tg.pool_capacity(3, 72, 16), 16, dev)
    free0 = pool.num_free_blocks
    runner = tg.DecodeGraphRunner(model.eval(), pool, dev, max_pages_per_seq=72 // 16 + 1) if graphs else None
    res = tg.run_textgen(model.eval(), rs, tg.TextGenConfig(3, prefill_chunk=chunk), pool, dev, sync=torch.cuda.synchronize,
                         keep_tokens=True, decode_runner=runner)
    assert pool.num_free_blocks == free0
    assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
    assert all(0 <= t < 128 for toks in res.tokens for t in toks)
    assert (res.graphed_steps > 0) == graphs
    return res.tokens


@pytest.mark.timeout(600)
def test_textgen_with_chunked_prefill():
    base = _textgen(None)
    assert _textgen(10 ** 6) == base                    # a budget no step reaches: today's schedule, the same tokens
    _textgen(16)
    _textgen(64)
    _textgen(16, graphs=True)
