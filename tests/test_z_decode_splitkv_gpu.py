"""GPU suite (-m gpu): split-KV decode attention -- batch_decode_kernel<G, kMaxTpl, kP, true>, each sequence's pages spread over a
cluster of C CTAs and merged through distributed shared memory.

  * every split instantiation (C in {2, 4, 8} x G in {1, 2, 4, 8} x every page size) inside the float64 bound of
    tests/attn_ref64.py, at lengths around the cluster's stripe period S*C*P, at 8k and 32k tokens, with peaked softmax and V
    scales of 16;
  * the result depends neither on the call nor on where the pages sit (dirty pools, other page orders: identical bytes);
  * kv_split = 0 is bit for bit the cluster size atom_decode_kv_split names, on both sides of the SM count;
  * kv_split = 1 is bit for bit the kernel of the parent revision (digests in tests/golden/decode_unsplit_h100.npz, written by
    tools/decode_unsplit_digests.py from that revision's library);
  * a CUDA graph (append + split decode, PDL on) replays bit for bit across a page boundary;
  * a one-KV-head Llama model checked step by step against tests/layer_ref64.py at batch 1 and 3, where the decode splits.

The bound is attn_ref64.decode_bound, unchanged.  Its FP32 term e (len/4 + 16) covers the cluster merge; the recount is in
DESIGN.md 5.3.  With k of the C <= 8 ranks holding pages, the rank-order merge adds k - 1 fmaf roundings and 2 ulp of exp2f to a
term's path: an empty rank adds an exact zero, and the rank holding the maximum is scaled by exactly 1.  Each lane's chain of
page adds loses at least k - 1 adds, so the path grows by at most 2 roundings, inside the term's len/8 of slack from len 16 on.
Below that, a second rank holds pages only at S = 1 and P = 8, where the stripe merge is one exact fmaf."""
import hashlib
import os
import types

import numpy as np
import pytest
import torch

from tests import attn_ref64 as R
from tests.test_z_attention_accuracy_gpu import A63, LN2, SIGMA_Q, _centred, _check, _pattern_seq, _scores

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decode_unsplit_h100.npz")
PAGES = [8, 16, 24, 32, 64]
THETAS = [1e4, 5e5, 1e6]


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


class _KV:
    def __init__(self, data, param, indptr, indices, last):
        self.data, self.param, self.indptr, self.indicies, self.last_page_offset = T(data), T(param), T(indptr), T(indices), T(last)


def stripes(G):
    """Page stripes of one CTA (kv_kernels.cuh dec_consumers(G) / G)."""
    return (4 if G == 1 else 8) // G


def _decode(q, pool, layer, theta, split):
    from atom_b200 import ops
    return ops.batch_decode_i4(T(q), _KV(*pool), layer, rope_theta=theta, kv_split=split).cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint16)


# ------------------------------------------------------------------------------------------------ 1. every split instantiation
@pytest.mark.parametrize("P", PAGES)
@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("C", [2, 4, 8])
def test_split_within_bound_and_independent_of_page_placement(C, G, P):
    """One token (every rank but rank 0 empty), a page and a bit, S*C*P - 1 / S*C*P / S*C*P + 1 and two periods and a bit, in one
    batch; then the same call on a dirty pool, on a pool in another page order, and once more: identical bytes."""
    hkv, theta = 2 if G < 8 else 1, THETAS[(C + G + P) % 3]
    period = stripes(G) * C * P
    lens = [1, P + 3, period - 1, period, period + 1, 2 * period + P // 2 + 3]
    seed = 100000 * C + 1000 * G + P
    rng = np.random.default_rng(seed)
    seqs = [_centred(rng, hkv, n) for n in lens]
    q = (rng.standard_normal((len(lens), G * hkv, 128)) * SIGMA_Q["moderate"]).astype(np.float16)
    pool = R.make_pool(seqs, P, hkv, L=2, layer=1, rng=np.random.default_rng(seed))
    got = _decode(q, pool, 1, theta, C)
    ref, bnd = R.decode_bound(q, *pool, 1, G * hkv, theta)
    _check(got, ref, bnd, f"split C={C} G={G} P={P} theta={theta:g}")
    dirty = R.make_pool(seqs, P, hkv, L=2, layer=1, rng=np.random.default_rng(seed), dirty=True)
    assert np.array_equal(_bits(_decode(q, dirty, 1, theta, C)), _bits(got))
    other = R.make_pool(seqs, P, hkv, L=2, layer=1, rng=np.random.default_rng(seed + 1), extra_pages=11)
    assert not np.array_equal(other[3], pool[3])
    assert np.array_equal(_bits(_decode(q, other, 1, theta, C)), _bits(got))
    assert np.array_equal(_bits(_decode(q, pool, 1, theta, C)), _bits(got))


@pytest.mark.parametrize("n,C,G,P,theta,regime", [(8192, 8, 1, 16, 1e4, "moderate"), (32768, 4, 4, 32, 5e5, "peaked"),
                                                  (32768, 8, 8, 64, 1e6, "moderate"), (8192, 2, 2, 24, 1e6, "peaked"),
                                                  (32768, 8, 1, 8, 1e4, "peaked")])
def test_split_long_contexts_within_bound(n, C, G, P, theta, regime):
    rng = np.random.default_rng(n + P + C)
    lens = [n, n - 37]
    seqs = [_centred(rng, 1, m) for m in lens]
    q = (rng.standard_normal((2, G, 128)) * SIGMA_Q[regime]).astype(np.float16)
    pool = R.make_pool(seqs, P, 1, rng=rng)
    got = _decode(q, pool, 0, theta, C)
    ref, bnd = R.decode_bound(q, *pool, 0, G, theta)
    _check(got, ref, bnd, f"split long {regime} C={C} G={G} len={n} P={P}")


@pytest.mark.parametrize("P", [32, 64])
@pytest.mark.parametrize("G", [1, 4])
@pytest.mark.parametrize("C", [2, 8])
def test_split_peaked_patterns_within_bound(C, G, P):
    """The maximum on the first token, on the last token, on a page of every rank, one token 45 nats above the rest."""
    theta = THETAS[P % 3]
    period = stripes(G) * C * P
    rng = np.random.default_rng(7 * C + G + P)
    low = lambda n: rng.uniform(0, 2, n)
    pats = []
    lv = low(period + P // 2 + 1); lv[0] = 12.0; pats.append(lv)
    lv = low(2 * period + P // 2 + 1); lv[-1] = 12.0; pats.append(lv)
    for r in range(C):
        lv = low(2 * period + 3); lv[period + r * stripes(G) * P + rng.integers(P)] = 12.0; pats.append(lv)
    lv = low(period + 5); lv[rng.integers(len(lv))] = 45.0; pats.append(lv)
    seqs = [_pattern_seq(rng, lv, theta) for lv in pats]
    q = np.zeros((len(seqs), G, 128), np.float16)
    q[:, :, 63] = A63 * (1 - 0.05 * np.arange(G))
    pool = R.make_pool(seqs, P, 1, rng=np.random.default_rng(P))
    got = _decode(q, pool, 0, theta, C)
    ref, bnd = R.decode_bound(q, *pool, 0, G, theta)
    _check(got, ref, bnd, f"split patterns C={C} G={G} P={P}")


@pytest.mark.parametrize("P", [32, 64])
@pytest.mark.parametrize("G", [1, 4])
@pytest.mark.parametrize("C", [2, 8])
def test_split_v_scale_16_stays_finite_and_within_bound(C, G, P):
    """Every V nibble 15 at scale 16 and every page of every global stripe 5.95 log2 units above the stripe's running maximum (the
    lazy rescale keeps it), then 8 more (rescaled): the half2 page sums reach 59 000 of FP16's 65 504."""
    theta = THETAS[P % 3]
    period = stripes(G) * C * P
    rng = np.random.default_rng(16 + P + C + G)
    lv = np.concatenate([np.full(period, base) for base in LN2 * np.array([0.5, 6.45, 14.45])])
    seqs = [_pattern_seq(rng, lv, theta, nib_v=15, vscale=(16.0, 16.0))]
    top = [s.reshape(-1, P).max(1) for s in _scores(seqs, P, theta)][0]
    assert 5.9 < (top[period // P] - top[0]) / LN2 < 6.0
    q = np.zeros((1, G, 128), np.float16); q[0, :, 63] = A63
    pool = R.make_pool(seqs, P, 1)
    got = _decode(q, pool, 0, theta, C)
    ref, bnd = R.decode_bound(q, *pool, 0, G, theta)
    _check(got, ref, bnd, f"split V scale 16 C={C} G={G} P={P}")


# ------------------------------------------------------------------------------------------------ 2. automatic selection
def _short_batch(rng, B, hkv, G, P):
    lens = rng.integers(1, 4 * P, B)
    seqs = [_centred(rng, hkv, int(n)) for n in lens]
    q = (rng.standard_normal((B, G * hkv, 128)) * SIGMA_Q["moderate"]).astype(np.float16)
    return q, R.make_pool(seqs, P, hkv, rng=rng)


def test_auto_is_the_split_the_rule_names_on_both_sides_of_the_sm_count():
    from atom_b200 import ops
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    grids = [(sms - 1, 1, 8), (sms, 1, 8), (sms + 1, 1, 8), (1, 8, 4), (4, 8, 4), (16, 8, 4), (32, 8, 4), (5, 8, 1), (3, 1, 8),
             (sms // 2, 2, 2)]
    splits = []
    for i, (B, hkv, G) in enumerate(grids):
        P = [16, 32, 8][i % 3]
        q, pool = _short_batch(np.random.default_rng(i), B, hkv, G, P)
        c = ops.decode_kv_split(B, hkv, G)
        assert (c == 1) == (B * hkv >= sms) and c in (1, 2, 4, 8)
        auto = _decode(q, pool, 0, 5e5, 0)
        assert np.array_equal(_bits(auto), _bits(_decode(q, pool, 0, 5e5, c))), (B, hkv, G, c)
        splits.append(c)
    assert splits[:3] == [2, 1, 1] and max(splits) == 8


def test_invalid_kv_split_raises_with_the_message():
    q, pool = _short_batch(np.random.default_rng(0), 2, 1, 1, 16)
    for bad in (3, 16, -1):
        with pytest.raises(RuntimeError, match=f"kv_split={bad} must be 0"):
            _decode(q, pool, 0, 1e4, bad)


# ------------------------------------------------------------------------------------------------ 3. the unsplit kernel is unchanged
# (G, P) reaching each of the 13 unsplit instantiations: <G,2,16>, <G,4,32>, <G,8,0>, and <1,4,0> / <1,8,0> for G = 1
UNSPLIT_CASES = [(1, 16), (1, 32), (1, 8), (1, 64)] + [(g, p) for g in (2, 4, 8) for p in (16, 32, 24)]


def unsplit_case(G, P):
    """Seeded inputs (q, pool, theta) of one unsplit case: two KV heads, a batch of mixed lengths, a dirty pool."""
    rng = np.random.default_rng(4242 + 100 * G + P)
    lens = [1, P - 1, P + 1, 4 * P + 3, 300, 1000]
    seqs = [_centred(rng, 2, n) for n in lens]
    q = (rng.standard_normal((len(lens), 2 * G, 128)) * SIGMA_Q["moderate"]).astype(np.float16)
    pool = R.make_pool(seqs, P, 2, L=2, layer=1, rng=rng, dirty=True)
    return q, pool, THETAS[(G + P) % 3]


def digest(o):
    return hashlib.sha256(np.ascontiguousarray(o).view(np.uint16).tobytes()).hexdigest()


def test_unsplit_outputs_are_bit_for_bit_the_parent_kernels():
    gold = np.load(GOLDEN)
    assert sorted(gold.files) == sorted(f"g{G}_p{P}" for G, P in UNSPLIT_CASES)
    for G, P in UNSPLIT_CASES:
        q, pool, theta = unsplit_case(G, P)
        assert digest(_decode(q, pool, 1, theta, 1)) == str(gold[f"g{G}_p{P}"]), (G, P)


# ------------------------------------------------------------------------------------------------ 4. CUDA graph with PDL
def test_graph_of_append_and_split_decode_replays_bit_for_bit_across_a_page_boundary():
    from atom_b200 import _lib, ops
    B, hkv, G, P, theta = 1, 8, 4, 16, 5e5
    assert ops.decode_kv_split(B, hkv, G) > 1
    dev = torch.device(DEV)
    gen = torch.Generator(device=dev).manual_seed(9)
    data = torch.randint(0, 256, (8, 1, 2, hkv, P, 64), dtype=torch.uint8, device=dev, generator=gen)
    param = torch.empty((8, 1, 2, hkv, P, 2), dtype=torch.float16, device=dev)
    param[..., 0].uniform_(0.01, 0.05, generator=gen); param[..., 1].uniform_(0.0, 0.4, generator=gen)
    pages = torch.tensor([5, 2, 7, 0, 3, 6, 1, 4], dtype=torch.int32, device=dev)
    kv = types.SimpleNamespace(data=data, param=param, indicies=pages, indptr=torch.zeros(2, dtype=torch.int32, device=dev),
                               last_page_offset=torch.zeros(1, dtype=torch.int32, device=dev))
    k = torch.empty((B, hkv, 64), dtype=torch.uint8, device=dev); v = torch.empty_like(k)
    kp = torch.empty((B, hkv, 2), dtype=torch.float16, device=dev); vp = torch.empty_like(kp)
    q = torch.empty((B, hkv * G, 128), dtype=torch.float16, device=dev)

    def set_step(n):      # the table of a sequence of n tokens and fresh inputs of its newest token
        kv.indptr.copy_(torch.tensor([0, (n + P - 1) // P], dtype=torch.int32))
        kv.last_page_offset.fill_((n - 1) % P + 1)
        k.random_(0, 256, generator=gen); v.random_(0, 256, generator=gen)
        kp.uniform_(0.01, 0.05, generator=gen); vp.uniform_(0.01, 0.05, generator=gen)
        q.normal_(generator=gen)

    def step():
        ops.append_kv_i4(kv, k, v, kp, vp, 0)
        return ops.batch_decode_i4(q, kv, 0, rope_theta=theta)

    torch.cuda.synchronize()
    _lib.check(_lib.lib().atom_set_pdl(1), "atom_set_pdl")
    try:
        set_step(29)
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            step()
            st.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                out = step()
        torch.cuda.current_stream().wait_stream(st)
        for n in range(30, 37):                                  # 32 -> 33 opens the third page
            set_step(n)
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            replayed = out.clone()
            eager = step()                                       # rewrites the same token into the same slot
            assert torch.equal(replayed, eager), n
    finally:
        torch.cuda.synchronize()
        _lib.check(_lib.lib().atom_set_pdl(0), "atom_set_pdl")


# ------------------------------------------------------------------------------------------------ 5. layers
@pytest.mark.timeout(600)
@pytest.mark.parametrize("prompts", [[37], [5, 37, 16]])
def test_one_kv_head_llama_steps_split_and_match_the_float64_reference(monkeypatch, prompts):
    from atom_b200 import ops
    from atom_b200.kvcache import KvPoolInt4
    from tests import layer_ref64 as LR
    from tests.test_z_layer_ref64_gpu import DEV as LDEV, Run, _model
    assert ops.decode_kv_split(len(prompts), 1, 4) > 1
    # lm_head is a torch FP16 GEMM: keep its split-K reductions in FP32, the arithmetic the logits bound counts
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_fp16_reduced_precision_reduction", False)
    P = 16
    model = _model(2, 512, 1024, 4, 1, 5e5)
    pool = KvPoolInt4(2, 1, 128, 24, P, LDEV)
    pool.buf.random_(0, 256)
    pool.param.view(torch.int16).random_(-32768, 32767)
    run = Run(monkeypatch, model, LR.model_ref(model, P), pool)
    run.step(prompts)
    for _ in range(12):
        run.step([])
    assert [c.seqlen for c in run.seqs] == [n + 12 for n in prompts]
