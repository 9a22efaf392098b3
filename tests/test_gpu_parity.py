"""GPU parity suite (-m gpu): every kernel, called through the C ABI (atom_b200.ops -> libatom_b200.so), against
the CPU oracle on the same seeded inputs.  Integer / packing / index paths are bit-exact; FP paths carry the
tolerance written next to each assert.  The companion suite test_gpu_vs_reference.py compares with the
reference's own CUDA kernels (oracle/_ref) on the same GPU."""
import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def nib_diff(p, q):
    return np.abs(O.unpack_int4(p).astype(np.int32) - O.unpack_int4(q).astype(np.int32))


def _quant_inputs(rng, m, h):
    x = (rng.standard_normal((m, h)) * np.where(rng.random((1, h)) > 0.97, 12.0, 1.0)).astype(np.float16)
    idx = rng.permutation(h).astype(np.int16)
    return x, idx


def _cmp_quant(out, ref, exact):
    o8, o4, s8, s4 = [t.cpu().numpy() for t in out]
    r8, r4, rs8, rs4 = ref
    m = r8.shape[0]
    if exact:
        assert np.array_equal(o8, r8)
        assert np.array_equal(o4.view(np.uint8), r4)
        assert np.array_equal(O.a_scale_from_layout(s8, m).view(np.uint16), O.a_scale_from_layout(rs8, m).view(np.uint16))
        assert np.array_equal(O.a_scale_from_layout(s4, m).view(np.uint16), O.a_scale_from_layout(rs4, m).view(np.uint16))
    else:  # approximate rsqrtf / expf on the GPU: +-1 LSB, the reference's own tolerance (test_Reorder.cu:269-318)
        assert np.abs(o8.astype(np.int32) - r8.astype(np.int32)).max() <= 1
        assert nib_diff(o4.view(np.uint8), r4).max() <= 1
        assert (nib_diff(o4.view(np.uint8), r4) != 0).mean() < 5e-3
        assert np.allclose(O.a_scale_from_layout(s4, m).astype(np.float32), O.a_scale_from_layout(rs4, m).astype(np.float32), rtol=2e-3)
        assert np.allclose(O.a_scale_from_layout(s8, m).astype(np.float32), O.a_scale_from_layout(rs8, m).astype(np.float32), rtol=2e-3)
    # replicas of the scale layout: all four copies written
    idx = np.array([O.scale_index(r) for r in range(m)])
    for j in range(1, 4):
        assert np.array_equal(s8[idx + 2 * j].view(np.uint16), s8[idx].view(np.uint16))
        assert np.array_equal(s4[:, idx + 2 * j].view(np.uint16), s4[:, idx].view(np.uint16))


@pytest.mark.parametrize("m,h", [(1, 4096), (7, 4096), (16, 4096), (21, 4096), (129, 4096), (33, 5120), (5, 8192), (3, 256)])
def test_reorder_bit_exact(m, h):
    from atom_b200 import ops
    rng = np.random.default_rng(m * 131 + h)
    x, idx = _quant_inputs(rng, m, h)
    _cmp_quant(ops.reorder_fp16_i4(T(x), T(idx)), O.reorder_fp16_i4(x, idx), exact=True)


@pytest.mark.parametrize("m,h", [(1, 4096), (7, 4096), (16, 4096), (40, 4096), (9, 5120), (4, 8192)])
def test_rmsnorm_quant(m, h):
    from atom_b200 import ops
    rng = np.random.default_rng(m * 17 + h)
    x, idx = _quant_inputs(rng, m, h)
    w = (1 + 0.2 * rng.standard_normal(h)).astype(np.float16)
    _cmp_quant(ops.rmsnorm_fp16_i4(T(x), T(w), T(idx), 1e-5), O.rmsnorm_fp16_i4(x, w, idx, 1e-5), exact=False)


@pytest.mark.parametrize("m,h", [(1, 4096), (16, 4096), (33, 5120), (7, 8192), (3, 384)])
def test_add_rmsnorm_equals_add_then_rmsnorm(m, h):
    """EXTENSION op (launch-count reduction): residual add folded into the norm+quantise kernel -- must be bit-identical to the
    two-step form the reference's decoder layer executes (llama.py:266-292)."""
    from atom_b200 import ops
    rng = np.random.default_rng(m * 13 + h)
    x, idx = _quant_inputs(rng, m, h)
    res = (rng.standard_normal((m, h)) * 2).astype(np.float16)
    w = (1 + 0.2 * rng.standard_normal(h)).astype(np.float16)
    s, fused = ops.add_rmsnorm_fp16_i4(T(x), T(res), T(w), T(idx), 1e-5)
    s_ref = T(res) + T(x)
    two = ops.rmsnorm_fp16_i4(s_ref, T(w), T(idx), 1e-5)
    assert torch.equal(s, s_ref)
    assert torch.equal(fused[0], two[0]) and torch.equal(fused[1], two[1])
    sel = torch.tensor([O.scale_index(r) + 2 * j for r in range(m) for j in range(4)], device="cuda:0")
    assert torch.equal(fused[2][sel], two[2][sel]) and torch.equal(fused[3][:, sel], two[3][:, sel])


@pytest.mark.parametrize("m,h", [(1, 11008), (7, 11008), (16, 11008), (5, 13824), (3, 22016), (33, 4096), (2, 2816)])
def test_activate_quant(m, h):
    from atom_b200 import ops
    rng = np.random.default_rng(m * 29 + h)
    a = (rng.standard_normal((m, h)) * 2).astype(np.float16)
    b = (rng.standard_normal((m, h)) * 2).astype(np.float16)
    _cmp_quant(ops.activate_fp16_i4(T(a), T(b)), O.activate_fp16_i4(a, b), exact=False)


def _ulp_diff(a, b):
    """distance in fp16 ulps between two float16 arrays (monotone integer mapping)"""
    def key(x):
        u = x.view(np.uint16).astype(np.int32)
        return np.where(u & 0x8000, 0x8000 - u, u)
    return np.abs(key(a) - key(b))


GEMM_CASES = [
    # (M, N, K, flags, exact)   flags: 0 auto, 1 no split-K, 2 force tall, 4 force skinny
    (16, 256, 512, 2, True), (128, 128, 256, 2, True), (7, 128, 384, 2, True), (129, 384, 1024, 2, True),
    (300, 256, 4096, 2, True),
    (16, 256, 512, 5, True), (7, 128, 384, 5, True), (1, 128, 256, 5, True), (33, 256, 1024, 5, True),
    (64, 384, 4096, 5, True), (16, 4096, 4096, 1, True),
    (16, 4096, 4096, 0, False), (32, 1024, 4096, 0, False), (48, 512, 11008, 0, False), (5, 128, 2048, 0, False),
    (130, 2752, 1024, 0, True), (100, 256, 2048, 0, False), (128, 512, 512, 1, True), (65, 1024, 4096, 1, True),
    # 512 / 1024 = prefill tile hints of earlier versions, accepted and ignored: partial channel tiles, M tails, long K
    (300, 256, 4096, 512, True), (129, 384, 1024, 512, True), (130, 2752, 1024, 512, True), (7, 512, 384, 512, True),
    (1000, 1024, 2048, 1024, True),
]


@pytest.mark.parametrize("m,n,k,flags,exact", GEMM_CASES)
def test_gemm_o16(m, n, k, flags, exact):
    from atom_b200 import ops
    t = O.make_gemm_inputs(m, n, k, seed=m * 7919 + n * 31 + k, pair_shared=(m % 2 == 0))
    d = ops.dense_layer_gemm_i4_fp16(*[T(x) for x in t], flags=flags).cpu().numpy()
    rows = None if m * n * k <= (1 << 28) else sorted(set(np.random.default_rng(1).integers(0, m, 24).tolist() + [0, m - 1]))
    ref = O.gemm_i4_o16(*t, rows=rows)
    got = d if rows is None else d[rows]
    if exact:   # same association as the reference: groups in order, keeper last -> bit exact
        assert np.array_equal(got.view(np.uint16), ref.view(np.uint16)), f"max ulp {_ulp_diff(got, ref).max()}"
    else:       # split-K: FP32 partial sums are added in a different order -> at most 1 fp16 ulp, rarely
        ud = _ulp_diff(got, ref)
        assert ud.max() <= 1 and (ud != 0).mean() < 0.02
        assert np.allclose(got.astype(np.float32), ref.astype(np.float32), rtol=1e-3, atol=1e-3 * np.abs(ref.astype(np.float32)).mean())


@pytest.mark.parametrize("m,n,k,flags", [(16, 256, 512, 2), (130, 384, 1024, 2), (16, 256, 512, 5), (7, 128, 1024, 5),
                                         (48, 4096, 4096, 1), (16, 4096, 4096, 1), (130, 384, 1024, 512), (300, 512, 2048, 512)])
def test_gemm_o4(m, n, k, flags):
    from atom_b200 import ops
    t = O.make_gemm_inputs(m, n, k, seed=m + n + k)
    d, ds = ops.dense_layer_gemm_i4_o4(*[T(x) for x in t], flags=flags)
    d, ds = d.cpu().numpy(), ds.cpu().numpy()
    rows = None if m * n * k <= (1 << 28) else [0, 3, m - 1]
    rd, rds = O.gemm_i4_o4(*t, rows=rows)
    if rows is not None:
        d, ds = d[rows], ds[rows]
    assert np.array_equal(ds.view(np.uint16), rds.view(np.uint16))       # (scale, zero): bit exact
    assert np.array_equal(d, rd)                                           # packed INT4: bit exact


def _kv_fixture(rng, B, H, P, L, lens):
    pages = sum((l + P - 1) // P for l in lens) + 3
    data = rng.integers(0, 256, (pages, L, 2, H, P, 64), dtype=np.uint8)
    param = np.stack([rng.uniform(0.01, 0.05, (pages, L, 2, H, P)), rng.uniform(0, 0.4, (pages, L, 2, H, P))], -1).astype(np.float16)
    perm = rng.permutation(pages)
    indptr, indices, last, c = [0], [], [], 0
    for l in lens:
        npg = (l + P - 1) // P
        indices += list(perm[c:c + npg]); c += npg
        indptr.append(len(indices)); last.append((l - 1) % P + 1)
    return data, param, np.array(indptr, np.int32), np.array(indices, np.int32), np.array(last, np.int32)


class _KV:
    def __init__(self, data, param, indptr, indices, last):
        self.data, self.param, self.indptr, self.indicies, self.last_page_offset = T(data), T(param), T(indptr), T(indices), T(last)


@pytest.mark.parametrize("B,H,P,lens", [(3, 2, 16, [1, 37, 64]), (7, 4, 16, [5, 499, 16, 17, 250, 333, 32]),
                                        (2, 3, 32, [2048, 777]), (4, 2, 8, [8, 9, 1, 100])])
def test_batch_decode(B, H, P, lens):
    from atom_b200 import ops
    rng = np.random.default_rng(B * 100 + P)
    L = 2
    data, param, indptr, indices, last = _kv_fixture(rng, B, H, P, L, lens)
    q = rng.standard_normal((B, H, 128)).astype(np.float16)
    kv = _KV(data, param, indptr, indices, last)
    for layer in range(L):
        o = ops.batch_decode_i4(T(q), kv, layer).cpu().numpy()
        ref = O.batch_decode_i4(q, data, param, indptr, indices, last, layer)
        # FP16 output of an FP32 softmax-attention with approximate-vs-exact transcendental differences:
        # rtol/atol 5e-4: the bound the reference's own test intends (test_batch_decode_int4.py:9-14), SURVEY.md 8(c) policy (4)
        err = np.abs(o.astype(np.float32) - ref.astype(np.float32)) - 5e-4 * np.abs(ref.astype(np.float32))
        assert err.max() <= 5e-4, f"layer {layer}: worst excess over rtol*|ref| = {err.max():.2e} (atol 5e-4)"


def test_append_and_init_kv_bit_exact():
    from atom_b200 import ops
    rng = np.random.default_rng(5)
    B, H, P, L = 5, 8, 16, 3
    lens = [1, 16, 17, 40, 64]
    data, param, indptr, indices, last = _kv_fixture(rng, B, H, P, L, lens)
    k = rng.integers(0, 256, (B, H, 64), dtype=np.uint8); v = rng.integers(0, 256, (B, H, 64), dtype=np.uint8)
    kp = rng.random((B, H, 2)).astype(np.float16); vp = rng.random((B, H, 2)).astype(np.float16)
    kv = _KV(data, param, indptr, indices, last)
    ops.append_kv_i4(kv, T(k), T(v), T(kp), T(vp), 1)
    d_ref, p_ref = data.copy(), param.copy()
    O.append_kv_i4(d_ref, p_ref, indptr, indices, last, k, v, kp, vp, 1)
    assert np.array_equal(kv.data.cpu().numpy(), d_ref) and np.array_equal(kv.param.cpu().numpy().view(np.uint16), p_ref.view(np.uint16))
    tot = sum(lens)
    K = rng.integers(0, 256, (tot, H, 64), dtype=np.uint8); V = rng.integers(0, 256, (tot, H, 64), dtype=np.uint8)
    KP = rng.random((tot, H, 2)).astype(np.float16); VP = rng.random((tot, H, 2)).astype(np.float16)
    sl = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    kv2 = _KV(data, param, indptr, indices, last)
    ops.init_kv_i4(kv2, T(K), T(V), T(KP), T(VP), T(sl), 2)
    d_ref, p_ref = data.copy(), param.copy()
    O.init_kv_i4(d_ref, p_ref, indptr, indices, last, K, V, KP, VP, sl, 2)
    assert np.array_equal(kv2.data.cpu().numpy(), d_ref) and np.array_equal(kv2.param.cpu().numpy().view(np.uint16), p_ref.view(np.uint16))


def test_errors_are_loud():
    from atom_b200 import ops
    t = [T(x) for x in O.make_gemm_inputs(16, 100, 512)]   # N not a multiple of 8
    with pytest.raises(RuntimeError):
        ops.dense_layer_gemm_i4_fp16(*t)
    with pytest.raises(RuntimeError):
        ops.reorder_fp16_i4(torch.zeros(4, 4096, dtype=torch.float16), torch.zeros(4096, dtype=torch.int16))  # CPU tensors


def _concat_weights(parts):
    """Row-concatenate LinearInt4-style operand tuples (b, b_scale [G, N], b_keeper, b_keeper_scale) of equal K."""
    b = np.concatenate([p[0] for p in parts], 0)
    bs = np.concatenate([p[1] for p in parts], 1)
    bk = np.concatenate([p[2] for p in parts], 0)
    bks = np.concatenate([p[3] for p in parts], 0)
    return b, bs, bk, bks


@pytest.mark.parametrize("m,h,k", [(16, 256, 512), (7, 384, 1024), (32, 512, 2048), (48, 128, 512), (16, 4096, 4096), (100, 256, 1024)])
def test_fused_qkv_equals_three_projections(m, h, k):
    """EXTENSION op: one launch for q (fp16) + k, v (o4) must reproduce the three operator calls bit for bit."""
    from atom_b200 import ops
    t = [O.make_gemm_inputs(m, h, k, seed=m + h + k + i) for i in range(3)]
    act = [T(t[0][i]) for i in (0, 2, 4, 6)]                      # a, a_scale, a_keeper, a_keeper_scale of the first set
    ws = [(x[1], x[3], x[5], x[7]) for x in t]
    q_ref = ops.dense_layer_gemm_i4_fp16(act[0], T(ws[0][0]), act[1], T(ws[0][1]), act[2], T(ws[0][2]), act[3], T(ws[0][3]), flags=1)
    k_ref = ops.dense_layer_gemm_i4_o4(act[0], T(ws[1][0]), act[1], T(ws[1][1]), act[2], T(ws[1][2]), act[3], T(ws[1][3]))
    v_ref = ops.dense_layer_gemm_i4_o4(act[0], T(ws[2][0]), act[1], T(ws[2][1]), act[2], T(ws[2][2]), act[3], T(ws[2][3]))
    b, bs, bk, bks = _concat_weights(ws)
    q, (kk, ks), (vv, vs) = ops.dense_layer_gemm_i4_qkv(act[0], T(b), act[1], T(bs), act[2], T(bk), act[3], T(bks))
    assert torch.equal(q, q_ref)
    assert torch.equal(kk, k_ref[0]) and torch.equal(ks, k_ref[1])
    assert torch.equal(vv, v_ref[0]) and torch.equal(vs, v_ref[1])


@pytest.mark.parametrize("m,inter,k", [(16, 256, 512), (5, 384, 1024), (32, 512, 1024), (64, 256, 512), (16, 11008, 4096)])
def test_fused_gateup_activation_equals_three_calls(m, inter, k):
    """EXTENSION op: gate_proj + up_proj + activate_fp16_i4 in one launch: the activation 4-tuple must be bit-identical."""
    from atom_b200 import ops
    t = [O.make_gemm_inputs(m, inter, k, seed=3 * m + inter + k + i) for i in range(2)]
    act = [T(t[0][i]) for i in (0, 2, 4, 6)]
    ws = [(x[1], x[3], x[5], x[7]) for x in t]
    g = ops.dense_layer_gemm_i4_fp16(act[0], T(ws[0][0]), act[1], T(ws[0][1]), act[2], T(ws[0][2]), act[3], T(ws[0][3]), flags=1)
    u = ops.dense_layer_gemm_i4_fp16(act[0], T(ws[1][0]), act[1], T(ws[1][1]), act[2], T(ws[1][2]), act[3], T(ws[1][3]), flags=1)
    ref = ops.activate_fp16_i4(g, u)
    b, bs, bk, bks = _concat_weights(ws)
    got = ops.dense_layer_gemm_i4_gateup_act(act[0], T(b), act[1], T(bs), act[2], T(bk), act[3], T(bks))
    assert torch.equal(got[0], ref[0]), "INT8 outliers differ"
    if not torch.equal(got[1], ref[1]):        # say where: a whole tile (hand-off / launch problem) or single codes (arithmetic)
        bad = (got[1] != ref[1]).nonzero()
        cols = sorted(set((bad[:, 1] // 64).tolist()))
        raise AssertionError(f"packed INT4 differs: {bad.shape[0]} bytes, rows {sorted(set(bad[:, 0].tolist()))[:8]}, "
                             f"channel tiles {cols[:12]} ({len(cols)} tiles), first {bad[0].tolist()}: "
                             f"{int(got[1][tuple(bad[0])])} vs {int(ref[1][tuple(bad[0])])}")
    sel = torch.tensor([O.scale_index(r) + 2 * j for r in range(m) for j in range(4)], device="cuda:0")
    assert torch.equal(got[2][sel], ref[2][sel]) and torch.equal(got[3][:, sel], ref[3][:, sel]), "scales differ"
