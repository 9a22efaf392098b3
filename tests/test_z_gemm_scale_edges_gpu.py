"""The edges of the W4A4 GEMM's scale addressing (-m gpu): tail channel tiles (N % 128 = 8 / 64), partial token tiles on both
branches of S(M), more groups per rank than packed stages, the two weight segments of gate/up, q/k/v, grouped token tiles that
are not multiples of the tile, and token-scale pointers that are only 4-byte aligned (what the ABI asks for).  Every case is
bit for bit against the oracle at the dispatched split (tests/gemm_ref64.dispatch), o16 cases also within the float64 bound.
The kernel has one scale path for all of these (per-group loads through L2); the cases pin its addressing, so that a change
to how the scales are staged has to keep every edge.  The split cases also run the split-K reduction (test_z_gemm_configs_gpu
covers every split instantiation)."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import gemm_ref64 as R
from tests.test_z_gemm_configs_gpu import SPLIT_FLAG, T, _first_diff, _o16, _quant_parts, _segment

pytestmark = pytest.mark.gpu


def _auto(m, n, k, regime="random", seed=0):
    bn, split = R.dispatch(m, n, k, 0)
    _o16(R.operands(regime, m, n, k, seed=seed), 0, split, bn, f"auto {regime} {m}x{n}x{k} (BN {bn}, split {split})")


@pytest.mark.parametrize("n_tail", [8, 64])
@pytest.mark.parametrize("m", [13, 27, 57, 100])
def test_tail_channel_tiles(m, n_tail):
    """N % 128 = 8 / 64: the last channel tile holds 8 / 64 valid channels and their weight and keeper scales."""
    for j, k in enumerate((1152, 2048)):
        _auto(m, 1024 + n_tail, k, seed=10 * m + n_tail + j)


@pytest.mark.parametrize("m", [1, 7, 9, 17, 33, 65])
def test_partial_token_tiles(m):
    """The last token tile reaches the end of S(M), on both branches of scale_size (M % 16 below and at or above 8)."""
    for j, (n, k) in enumerate(((264, 1152), (1024, 2048))):
        for regime in ("random", "cancel"):
            _auto(m, n, k, regime, seed=100 * m + j)


@pytest.mark.parametrize("m,split,groups", [(9, 1, 21), (9, 4, 40), (40, 2, 13), (40, 1, 11), (100, 2, 12)])
def test_ring_wrap(m, split, groups):
    """More INT4 groups per rank than packed stages: every refill of the ring pairs its group with that group's scales."""
    bn, s = R.dispatch(m, 8, 128, SPLIT_FLAG[split])
    assert s == split
    _o16(R.operands("random", m, 264, 128 * groups, seed=m + split), SPLIT_FLAG[split], split, bn, f"wrap {m} split {split} K/128 {groups}")


@pytest.mark.parametrize("m", [7, 17, 33])
def test_gateup(m):
    """Two weight-scale segments (gate rows at n0, up rows at I + n0) per packed group and for the keeper; K with ring wrap."""
    from atom_b200 import ops
    inter = 384
    for j, k in enumerate((1152, 128 * 12)):
        t = R.operands("random", m, 2 * inter, k, seed=7 * m + j)
        got = _quant_parts(ops.dense_layer_gemm_i4_gateup_act(*[T(x) for x in t]), m)
        gate, up = O.gemm_i4_o16(*_segment(t, 0, inter)), O.gemm_i4_o16(*_segment(t, inter, 2 * inter))
        ref = _quant_parts(ops.activate_fp16_i4(T(gate), T(up)), m)
        for name, a, b in zip(("INT8 outliers", "packed INT4", "outlier scales", "norm scales"), got, ref):
            assert torch.equal(a, b), f"gate/up M {m} K {k}: {name} differ"


def _qkv_check(t, hq, hkv, tensors, what):
    from atom_b200 import ops
    q, (kk, ks), (vv, vs) = ops.dense_layer_gemm_i4_qkv(*tensors, kv_rows=hkv)
    rq = O.gemm_i4_o16(*_segment(t, 0, hq))
    q = q.cpu().numpy()
    assert np.array_equal(q.view(np.uint16), rq.view(np.uint16)), f"{what}: q {_first_diff(q, rq)}"
    for name, (d, ds), (lo, hi) in (("k", (kk, ks), (hq, hq + hkv)), ("v", (vv, vs), (hq + hkv, hq + 2 * hkv))):
        rd, rds = O.gemm_i4_o4(*_segment(t, lo, hi))
        assert np.array_equal(ds.cpu().numpy().view(np.uint16), rds.view(np.uint16)), f"{what}: {name} (scale, zero)"
        assert np.array_equal(d.cpu().numpy(), rd), f"{what}: {name} codes"


@pytest.mark.parametrize("m", [7, 9, 65])
def test_qkv(m):
    hq, hkv = 256, 128
    t = R.operands("random", m, hq + 2 * hkv, 1408, seed=3 * m)
    _qkv_check(t, hq, hkv, [T(x) for x in t], f"qkv M {m}")


def _offset4(x):
    """x (fp16) copied into a view that starts 4 bytes past a 16-byte boundary."""
    buf = torch.zeros(x.numel() + 8, dtype=torch.float16, device="cuda:0")
    v = buf[2:2 + x.numel()].view(x.shape)
    v.copy_(x)
    assert v.data_ptr() % 16 == 4
    return v


@pytest.mark.parametrize("which", ["a_scale", "a_keeper_scale", "both"])
@pytest.mark.parametrize("m", [9, 13, 57])
def test_token_scales_4_byte_aligned(m, which):
    """Token-scale pointers that are 4- but not 16-byte aligned (all the ABI asks for), for o16 and for q/k/v.  The kernel
    reads them on its only path; a staging that needs 16-byte alignment must keep a path for these."""
    from atom_b200 import ops
    n, k = 264, 128 * 12
    t = R.operands("random", m, n, k, seed=m)
    x = [T(a) for a in t]
    if which in ("a_scale", "both"):
        x[2] = _offset4(x[2])
    if which in ("a_keeper_scale", "both"):
        x[6] = _offset4(x[6])
    bn, split = R.dispatch(m, n, k, 0)
    d = ops.dense_layer_gemm_i4_fp16(*x).cpu().numpy()
    ref = O.gemm_i4_o16(*t, ksplit=split)
    assert np.array_equal(d.view(np.uint16), ref.view(np.uint16)), f"{which} M {m}: {_first_diff(d, ref)}"
    hq, hkv = 256, 128
    tq = R.operands("random", m, hq + 2 * hkv, k, seed=m + 1)
    xq = [T(a) for a in tq]
    xq[2], xq[6] = _offset4(xq[2]), _offset4(xq[6])
    _qkv_check(tq, hq, hkv, xq, f"qkv {which} M {m}")


@pytest.mark.parametrize("bn", [16, 32, 64])
def test_grouped_segments(bn):
    """Grouped o16 over a hand-made tile table: segments of 1 .. BN rows (not multiples of BN), an empty tile, a tail channel
    tile (N % 128 = 8) and ring wrap.  Each valid row equals the oracle with its expert's weights."""
    from atom_b200 import ops
    e, n, k = 3, 264, 128 * 11
    segs = [(0, 5), (2, bn), (1, bn), (1, 3), (0, 0), (2, bn - 1), (0, 1)]          # (expert, valid rows) per token tile
    rows_cap = len(segs) * bn
    ta = R.operands("random", rows_cap, 8, k, seed=bn)                               # activations (its weights unused)
    tw = [R.operands("random", 8, n, k, seed=100 + bn + x) for x in range(e)]       # per-expert weights (activations unused)
    a, _, a_s, _, ak, _, aks, _ = ta
    w4 = np.stack([w[1] for w in tw]); s4 = np.stack([w[3] for w in tw])
    w8 = np.stack([w[5] for w in tw]); s8 = np.stack([w[7] for w in tw])
    tiles = np.array([[ex, i * bn, v, 0] for i, (ex, v) in enumerate(segs)], np.int32)
    x = (T(ak), T(a), T(aks), T(a_s))
    y = ops.dense_layer_gemm_i4_fp16_grouped(x, T(w4), T(s4), T(w8), T(s8), T(tiles), bn).cpu().numpy()
    for i, (ex, v) in enumerate(segs):
        if v == 0:
            continue
        rows = list(range(i * bn, i * bn + v))
        ref = O.gemm_i4_o16(a, w4[ex], a_s, s4[ex], ak, w8[ex], aks, s8[ex], rows=rows)
        got = y[rows]
        assert np.array_equal(got.view(np.uint16), ref.view(np.uint16)), f"BN {bn} tile {i}: {_first_diff(got, ref)}"
