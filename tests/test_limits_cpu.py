"""CPU checks that keep tests/test_z_limits_gpu.py at the edges the entry points accept: the limits are read from the CUDA sources
and compared with the edge constants of the GPU file, so raising a limit fails here until the edge tests follow it.  And the
oracle's reorder and rmsnorm against a numpy restatement at hidden sizes where reorder indices reach past 32767 (read as u16, as
the kernels read them), with the dequantisation bound of the GPU file held on the oracle's output."""
import os
import re

import numpy as np
import pytest

from oracle import oracle as O
from tests import test_z_limits_gpu as L

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "atom_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _const(name, header):
    m = re.search(r"\b" + name + r"\s*=\s*(\d+)", _src(header))
    assert m, f"{name} not found in {header}"
    return int(m.group(1))


def _entry(name):
    """The body of the C ABI entry point `name` in atom_b200.cu."""
    src = _src("atom_b200.cu")
    start = src.index(f"int {name}(")
    return src[start:src.index("\n}\n", start)]


def _bound(body, pattern):
    m = re.search(pattern, body)
    assert m, pattern
    return int(m.group(1))


def test_vocabulary_edges_follow_the_sampler_limits():
    cluster, slice_max = _const("SAMPLE_MAX_CLUSTER", "sample_kernels.cuh"), _const("SAMPLE_SLICE_MAX", "sample_kernels.cuh")
    vmax = cluster * slice_max
    assert max(L.SAMPLE_VOCABS) == vmax and L.SAMPLE_VOCAB_REJECTED == vmax + 1
    assert max(L.BEAM_VOCABS) == vmax
    assert {slice_max, slice_max + 1} <= set(L.SAMPLE_VOCABS)        # one full slice, and the first two-CTA row
    assert {L.cluster(v)[0] for v in L.SAMPLE_VOCABS} >= {1, 2, cluster - 3, cluster}
    # the slice rule restated in the GPU file is the one the kernels use
    m = re.search(r"inline int sample_slice\(int V\) \{ const int c = sample_cluster\(V\); return \(\(V \+ c - 1\) / c \+ 7\) & ~7; \}",
                  _src("sample_kernels.cuh"))
    assert m, "sample_slice changed: update cluster() in test_z_limits_gpu.py"
    assert re.search(r"inline int sample_cluster\(int V\) \{ return \(V \+ SAMPLE_SLICE_MAX - 1\) / SAMPLE_SLICE_MAX; \}",
                     _src("sample_kernels.cuh"))
    for v in L.SAMPLE_VOCABS:
        c, s = L.cluster(v)
        assert 1 <= c <= cluster and s % 8 == 0 and s <= slice_max and (c - 1) * s < v <= c * s, v


def test_beam_edges_follow_the_beam_limits():
    assert L.BEAM_WIDTH == _const("BEAM_MAX_WIDTH", "beam_kernels.cuh")
    assert L.BEAM_STOPS == _const("BEAM_MAX_STOP", "beam_kernels.cuh")
    assert min(L.BEAM_SMALL_VOCABS) < L.BEAM_WIDTH < max(L.BEAM_SMALL_VOCABS)


def test_hidden_edges_follow_the_quantiser_limits():
    quant = _bound(_entry("quant_check"), r"hidden % 128 == 0 && hidden <= (\d+)")
    assert max(L.REORDER_HIDDEN) == quant and L.QUANT_HIDDEN_REJECTED == quant + 128
    for name in ("atom_rmsnorm_fp16_i4", "atom_add_rmsnorm_fp16_i4"):
        assert max(L.RMSNORM_HIDDEN) == _bound(_entry(name), r"ATOM_REQUIRE\(hidden_dim <= (\d+),")
    assert L.RMSNORM_HIDDEN_REJECTED == max(L.RMSNORM_HIDDEN) + 128
    assert L.HIDDEN_TOO_SMALL == 256 - 128
    assert any(32768 < h < 65536 and h % 32768 for h in L.REORDER_HIDDEN)    # u16 indices where int16 would not alias
    # the rmsnorm scalar path (hidden / 128 not a multiple of 8) with more than 16 groups per row
    assert any((h // 128) % 8 and h // 128 > 16 for h in L.RMSNORM_HIDDEN)


def test_moe_edges_follow_the_moe_limits():
    experts, topk = _const("MOE_MAX_EXPERTS", "moe_kernels.cuh"), _const("MOE_MAX_TOPK", "moe_kernels.cuh")
    assert L.MOE_EXPERTS == experts and L.MOE_TOPK == topk and L.MOE_TOPK_REJECTED == topk + 1
    assert max(e for e, _ in L.ROUTE_EXPERTS_TOPK) == experts and max(k for _, k in L.ROUTE_EXPERTS_TOPK) == topk
    assert (1, 1) in L.ROUTE_EXPERTS_TOPK and (topk, topk) in L.ROUTE_EXPERTS_TOPK
    assert max(L.ROUTE_HIDDEN) == _bound(_entry("atom_moe_route_f16"), r"hidden_dim <= (\d+)")


def test_verify_edge_follows_the_chunk_limit():
    n = _bound(_entry("atom_batch_verify_gqa_i4"), r"nchunks >= 1 && nchunks <= (\d+)")
    assert L.VERIFY_NCHUNKS == n and L.VERIFY_NCHUNKS_REJECTED == n + 1


# ------------------------------------------------------------------------------------------------ the oracle at u16 indices
def _roundf(v):
    """C roundf (half away from zero) of FP32 values, NaN -> 0 as cvt.rzi.s32.f32 gives."""
    v = v.astype(np.float64)
    return np.where(np.isnan(v), 0.0, np.sign(v) * np.floor(np.abs(v) + 0.5))


def _quantise_np(x):
    """The shared quantiser tail on FP32 rows x [m, h] (already in quantiser order): codes [m, h] and FP16 scales [m, h / 128]."""
    m, h = x.shape
    g = h // 128
    xg = x.reshape(m, g, 128)
    d = np.where(np.arange(g) == g - 1, np.float32(127), np.float32(7)).astype(np.float32)
    s = (np.abs(xg).max(-1) / d).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = (np.float32(1) / s).astype(np.float32)
        q = _roundf((xg * r[..., None]).astype(np.float32))
    lo, hi = np.where(d == 127, -128, -8), np.where(d == 127, 127, 7)
    q = np.clip(q, lo[None, :, None], hi[None, :, None])
    return q.reshape(m, h).astype(np.int32), s.astype(np.float16)


def _oracle_codes(out, m):
    o8, o4, s8, s4 = out
    q = np.concatenate([O.unpack_int4(o4).astype(np.int32), o8.astype(np.int32)], 1)
    s = np.concatenate([O.a_scale_from_layout(s4, m).T, O.a_scale_from_layout(s8[None], m).T], 1)
    return q, s


def _assert_same(out, ref, m, what):
    q, s = _oracle_codes(out, m)
    rq, rs = ref
    assert np.array_equal(q, rq), f"{what}: {int((q != rq).sum())} codes differ"
    assert np.array_equal(s.view(np.uint16), rs.view(np.uint16)), f"{what}: scales differ"


def _inputs(h, m, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((m, h)) * np.where(rng.random((1, h)) > 0.97, 12.0, 1.0)).astype(np.float16)
    return rng, x, rng.permutation(h).astype(np.int16)      # int16 bits of the u16 indices, as a model stores them


@pytest.mark.parametrize("h", [4096, 40960, 65536])
def test_oracle_reorder_reads_indices_as_u16(h):
    m = 5
    _, x, idx = _inputs(h, m, h)
    out = O.reorder_fp16_i4(x, idx)
    cols = idx.view(np.uint16)
    _assert_same(out, _quantise_np(x[:, cols].astype(np.float32)), m, f"reorder h={h}")
    L.dequant_check([_Host(a) for a in out], x[:, cols].astype(np.float64), 0.0, f"oracle reorder h={h}")


def _rmsnorm_np(x, w, cols, eps):
    """rmsnorm_fp16_i4's row before the quantiser: the sum of squares in the kernel's order (128 threads fold h / 128 contiguous
    squares each -- exact FP16 squares, so fmaf is one FP32 add -- then halving trees), rstd = 1 / sqrt, the FP32 products, FP16."""
    m, h = x.shape
    ept = h // 128
    x32 = x.astype(np.float32)
    sq = (x32 * x32).reshape(m, 128, ept)
    part = np.zeros((m, 128), np.float32)
    for i in range(ept):
        part = (part + sq[:, :, i]).astype(np.float32)
    for s in (64, 32, 16, 8, 4, 2, 1):
        part = (part[:, :s] + part[:, s:2 * s]).astype(np.float32)
    rstd = (np.float32(1) / np.sqrt((part[:, 0] / np.float32(h) + np.float32(eps)).astype(np.float32))).astype(np.float32)
    y = ((x32[:, cols] * w.astype(np.float32)[cols]).astype(np.float32) * rstd[:, None]).astype(np.float32)
    return y.astype(np.float16).astype(np.float32)


@pytest.mark.parametrize("h", [4096, 2176, 32768])
def test_oracle_rmsnorm_reads_indices_as_u16(h):
    m = 5
    rng, x, idx = _inputs(h, m, h + 1)
    w = (1 + 0.2 * rng.standard_normal(h)).astype(np.float16)
    if h == 32768:          # indices >= 32768 are out of this row's range: the largest index is 32767, the u16 view is the same
        assert idx.view(np.uint16).max() == h - 1
    out = O.rmsnorm_fp16_i4(x, w, idx, 1e-5)
    cols = idx.view(np.uint16)
    _assert_same(out, _quantise_np(_rmsnorm_np(x, w, cols, 1e-5)), m, f"rmsnorm h={h}")
    L.dequant_check([_Host(a) for a in out], L._rms64(x, w, cols, 1e-5), L._rms_rel(h), f"oracle rmsnorm h={h}", fp16_input=True)


def test_oracle_activate_within_the_dequantisation_bound():
    for h in (256, 2176, 40960):
        rng = np.random.default_rng(h)
        a = (rng.standard_normal((3, h)) * 2).astype(np.float16)
        b = (rng.standard_normal((3, h)) * 2).astype(np.float16)
        b[1] = 0                                                        # an all-zero row: scales 0, codes 0
        a64, b64 = a.astype(np.float64), b.astype(np.float64)
        L.dequant_check([_Host(x) for x in O.activate_fp16_i4(a, b)], a64 / (1 + np.exp(-a64)) * b64, 16 * L.U32,
                        f"oracle activate h={h}")


def test_dequantisation_bound_catches_a_wrong_code_and_a_wrong_scale():
    """The bound has power: one code off by one step, or one scale one FP16 ulp off, fails it."""
    h, m = 2176, 3
    _, x, idx = _inputs(h, m, 9)
    cols = idx.view(np.uint16)
    X = x[:, cols].astype(np.float64)
    o8, o4, s8, s4 = O.reorder_fp16_i4(x, idx)
    q = O.unpack_int4(o4)
    j = int(np.argmax(np.abs(q[1, :128])))
    q[1, j] -= np.sign(q[1, j])
    with pytest.raises(AssertionError, match="the bound"):
        L.dequant_check([_Host(a) for a in (o8, O.pack_int4(q), s8, s4)], X, 0.0, "one code off")
    s4b = s4.copy()
    s4b[0] = (s4b[0].view(np.uint16) + 1).view(np.float16)
    with pytest.raises(AssertionError):
        L.dequant_check([_Host(a) for a in (o8, o4, s8, s4b)], X, 0.0, "one scale off")


class _Host:
    """A numpy array standing in for the device tensors dequant_check reads (it calls .cpu().numpy())."""

    def __init__(self, a):
        self.a = a

    def cpu(self):
        return self

    def numpy(self):
        return self.a
