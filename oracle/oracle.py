"""numpy front-end of the CPU oracle (oracle/atom_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of atom_oracle.c.  Imported by tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline leg; never by atom_b200/.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libatom_oracle.so")


def build(force=False):
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, "atom_oracle.c")):
        subprocess.check_call(["make", "-C", _HERE, "libatom_oracle.so"], stdout=subprocess.DEVNULL)


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
        _lib.atom_oracle_scale_index.restype = ctypes.c_int
        _lib.atom_oracle_scale_size.restype = ctypes.c_int
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _c(a, dt):
    a = np.ascontiguousarray(a)
    if a.dtype != np.dtype(dt):
        a = a.view(dt) if a.dtype.itemsize == np.dtype(dt).itemsize else a.astype(dt)
    return a


def scale_index(row):
    return lib().atom_oracle_scale_index(int(row))


def scale_size(m):
    return lib().atom_oracle_scale_size(int(m))


def _quant_outputs(m, hidden):
    ldm = scale_size(m)
    o8 = np.zeros((m, 128), np.int8)
    o4 = np.zeros((m, (hidden - 128) // 2), np.uint8)
    s8 = np.zeros((ldm,), np.float16)
    s4 = np.zeros((hidden // 128 - 1, ldm), np.float16)
    return o8, o4, s8, s4


def reorder_fp16_i4(x, idx):
    """`idx` holds 16-bit column indices read as unsigned (hidden <= 65536): an int16 array is taken bit for bit."""
    x, idx = _c(x, np.float16), _c(idx, np.uint16)
    m, h = x.shape
    o8, o4, s8, s4 = _quant_outputs(m, h)
    lib().atom_oracle_reorder_fp16_i4(_p(x), m, h, _p(idx), _p(o8), _p(o4), _p(s8), _p(s4))
    return o8, o4, s8, s4


def rmsnorm_fp16_i4(x, w, idx, eps):
    x, w, idx = _c(x, np.float16), _c(w, np.float16), _c(idx, np.uint16)
    m, h = x.shape
    o8, o4, s8, s4 = _quant_outputs(m, h)
    lib().atom_oracle_rmsnorm_fp16_i4(_p(x), _p(w), ctypes.c_float(eps), m, h, _p(idx), _p(o8), _p(o4), _p(s8), _p(s4))
    return o8, o4, s8, s4


def activate_fp16_i4(a, b):
    a, b = _c(a, np.float16), _c(b, np.float16)
    m, h = a.shape
    o8, o4, s8, s4 = _quant_outputs(m, h)
    lib().atom_oracle_activate_fp16_i4(_p(a), _p(b), m, h, _p(o8), _p(o4), _p(s8), _p(s4))
    return o8, o4, s8, s4


def _gemm_args(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale):
    a, b = _c(a, np.uint8), _c(b, np.uint8)
    a_scale, b_scale = _c(a_scale, np.float16), _c(b_scale, np.float16)
    a_keeper, b_keeper = _c(a_keeper, np.int8), _c(b_keeper, np.int8)
    a_keeper_scale, b_keeper_scale = _c(a_keeper_scale, np.float16), _c(b_keeper_scale, np.float16)
    m, n, k = a.shape[0], b.shape[0], a.shape[1] * 2 + a_keeper.shape[1]
    return (a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale), m, n, k


def split_ranges(g, ksplit):
    """The K partition of a split GEMM with g INT4 groups: rank r's groups [g_begin, g_end) of the g + 1 groups, index g
    being the INT8 keeper (gemm_i4_sm90.cuh, `per` = ceil((g + 1) / ksplit)).  Ranks past the end hold no group."""
    per = -(-(g + 1) // ksplit)
    return [(min(r * per, g + 1), min(min(r * per, g + 1) + per, g + 1)) for r in range(ksplit)]


def gemm_i4_o16(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, faithful=True, rows=None, ksplit=1):
    """D[m,n] fp16.  rows: optional int32 list of A rows to evaluate (spot checks at full size).  ksplit: the K split of the
    kernel (split_ranges; per-rank FP32 chains summed in rank order), 1 = the reference's single chain."""
    if ksplit not in (1, 2, 4, 8):
        raise ValueError(f"ksplit={ksplit}: the kernel splits K 1, 2, 4 or 8 ways")
    t, m, n, k = _gemm_args(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale)
    rows_a = None if rows is None else _c(np.asarray(rows), np.int32)
    nr = m if rows is None else len(rows_a)
    d = np.zeros((nr, n), np.float16)
    lib().atom_oracle_gemm_i4_o16(*[_p(x) for x in t], _p(d), m, n, k, int(faithful), int(ksplit), _p(rows_a), nr)
    return d


def gemm_i4_o4(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, faithful=True,
               signed_minmax=True, rows=None):
    """(codes u8 [rows, N/2], (scale, zero) f16 [rows, N/128 * 2]) of the o4 epilogue: signed min/max per 128-channel head,
    codes clamped to [0, 15].  signed_minmax=False is the reference kernel's |v| min/max with `& 0xF` (wrong for negative
    values; only for pinning this oracle to the reference's recorded outputs)."""
    t, m, n, k = _gemm_args(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale)
    rows_a = None if rows is None else _c(np.asarray(rows), np.int32)
    nr = m if rows is None else len(rows_a)
    d = np.zeros((nr, n // 2), np.uint8)
    ds = np.zeros((nr, n // 128 * 2), np.float16)
    lib().atom_oracle_gemm_i4_o4(*[_p(x) for x in t], _p(d), _p(ds), m, n, k, int(faithful), int(signed_minmax),
                                 _p(rows_a), nr)
    return d, ds


def append_kv_i4(data, param, indptr, indices, last_off, k, v, kp, vp, layer):
    """In place on data/param (numpy, layouts of kvcache.py:17-24)."""
    _, L, _, H, P, _ = data.shape
    B = len(last_off)
    lib().atom_oracle_append_kv_i4(_p(data), _p(param), _p(_c(indptr, np.int32)), _p(_c(indices, np.int32)),
                                   _p(_c(last_off, np.int32)), _p(_c(k, np.uint8)), _p(_c(v, np.uint8)),
                                   _p(_c(kp, np.float16)), _p(_c(vp, np.float16)), L, layer, H, P, B)


def init_kv_i4(data, param, indptr, indices, last_off, k, v, kp, vp, seqlen_indptr, layer):
    _, L, _, H, P, _ = data.shape
    B = len(last_off)
    lib().atom_oracle_init_kv_i4(_p(data), _p(param), _p(_c(indptr, np.int32)), _p(_c(indices, np.int32)),
                                 _p(_c(last_off, np.int32)), _p(_c(k, np.uint8)), _p(_c(v, np.uint8)),
                                 _p(_c(kp, np.float16)), _p(_c(vp, np.float16)), _p(_c(seqlen_indptr, np.int32)),
                                 L, layer, H, P, B)


def batch_decode_i4(q, data, param, indptr, indices, last_off, layer):
    q = _c(q, np.float16)
    B, H, D = q.shape
    assert D == 128
    _, L, _, H2, P, _ = data.shape
    assert H2 == H
    o = np.zeros_like(q)
    lib().atom_oracle_batch_decode_i4(_p(o), _p(q), _p(_c(data, np.uint8)), _p(_c(param, np.float16)),
                                      _p(_c(indptr, np.int32)), _p(_c(indices, np.int32)),
                                      _p(_c(last_off, np.int32)), L, layer, H, P, B)
    return o


# ----------------------------------------------------------------------------------------------
# helpers shared by tests / bench to build synthetic quantised operands (SURVEY 8d "C2 inputs")
def pack_int4(q):
    """q: int array [-8,7], last dim even -> uint8 packed low-nibble-first (Reorder.cuh:16-19)."""
    q = np.asarray(q).astype(np.int16)
    lo, hi = q[..., 0::2] & 0xF, q[..., 1::2] & 0xF
    return (lo | (hi << 4)).astype(np.uint8)


def unpack_int4(p):
    p = np.asarray(p, np.uint8)
    lo = (p & 0xF).astype(np.int8)
    hi = (p >> 4).astype(np.int8)
    lo = np.where(lo >= 8, lo - 16, lo)
    hi = np.where(hi >= 8, hi - 16, hi)
    out = np.empty(p.shape[:-1] + (p.shape[-1] * 2,), np.int8)
    out[..., 0::2], out[..., 1::2] = lo, hi
    return out


def a_scale_to_layout(scales):
    """scales: [G, M] float -> [G, S(M)] fp16 in the ldmatrix-replicated layout (x4), zeros elsewhere."""
    scales = np.asarray(scales)
    g, m = scales.shape
    out = np.zeros((g, scale_size(m)), np.float16)
    for r in range(m):
        si = scale_index(r)
        for j in range(4):
            out[:, si + 2 * j] = scales[:, r]
    return out


def a_scale_from_layout(layout, m):
    layout = np.asarray(layout)
    idx = [scale_index(r) for r in range(m)]
    return layout[..., idx]


def make_gemm_inputs(m, n, k, seed=0xabcdabcd987 & 0x7fffffff, pair_shared=True):
    """Synthetic random-quantised GEMM operands in the reference layouts (K includes the keeper)."""
    rng = np.random.default_rng(seed)
    g = k // 128 - 1
    a = pack_int4(rng.integers(-8, 8, (m, k - 128)))
    b = pack_int4(rng.integers(-8, 8, (n, k - 128)))
    ak = rng.integers(-128, 128, (m, 128)).astype(np.int8)
    bk = rng.integers(-128, 128, (n, 128)).astype(np.int8)
    sa = (np.abs(rng.standard_normal((g + 1, m))) * 0.2 + 0.3) / 7.0
    a_scale = a_scale_to_layout(sa[:g])
    # outlier channels are ~30x larger than normal ones (that is why they are kept in INT8)
    a_keeper_scale = a_scale_to_layout(rng.uniform(8.0, 24.0, (1, m)) / 127.0)[0]
    if pair_shared:
        sb = np.repeat(0.01 * (1.0 + rng.random((g + 1, n // 2))), 2, axis=1)
    else:
        sb = 0.01 * (1.0 + rng.random((g + 1, n)))
    b_scale = sb[:g].astype(np.float16)
    b_keeper_scale = (sb[g] * 7.0 / 127.0).astype(np.float16)
    return a, b, a_scale, b_scale, ak, bk, a_keeper_scale, b_keeper_scale
