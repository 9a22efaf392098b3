"""Operator API -- mirrors /root/reference/e2e/punica-atom/punica/ops/__init__.py (names, argument order,
output allocation and return tuples) on top of the sm_90a kernels in libatom_b200.so.

Differences from the reference (all widening, none changes a result):
  * kernels run on torch's current CUDA stream (the reference uses the legacy default stream);
  * hidden_dim is any multiple of 128 (reference: 4096 for reorder/rmsnorm, 11008 for activate);
  * errors raise RuntimeError with the library's message instead of being silently ignored.
"""
import torch

from . import _lib

__all__ = [
    "batch_decode_i4", "append_kv_i4", "init_kv_i4", "activate_fp16_i4", "dense_layer_gemm_i4_fp16",
    "dense_layer_gemm_i4_o4", "rmsnorm_fp16_i4", "reorder_fp16_i4", "scale_size",
]

GEMM_AUTO, GEMM_NO_SPLITK, GEMM_FORCE_TALL, GEMM_FORCE_SKINNY = 0, 1, 2, 4
GEMM_SPLITK2, GEMM_SPLITK4, GEMM_SPLITK8 = 16, 32, 64
GEMM_FORCE_WIDE, GEMM_NO_WIDE = 512, 1024   # kernel selectors of earlier versions: accepted and ignored
GEMM_LEGACY_TALL = 256    # kernel selector of earlier versions: accepted and ignored
GEMM_LEGACY_SKINNY = 128  # kernel selector of earlier versions: accepted and ignored


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _req_cuda(*ts):
    for t in ts:
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise RuntimeError("atom_b200.ops: all tensors must live on a CUDA device (there is no CPU path)")
        if not t.is_contiguous():
            raise RuntimeError("atom_b200.ops: tensors must be contiguous")


def _req_width(what, **named):
    """Element-width checks (the C ABI takes raw pointers: a float32 tensor where float16 is meant would be silently
    misread).  Packed INT4 / INT8 operands may be int8 or uint8 views, so only the width is fixed for them."""
    for spec, t in named.items():
        name, width = spec.rsplit("_", 1)
        is_f16 = name.startswith("f16_")
        name = name[4:] if is_f16 else name
        ok = isinstance(t, torch.Tensor) and t.element_size() == int(width) and (not is_f16 or t.dtype == torch.float16)
        if not ok:
            raise RuntimeError(f"atom_b200.ops.{what}: `{name}` must be a tensor of {width}-byte elements"
                               f"{' (float16)' if is_f16 else ''}, got {getattr(t, 'dtype', type(t))}")


def scale_size(x):
    """ops/__init__.py:137-138"""
    return ((x) // 16 * 64 + 64 - (1 - (x % 16) // 8) * (8 - (x % 8)) * 8)


def _quant_outputs(bs, hidden_dim, device):
    group_size = 128
    o_outlier = torch.empty((bs, group_size), dtype=torch.int8, device=device)
    o_norms = torch.empty((bs, (hidden_dim - group_size) // 2), dtype=torch.int8, device=device)
    outlier_scales = torch.empty((scale_size(bs),), dtype=torch.float16, device=device)
    norm_scales = torch.empty((hidden_dim // group_size - 1, scale_size(bs)), dtype=torch.float16, device=device)
    return o_outlier, o_norms, outlier_scales, norm_scales


def reorder_fp16_i4(hidden_states, reorder_index):
    """ops/__init__.py:200-219"""
    _req_width("reorder_fp16_i4", f16_hidden_states_2=hidden_states, reorder_index_2=reorder_index)
    _req_cuda(hidden_states, reorder_index)
    bs, hidden_dim = hidden_states.shape
    out = _quant_outputs(bs, hidden_dim, hidden_states.device)
    with torch.cuda.device(hidden_states.device):
        _lib.check(_lib.lib().atom_reorder_fp16_i4(hidden_states.data_ptr(), reorder_index.data_ptr(), bs, hidden_dim,
                                                   out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
                                                   out[3].data_ptr(), _stream(hidden_states)), "reorder_fp16_i4")
    return out


def rmsnorm_fp16_i4(hidden_states, weight, reorder_index, eps):
    """ops/__init__.py:179-198.  `weight` may be fp32 (LlamaRMSNormInt4 keeps torch.ones fp32, llama.py:237); the
    reference reinterprets its storage as half -- here it is converted, which is what was meant."""
    if isinstance(weight, torch.Tensor) and weight.dtype != torch.float16:
        weight = weight.to(torch.float16)
    _req_width("rmsnorm_fp16_i4", f16_hidden_states_2=hidden_states, f16_weight_2=weight, reorder_index_2=reorder_index)
    _req_cuda(hidden_states, weight, reorder_index)
    bs, hidden_dim = hidden_states.shape
    out = _quant_outputs(bs, hidden_dim, hidden_states.device)
    with torch.cuda.device(hidden_states.device):
        _lib.check(_lib.lib().atom_rmsnorm_fp16_i4(hidden_states.data_ptr(), weight.data_ptr(), float(eps),
                                                   reorder_index.data_ptr(), bs, hidden_dim, out[0].data_ptr(),
                                                   out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(),
                                                   _stream(hidden_states)), "rmsnorm_fp16_i4")
    return out


def add_rmsnorm_fp16_i4(hidden_states, residual, weight, reorder_index, eps):
    """EXTENSION: (residual + hidden_states) and rmsnorm_fp16_i4 of the sum in one launch.  Returns (sum, 4-tuple);
    both bit-identical to `s = residual + hidden_states; rmsnorm_fp16_i4(s, ...)`."""
    if isinstance(weight, torch.Tensor) and weight.dtype != torch.float16:
        weight = weight.to(torch.float16)
    _req_width("add_rmsnorm_fp16_i4", f16_hidden_states_2=hidden_states, f16_residual_2=residual, f16_weight_2=weight,
               reorder_index_2=reorder_index)
    _req_cuda(hidden_states, residual, weight, reorder_index)
    if hidden_states.shape != residual.shape:
        raise RuntimeError("add_rmsnorm_fp16_i4: hidden_states and residual must have the same shape")
    bs, hidden_dim = hidden_states.shape
    out = _quant_outputs(bs, hidden_dim, hidden_states.device)
    s = torch.empty_like(hidden_states)
    with torch.cuda.device(hidden_states.device):
        _lib.check(_lib.lib().atom_add_rmsnorm_fp16_i4(hidden_states.data_ptr(), residual.data_ptr(), s.data_ptr(), weight.data_ptr(),
                                                       float(eps), reorder_index.data_ptr(), bs, hidden_dim, out[0].data_ptr(),
                                                       out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(),
                                                       _stream(hidden_states)), "add_rmsnorm_fp16_i4")
    return s, out


def activate_fp16_i4(a, b):
    """ops/__init__.py:141-157"""
    _req_width("activate_fp16_i4", f16_a_2=a, f16_b_2=b)
    _req_cuda(a, b)
    bs, hidden_dim = a.shape
    out = _quant_outputs(bs, hidden_dim, a.device)
    with torch.cuda.device(a.device):
        _lib.check(_lib.lib().atom_activate_fp16_i4(a.data_ptr(), b.data_ptr(), bs, hidden_dim, out[0].data_ptr(),
                                                    out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(),
                                                    _stream(a)), "activate_fp16_i4")
    return out


def dense_layer_gemm_i4_fp16(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, flags=GEMM_AUTO):
    """ops/__init__.py:160-168; dims as punica_ops.cc:236-237 (K = a.size(1)*2 + a_keeper.size(1))."""
    _req_width("dense_layer_gemm_i4_fp16", a_1=a, b_1=b, f16_a_scale_2=a_scale, f16_b_scale_2=b_scale, a_keeper_1=a_keeper,
               b_keeper_1=b_keeper, f16_a_keeper_scale_2=a_keeper_scale, f16_b_keeper_scale_2=b_keeper_scale)
    _req_cuda(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale)
    m, n = a.size(0), b.size(0)
    k = a.size(1) * 2 + a_keeper.size(1)
    d = torch.empty((m, n), dtype=torch.float16, device=a.device)
    with torch.cuda.device(a.device):
        _lib.check(_lib.lib().atom_gemm_i4_o16(a.data_ptr(), b.data_ptr(), a_scale.data_ptr(), b_scale.data_ptr(),
                                               a_keeper.data_ptr(), b_keeper.data_ptr(), a_keeper_scale.data_ptr(),
                                               b_keeper_scale.data_ptr(), d.data_ptr(), m, n, k, flags, _stream(a)),
                   "dense_layer_gemm_i4_fp16")
    return d


class ArHandle:
    """What the fused all-reduce entry points need of a comm.PushAllReduce: the device table of every rank's receive buffer, the
    local call-counter block, the slot size, and this rank's place in the group."""
    __slots__ = ("peer_ptrs", "state", "slot", "rank", "world")

    def __init__(self, peer_ptrs, state, slot, rank, world):
        self.peer_ptrs, self.state, self.slot, self.rank, self.world = int(peer_ptrs), state, int(slot), int(rank), int(world)


class PendingAllReduce:
    """Result of dense_layer_gemm_i4_fp16_push: the partial products sit in the receive buffers of all ranks; only
    reduce_add_rmsnorm_fp16_i4 (the very next consumer) can turn them into the all-reduced tensor."""
    __slots__ = ("ar", "shape", "device")

    def __init__(self, ar, shape, device):
        self.ar, self.shape, self.device = ar, tuple(shape), device


def dense_layer_gemm_i4_fp16_push(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, ar, flags=GEMM_AUTO):
    """EXTENSION (tensor parallelism, decode batches M <= 64): dense_layer_gemm_i4_fp16 of a row-parallel shard whose epilogue pushes
    the FP16 partial into every rank's all-reduce receive buffer (csrc/comm_kernels.cuh).  Returns a PendingAllReduce."""
    _req_width("dense_layer_gemm_i4_fp16_push", a_1=a, b_1=b, f16_a_scale_2=a_scale, f16_b_scale_2=b_scale, a_keeper_1=a_keeper,
               b_keeper_1=b_keeper, f16_a_keeper_scale_2=a_keeper_scale, f16_b_keeper_scale_2=b_keeper_scale)
    _req_cuda(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale)
    m, n = a.size(0), b.size(0)
    k = a.size(1) * 2 + a_keeper.size(1)
    with torch.cuda.device(a.device):
        _lib.check(_lib.lib().atom_gemm_i4_o16_push(a.data_ptr(), b.data_ptr(), a_scale.data_ptr(), b_scale.data_ptr(),
                                                    a_keeper.data_ptr(), b_keeper.data_ptr(), a_keeper_scale.data_ptr(),
                                                    b_keeper_scale.data_ptr(), ar.peer_ptrs, ar.state.data_ptr(), ar.slot, ar.rank,
                                                    ar.world, m, n, k, flags, _stream(a)), "dense_layer_gemm_i4_fp16_push")
    return PendingAllReduce(ar, (m, n), a.device)


def reduce_add_rmsnorm_fp16_i4(pending, residual, weight, reorder_index, eps):
    """EXTENSION: add_rmsnorm_fp16_i4 whose `hidden_states` is the all-reduce of a PendingAllReduce, formed while the row is loaded.
    Returns (sum, 4-tuple), bit-identical to all-reducing first (rank-order FP32 sum, FP16 result) and calling add_rmsnorm_fp16_i4."""
    if isinstance(weight, torch.Tensor) and weight.dtype != torch.float16:
        weight = weight.to(torch.float16)
    _req_width("reduce_add_rmsnorm_fp16_i4", f16_residual_2=residual, f16_weight_2=weight, reorder_index_2=reorder_index)
    _req_cuda(residual, weight, reorder_index)
    if tuple(residual.shape) != pending.shape:
        raise RuntimeError("reduce_add_rmsnorm_fp16_i4: residual must have the shape of the pending all-reduce")
    bs, hidden_dim = residual.shape
    out = _quant_outputs(bs, hidden_dim, residual.device)
    s = torch.empty_like(residual)
    ar = pending.ar
    with torch.cuda.device(residual.device):
        _lib.check(_lib.lib().atom_reduce_add_rmsnorm_fp16_i4(ar.peer_ptrs, ar.state.data_ptr(), ar.slot, ar.rank, ar.world,
                                                              residual.data_ptr(), s.data_ptr(), weight.data_ptr(), float(eps),
                                                              reorder_index.data_ptr(), bs, hidden_dim, out[0].data_ptr(),
                                                              out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(),
                                                              _stream(residual)), "reduce_add_rmsnorm_fp16_i4")
    return s, out


def dense_layer_gemm_i4_o4(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, flags=GEMM_AUTO):
    """ops/__init__.py:171-176"""
    _req_width("dense_layer_gemm_i4_o4", a_1=a, b_1=b, f16_a_scale_2=a_scale, f16_b_scale_2=b_scale, a_keeper_1=a_keeper,
               b_keeper_1=b_keeper, f16_a_keeper_scale_2=a_keeper_scale, f16_b_keeper_scale_2=b_keeper_scale)
    _req_cuda(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale)
    m, n = a.size(0), b.size(0)
    k = a.size(1) * 2 + a_keeper.size(1)
    d = torch.empty((m, n // 2), dtype=torch.uint8, device=a.device)
    assert n % 128 == 0
    d_scale = torch.empty((m, n // 128 * 2), dtype=torch.float16, device=a.device)
    with torch.cuda.device(a.device):
        _lib.check(_lib.lib().atom_gemm_i4_o4(a.data_ptr(), b.data_ptr(), a_scale.data_ptr(), b_scale.data_ptr(),
                                              a_keeper.data_ptr(), b_keeper.data_ptr(), a_keeper_scale.data_ptr(),
                                              b_keeper_scale.data_ptr(), d.data_ptr(), d_scale.data_ptr(), m, n, k,
                                              flags, _stream(a)), "dense_layer_gemm_i4_o4")
    return d, d_scale


def dense_layer_gemm_i4_qkv(a, b_qkv, a_scale, b_scale_qkv, a_keeper, b_keeper_qkv, a_keeper_scale, b_keeper_scale_qkv, flags=GEMM_AUTO,
                            kv_rows=None):
    """EXTENSION: q (fp16), k and v (o4) projections of one input over row-concatenated weights [3H, ...] in one launch for
    decode batches.  Returns (q, (k, k_scale), (v, v_scale)), bit-identical to the three separate operator calls.
    kv_rows (grouped-query attention): rows of the k part (= of the v part) of `b_qkv`; the q part is the rest.  None = three
    equal parts."""
    _req_width("dense_layer_gemm_i4_qkv", a_1=a, b_qkv_1=b_qkv, f16_a_scale_2=a_scale, f16_b_scale_qkv_2=b_scale_qkv, a_keeper_1=a_keeper,
               b_keeper_qkv_1=b_keeper_qkv, f16_a_keeper_scale_2=a_keeper_scale, f16_b_keeper_scale_qkv_2=b_keeper_scale_qkv)
    _req_cuda(a, b_qkv, a_scale, b_scale_qkv, a_keeper, b_keeper_qkv, a_keeper_scale, b_keeper_scale_qkv)
    m, n3 = a.size(0), b_qkv.size(0)
    k = a.size(1) * 2 + a_keeper.size(1)
    kv_rows = n3 // 3 if kv_rows is None else int(kv_rows)
    hq = n3 - 2 * kv_rows
    if kv_rows <= 0 or hq <= 0 or kv_rows % 128 or hq % 128 or b_scale_qkv.numel() < (k // 128 - 1) * n3 or b_keeper_qkv.size(0) != n3:
        raise RuntimeError("dense_layer_gemm_i4_qkv: weights must be the row concatenation [q; k; v] with kv_rows rows of k and of v, "
                           "q and kv_rows multiples of 128")
    q = torch.empty((m, hq), dtype=torch.float16, device=a.device)
    kk = torch.empty((m, kv_rows // 2), dtype=torch.uint8, device=a.device)
    vv = torch.empty((m, kv_rows // 2), dtype=torch.uint8, device=a.device)
    ks = torch.empty((m, kv_rows // 128 * 2), dtype=torch.float16, device=a.device)
    vs = torch.empty((m, kv_rows // 128 * 2), dtype=torch.float16, device=a.device)
    with torch.cuda.device(a.device):
        _lib.check(_lib.lib().atom_gemm_i4_qkv_gqa(a.data_ptr(), b_qkv.data_ptr(), a_scale.data_ptr(), b_scale_qkv.data_ptr(),
                                                   a_keeper.data_ptr(), b_keeper_qkv.data_ptr(), a_keeper_scale.data_ptr(),
                                                   b_keeper_scale_qkv.data_ptr(), q.data_ptr(), kk.data_ptr(), ks.data_ptr(), vv.data_ptr(),
                                                   vs.data_ptr(), m, hq, kv_rows, k, flags, _stream(a)), "dense_layer_gemm_i4_qkv")
    return q, (kk, ks), (vv, vs)


def dense_layer_gemm_i4_gateup_act(a, b_gu, a_scale, b_scale_gu, a_keeper, b_keeper_gu, a_keeper_scale, b_keeper_scale_gu, flags=GEMM_AUTO):
    """EXTENSION: activate_fp16_i4(gate_proj(x), up_proj(x)) in one launch over row-concatenated weights [2I, ...] (decode
    batches, M <= 64).  Returns the activation 4-tuple, bit-identical to the three separate operator calls."""
    _req_width("dense_layer_gemm_i4_gateup_act", a_1=a, b_gu_1=b_gu, f16_a_scale_2=a_scale, f16_b_scale_gu_2=b_scale_gu, a_keeper_1=a_keeper,
               b_keeper_gu_1=b_keeper_gu, f16_a_keeper_scale_2=a_keeper_scale, f16_b_keeper_scale_gu_2=b_keeper_scale_gu)
    _req_cuda(a, b_gu, a_scale, b_scale_gu, a_keeper, b_keeper_gu, a_keeper_scale, b_keeper_scale_gu)
    m, n2 = a.size(0), b_gu.size(0)
    k = a.size(1) * 2 + a_keeper.size(1)
    if n2 % 256 != 0 or b_keeper_gu.size(0) != n2:
        raise RuntimeError("dense_layer_gemm_i4_gateup_act: weights must be the row concatenation [gate; up] with I % 128 == 0")
    inter = n2 // 2
    out = _quant_outputs(m, inter, a.device)
    with torch.cuda.device(a.device):
        _lib.check(_lib.lib().atom_gemm_i4_gateup_act(a.data_ptr(), b_gu.data_ptr(), a_scale.data_ptr(), b_scale_gu.data_ptr(),
                                                      a_keeper.data_ptr(), b_keeper_gu.data_ptr(), a_keeper_scale.data_ptr(),
                                                      b_keeper_scale_gu.data_ptr(), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
                                                      out[3].data_ptr(), m, inter, k, flags, _stream(a)), "dense_layer_gemm_i4_gateup_act")
    return out


def _kv_dims(kv):
    # CHECK_DIM(6, kv_data) etc., punica_ops.cc:93-112
    if kv.data.dim() != 6 or kv.param.dim() != 6:
        raise RuntimeError("kv_data / kv_param must be 6-D [pages, L, 2, H, P, D]")
    if kv.data.dtype != torch.uint8 or kv.param.dtype != torch.float16:
        raise RuntimeError("kv_data must be uint8 and kv_param float16")
    if kv.data.size(5) * 2 != 128:
        raise RuntimeError("head_dim must be 128")
    return kv.data.size(1), kv.data.size(3), kv.data.size(4)


def batch_decode_i4(q, kv, layer_idx, rope_theta=10000.0, kv_split=0):
    """ops/__init__.py:21-32.  EXTENSION (grouped-query attention): q may hold G = 2, 4 or 8 query heads per head of the cache
    (query head h attends KV head h // G), and `rope_theta` is the RoPE base; one query head per KV head at the default base
    is the reference's operator.  EXTENSION (split-KV): `kv_split` spreads each sequence's pages over a cluster of that many
    CTAs -- 0 = automatic (`decode_kv_split`: only grids of fewer (sequence, KV head) pairs than SMs split), 1 = never,
    2 / 4 / 8 = forced; other values raise.  EXTENSION (shared-prefix decode): when `kv` carries prefix groups (a
    BatchedKvCacheInt4 over forked sequences) and `decode_cascade` picks it, kv_split=0 runs the cascade: each group's shared
    pages are attended once per KV head for all its members on tensor cores, then each row's private pages by the decode kernel;
    rows outside the groups get exactly what kv_split=1 gives them."""
    _req_cuda(q, kv.data, kv.param, kv.indptr, kv.indicies, kv.last_page_offset)
    L, H, P = _kv_dims(kv)
    if q.dim() != 3 or q.size(2) != 128 or kv.indptr.size(0) != q.size(0) + 1 or kv.last_page_offset.size(0) != q.size(0):
        raise RuntimeError("batch_decode_i4: shape mismatch")
    o = torch.empty(q.shape, dtype=q.dtype, device=q.device)
    groups = getattr(kv, "groups", None)
    if groups and kv_split == 0:
        sms = torch.cuda.get_device_properties(q.device).multi_processor_count
        if decode_cascade(groups, q.size(0), P, H, q.size(1) // H, sms):
            return _batch_decode_shared(o, q, kv, groups, L, H, P, layer_idx, rope_theta, sms)
    with torch.cuda.device(q.device):
        _lib.check(_lib.lib().atom_batch_decode_split_gqa_i4(o.data_ptr(), q.data_ptr(), kv.data.data_ptr(), kv.param.data_ptr(),
                                                             kv.indptr.data_ptr(), kv.indicies.data_ptr(),
                                                             kv.last_page_offset.data_ptr(), L, layer_idx, q.size(1), H, P, q.size(0),
                                                             float(rope_theta), int(kv_split), _stream(q)), "batch_decode_i4")
    return o


def decode_kv_split(batch, num_kv_heads, group, device=None):
    """The cluster size `batch_decode_i4(..., kv_split=0)` uses for `batch` sequences of `num_kv_heads` KV heads with `group`
    query heads each on `device` (default: the current CUDA device): 1 when the grid already gives every SM a CTA."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    c = _lib.lib().atom_decode_kv_split(int(batch), int(num_kv_heads), int(group), int(sms))
    _lib.check(min(c, 0), "decode_kv_split")
    return c


# Shared-prefix decode rule, from host-known sizes only (a captured graph replays it with new lengths): the cascade runs when
#   (1) more than half of the batch's rows are group members,
#   (2) every group has at least DECODE_CASCADE_MIN_ROWS query rows per KV head (members x G): the prefix pass's MMAs take 64
#       rows, and fewer leave the tile mostly empty while the pages are streamed at the same cost, and
#   (3) the token-heads it saves, num_kv_heads x sum over groups of (members - 1) x shared tokens, reach
#       DECODE_CASCADE_MIN_PER_SM per SM: enough to pay for the prefix pass's launch and the partial merge.
# (1) because the suffix pass runs unsplit: lone rows (of unknown length) keep the time a batch of them takes, and a small
# grid loses the split-KV the plain kernel would get.  Thresholds measured on an H100 with tools/shared_prefix_bench.py
# (DESIGN.md section 6).
DECODE_CASCADE_MIN_ROWS = 16
DECODE_CASCADE_MIN_PER_SM = 256


def decode_cascade(groups, batch, page_size, num_kv_heads, group, sm_count):
    """Whether `batch_decode_i4(..., kv_split=0)` runs the cascade for a batch of `batch` rows with these prefix groups ((rows,
    shared pages) pairs, as BatchedKvCacheInt4.groups holds them), `num_kv_heads` KV heads, `group` query heads per KV head, on
    a device of `sm_count` SMs."""
    members = sum(len(rows) for rows, _ in groups)
    saved = num_kv_heads * sum((len(rows) - 1) * n * page_size for rows, n in groups)
    return bool(groups) and 2 * members > batch and min(len(rows) for rows, _ in groups) * group >= DECODE_CASCADE_MIN_ROWS \
        and saved >= DECODE_CASCADE_MIN_PER_SM * sm_count


def _batch_decode_shared(o, q, kv, groups, L, H, P, layer_idx, rope_theta, sms):
    """The cascade: prefix pass over each group's shared pages, then the decode kernel over the private pages."""
    b, hq = q.size(0), q.size(1)
    # a table in static buffers (a CUDA-graph replay) states bounds that hold for every step it will carry: (members of a group,
    # shared pages) at most; the launch is sized from them, so the replay stays valid as members and lengths change
    bounds = getattr(kv, "group_bounds", None)
    if bounds is not None:
        max_size, max_shared = int(bounds[0]), int(bounds[1]) * P
    else:
        max_size, max_shared = max(len(rows) for rows, _ in groups), max(n for _, n in groups) * P
    lib = _lib.lib()
    nchunks = lib.atom_decode_shared_chunks(len(groups), b, hq // H, H, sms)
    _lib.check(min(nchunks, 0), "decode_shared_chunks")
    ws = torch.empty((b, hq, nchunks, 130), dtype=torch.float32, device=q.device)
    table = rope_table(max_shared, q.device, rope_theta)
    with torch.cuda.device(q.device):
        _lib.check(lib.atom_batch_decode_shared_gqa_i4(
            o.data_ptr(), q.data_ptr(), kv.data.data_ptr(), kv.param.data_ptr(), kv.indptr.data_ptr(), kv.indicies.data_ptr(),
            kv.last_page_offset.data_ptr(), L, layer_idx, hq, H, P, b, float(rope_theta), kv.group_indptr.data_ptr(),
            kv.group_members.data_ptr(), kv.shared_pages.data_ptr(), len(groups), max_size, table.data_ptr(), ws.data_ptr(), nchunks,
            _stream(q)), "batch_decode_i4 (shared prefix)")
    return o


def verify_chunks(batch, num_kv_heads, device=None):
    """The chunk count `batch_verify_i4(..., nchunks=0)` uses for `batch` sequences of `num_kv_heads` KV heads on `device`
    (default: the current CUDA device): 1 when the (sequence, KV head) grid already gives every SM a CTA."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    c = _lib.lib().atom_verify_chunks(int(batch), int(num_kv_heads), int(sms))
    _lib.check(min(c, 0), "verify_chunks")
    return c


def batch_verify_i4(q, kv, layer_idx, tokens_per_seq, rope_theta=10000.0, max_len=None, nchunks=0):
    """EXTENSION (speculative decoding): multi-token decode attention of a verify step.  Sequence b of `kv` ends with S =
    `tokens_per_seq` query tokens (1 <= S <= 8) whose K/V are already in the pages (init_kv_i4 with a stride-S indptr), at
    positions len_b - S .. len_b - 1; token i attends to every cached token before the tail and, causally, to the tail up to
    itself.  q f16 [B*S, Hq, 128], sequence-major and token-minor (row b*S + i); returns the same shape.  Query head counts per
    KV head of 1, 2, 4 or 8, as batch_decode_i4.  Positions come from the page table on the device; `max_len` bounds every
    sequence's length and sizes the RoPE table (a CUDA graph captured with a bound replays as lengths grow up to it); without it
    the bound is read from `kv.seqlens` (a BatchedKvCacheInt4).  nchunks: 0 = automatic (`verify_chunks`), n = cut each
    sequence's tiles into n runs merged in order (1 = unsplit)."""
    _req_width("batch_verify_i4", f16_q_2=q)
    _req_cuda(q, kv.data, kv.param, kv.indptr, kv.indicies, kv.last_page_offset)
    L, H, P = _kv_dims(kv)
    S = int(tokens_per_seq)
    if not 1 <= S <= 8:
        raise RuntimeError(f"batch_verify_i4: tokens_per_seq={S} must be in [1, 8]")
    B = kv.last_page_offset.size(0)
    if q.dim() != 3 or q.size(2) != 128 or q.size(0) != B * S or kv.indptr.size(0) != B + 1:
        raise RuntimeError(f"batch_verify_i4: q {tuple(q.shape)} does not hold {S} tokens of 128 per head for each of {B} sequences")
    if max_len is None:
        lens = getattr(kv, "seqlens", None)
        if lens is None:
            raise RuntimeError("batch_verify_i4: pass `max_len` or a `kv` with host sequence lengths (`seqlens`)")
        if min(lens) < S:
            raise RuntimeError(f"batch_verify_i4: a sequence holds {min(lens)} tokens, fewer than its {S} query tokens")
        max_len = max(lens)
    hq = q.size(1)
    nchunks = int(nchunks) if nchunks else verify_chunks(B, H, q.device)
    ws = torch.empty((B * S, hq, nchunks, 130), dtype=torch.float32, device=q.device) if nchunks > 1 else None
    table = rope_table(max_len, q.device, rope_theta)
    o = torch.empty_like(q)
    with torch.cuda.device(q.device):
        _lib.check(_lib.lib().atom_batch_verify_gqa_i4(
            o.data_ptr(), q.data_ptr(), kv.data.data_ptr(), kv.param.data_ptr(), kv.indptr.data_ptr(), kv.indicies.data_ptr(),
            kv.last_page_offset.data_ptr(), L, int(layer_idx), hq, H, P, B, S, float(rope_theta), table.data_ptr(),
            None if ws is None else ws.data_ptr(), nchunks, _stream(q)), "batch_verify_i4")
    return o


_rope_tables = {}


def rope_table(max_len, device, theta=10000.0):
    """(cos, sin)(pos * theta_i) for pos < max_len, i < 64, theta_i = theta^(-i/64), float32 [max_len, 64, 2] -- the factors of
    punica/models/llama.py:18-32 (`rotary_pos_emb`), computed the same way and cached per (device, base)."""
    size = max(256, 1 << (int(max_len) - 1).bit_length())
    key = (str(device), size) if float(theta) == 10000.0 else (str(device), size, float(theta))
    t = _rope_tables.get(key)
    if t is None:
        base = 10000 if float(theta) == 10000.0 else float(theta)
        inv_freq = 1.0 / (base ** (torch.arange(0, 128, 2, device=device).float() / 128))
        freqs = torch.einsum("i,j->ij", torch.arange(0, size, device=device, dtype=torch.float32), inv_freq)
        t = torch.stack((freqs.cos(), freqs.sin()), dim=-1).contiguous()
        _rope_tables[key] = t
    return t


def prefill_attention_i4(q, k, k_param, v, v_param, seqlen_indptr, seqlens=None, rope_theta=10000.0, *, kv=None, layer_idx=None):
    """EXTENSION: causal prefill attention of every prompt over its own quantised K/V (the o4 projection outputs) with RoPE,
    one launch for all prompts and heads.  q f16 [T, H*128]; k, v u8 [T, Hkv*64]; k_param, v_param f16 [T, Hkv*2] (Hkv = H, or
    a divisor of it for grouped-query attention: taken from k's shape); seqlen_indptr i32 [B+1] (device); seqlens: the prompt
    lengths as host ints (avoids a device read); rope_theta: the RoPE base.  Returns f16 [T, H*128].
    EXTENSION (chunked prefill, prompt continuation): with `kv` (a BatchedKvCacheInt4 of the B sequences) and `layer_idx`, prompt b
    is the tail of sequence b of the cache -- what init_kv_i4 just wrote there -- at positions ctx_b .. ctx_b + n_b - 1, ctx_b =
    kv.seqlens[b] - n_b.  It attends to the whole cached prefix and, causally, to its own tokens; query head counts per KV head
    of 1, 2, 4 or 8.  When every ctx_b is 0 this is the call without `kv`, bit for bit."""
    _req_width("prefill_attention_i4", f16_q_2=q, k_1=k, f16_k_param_2=k_param, v_1=v, f16_v_param_2=v_param)
    _req_cuda(q, k, k_param, v, v_param, seqlen_indptr)
    t, hd = q.shape
    h = hd // 128
    hkv = k.shape[1] // 64 if k.dim() == 2 else 0
    if hd % 128 or k.dim() != 2 or k.shape != (t, hkv * 64) or hkv == 0 or v.shape != k.shape or k_param.numel() != t * hkv * 2 or \
            v_param.numel() != t * hkv * 2:
        raise RuntimeError("prefill_attention_i4: shape mismatch (head_dim must be 128)")
    if seqlens is None:
        ip = seqlen_indptr.cpu()
        seqlens = (ip[1:] - ip[:-1]).tolist()
    b, max_len = len(seqlens), max(seqlens)
    if sum(seqlens) != t or seqlen_indptr.numel() != b + 1:
        raise RuntimeError("prefill_attention_i4: seqlen_indptr does not cover the tokens")
    ctx = _prefill_contexts(kv, layer_idx, seqlens)
    if not any(ctx):
        pos = torch.cat([torch.arange(n, dtype=torch.int32) for n in seqlens]).to(q.device, non_blocking=True)
        table = rope_table(max_len, q.device, rope_theta)
    else:
        _req_cuda(kv.data, kv.param, kv.indptr, kv.indicies, kv.last_page_offset)
        L, H, P = _kv_dims(kv)
        if H != hkv:
            raise RuntimeError(f"prefill_attention_i4: the cache has {H} KV heads, k has {hkv}")
        pos = torch.cat([torch.arange(c, c + n, dtype=torch.int32) for c, n in zip(ctx, seqlens)]).to(q.device, non_blocking=True)
        table = rope_table(max(c + n for c, n in zip(ctx, seqlens)), q.device, rope_theta)
    kf = torch.empty((t, hkv * 128), dtype=q.dtype, device=q.device)
    vf, out = torch.empty_like(kf), torch.empty_like(q)
    with torch.cuda.device(q.device):
        if not any(ctx):
            _lib.check(_lib.lib().atom_prefill_attention_gqa_i4(q.data_ptr(), k.data_ptr(), k_param.data_ptr(), v.data_ptr(),
                                                                v_param.data_ptr(), seqlen_indptr.data_ptr(), pos.data_ptr(),
                                                                table.data_ptr(), kf.data_ptr(), vf.data_ptr(), out.data_ptr(), t, b,
                                                                max_len, h, hkv, _stream(q)), "prefill_attention_i4")
        else:
            _lib.check(_lib.lib().atom_prefill_attention_ctx_gqa_i4(
                q.data_ptr(), k.data_ptr(), k_param.data_ptr(), v.data_ptr(), v_param.data_ptr(), seqlen_indptr.data_ptr(),
                pos.data_ptr(), table.data_ptr(), kf.data_ptr(), vf.data_ptr(), out.data_ptr(), t, b, max_len, h, hkv,
                kv.data.data_ptr(), kv.param.data_ptr(), kv.indptr.data_ptr(), kv.indicies.data_ptr(), kv.last_page_offset.data_ptr(),
                L, int(layer_idx), P, _stream(q)), "prefill_attention_i4")
    return out


def _prefill_contexts(kv, layer_idx, seqlens):
    """Cached tokens before each prompt (all zeros without a cache), from the host lengths the batch recorded."""
    if kv is None:
        return [0] * len(seqlens)
    lens = getattr(kv, "seqlens", None)
    if lens is None:
        raise RuntimeError("prefill_attention_i4: `kv` carries no host sequence lengths (`seqlens`): build it as a BatchedKvCacheInt4")
    if layer_idx is None:
        raise RuntimeError("prefill_attention_i4: `kv` needs `layer_idx`")
    if len(lens) != len(seqlens):
        raise RuntimeError(f"prefill_attention_i4: `kv` holds {len(lens)} sequences for {len(seqlens)} prompts")
    ctx = [int(s) - int(n) for s, n in zip(lens, seqlens)]
    if min(ctx) < 0:
        b = min(range(len(ctx)), key=ctx.__getitem__)
        raise RuntimeError(f"prefill_attention_i4: sequence {b} holds {lens[b]} tokens, fewer than its prompt of {seqlens[b]}")
    return ctx


def init_kv_i4(kv, k, v, k_param, v_param, seqlen_indptr, layer_idx):
    """ops/__init__.py:35-46"""
    _req_cuda(kv.data, kv.param, kv.indptr, kv.indicies, kv.last_page_offset, k, v, k_param, v_param, seqlen_indptr)
    L, H, P = _kv_dims(kv)
    B = kv.last_page_offset.size(0)
    if kv.indptr.size(0) != B + 1 or seqlen_indptr.size(0) != B + 1:
        raise RuntimeError("init_kv_i4: indptr sizes do not match the batch")
    with torch.cuda.device(k.device):
        _lib.check(_lib.lib().atom_init_kv_i4(kv.data.data_ptr(), kv.param.data_ptr(), kv.indptr.data_ptr(),
                                              kv.indicies.data_ptr(), kv.last_page_offset.data_ptr(), k.data_ptr(),
                                              v.data_ptr(), k_param.data_ptr(), v_param.data_ptr(),
                                              seqlen_indptr.data_ptr(), k.size(0), L, layer_idx, H, P, B, _stream(k)),
                   "init_kv_i4")


def append_kv_i4(kv, k, v, k_param, v_param, layer_idx):
    """ops/__init__.py:49-59"""
    _req_cuda(kv.data, kv.param, kv.indptr, kv.indicies, kv.last_page_offset, k, v, k_param, v_param)
    L, H, P = _kv_dims(kv)
    B = k.size(0)
    if kv.indptr.size(0) != B + 1 or kv.last_page_offset.size(0) != B or k.shape != v.shape:
        raise RuntimeError("append_kv_i4: shape mismatch")
    with torch.cuda.device(k.device):
        _lib.check(_lib.lib().atom_append_kv_i4(kv.data.data_ptr(), kv.param.data_ptr(), kv.indptr.data_ptr(),
                                                kv.indicies.data_ptr(), kv.last_page_offset.data_ptr(), k.data_ptr(),
                                                v.data_ptr(), k_param.data_ptr(), v_param.data_ptr(), L, layer_idx, H,
                                                P, B, _stream(k)), "append_kv_i4")


# ------------------------------------------------------------------------------------------------ sparse MoE block (Mixtral)
def moe_token_tile(seq_len, num_experts, top_k):
    """Token tile of the grouped expert GEMM: the smallest of 16 / 32 / 64 that holds the mean rows per expert."""
    mean = -(-int(seq_len) * int(top_k) // int(num_experts))
    return 16 if mean <= 16 else (32 if mean <= 32 else 64)


def moe_tiles(seq_len, num_experts, top_k):
    """(BN, tiles_max, rows_cap) of one MoE block: the token tile, the length of the tile table (every expert's segment padded to
    BN rows: at most min(T*k, (T*k + E*(BN-1)) // BN) tiles) and the rows of the permuted workspace.  Host-known sizes only, so
    the block can be captured in a CUDA graph whatever the routing."""
    bn = moe_token_tile(seq_len, num_experts, top_k)
    slots = int(seq_len) * int(top_k)
    tiles_max = min(slots, (slots + int(num_experts) * (bn - 1)) // bn)
    return bn, tiles_max, tiles_max * bn


def moe_route_f16(hidden_sum, norm_weight, reorder_index, eps, router_weight, top_k, router_logits=False, normed=False):
    """EXTENSION: the FP router of the MoE block on the FP16 normalised row (formed exactly as rmsnorm_fp16_i4 forms it, in the
    reordered channel order of `router_weight` f16 [E, H]).  Returns (topk_ids i32 [T,k], topk_weights f16 [T,k]) plus, on request,
    the FP32 logits [T,E] and the normalised row f16 [T,H]."""
    if isinstance(norm_weight, torch.Tensor) and norm_weight.dtype != torch.float16:
        norm_weight = norm_weight.to(torch.float16)
    _req_width("moe_route_f16", f16_hidden_sum_2=hidden_sum, f16_norm_weight_2=norm_weight, reorder_index_2=reorder_index,
               f16_router_weight_2=router_weight)
    _req_cuda(hidden_sum, norm_weight, reorder_index, router_weight)
    t, h = hidden_sum.shape
    e = router_weight.size(0)
    if router_weight.shape != (e, h) or norm_weight.numel() != h or reorder_index.numel() != h:
        raise RuntimeError("moe_route_f16: router_weight must be [E, H], norm_weight and reorder_index [H]")
    dev = hidden_sum.device
    ids = torch.empty((t, top_k), dtype=torch.int32, device=dev)
    w = torch.empty((t, top_k), dtype=torch.float16, device=dev)
    lg = torch.empty((t, e), dtype=torch.float32, device=dev) if router_logits else None
    yn = torch.empty((t, h), dtype=torch.float16, device=dev) if normed else None
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().atom_moe_route_f16(hidden_sum.data_ptr(), norm_weight.data_ptr(), float(eps), reorder_index.data_ptr(),
                                                 router_weight.data_ptr(), t, h, e, int(top_k), ids.data_ptr(), w.data_ptr(),
                                                 lg.data_ptr() if lg is not None else None, yn.data_ptr() if yn is not None else None,
                                                 _stream(hidden_sum)), "moe_route_f16")
    return (ids, w) + ((lg,) if router_logits else ()) + ((yn,) if normed else ())


def moe_plan(topk_ids, num_experts, token_tile=None, tiles_max=None):
    """EXTENSION: (dest_row i32 [T,k], tiles i32 [tiles_max,4]) of the routing -- see include/atom_b200.h.  token_tile / tiles_max
    default to moe_tiles()."""
    _req_width("moe_plan", topk_ids_4=topk_ids)
    _req_cuda(topk_ids)
    t, k = topk_ids.shape
    bn, tmax, _ = moe_tiles(t, num_experts, k)
    bn = bn if token_tile is None else int(token_tile)
    tmax = tmax if tiles_max is None else int(tiles_max)
    dest = torch.empty((t, k), dtype=torch.int32, device=topk_ids.device)
    tiles = torch.empty((tmax, 4), dtype=torch.int32, device=topk_ids.device)
    with torch.cuda.device(topk_ids.device):
        _lib.check(_lib.lib().atom_moe_plan(topk_ids.data_ptr(), t, int(num_experts), k, bn, tmax, dest.data_ptr(), tiles.data_ptr(),
                                            _stream(topk_ids)), "moe_plan")
    return dest, tiles


def moe_gather_i4(x, dest_row, rows_cap, out=None):
    """EXTENSION: the activation 4-tuple `x` of T tokens permuted into the experts' segments: a 4-tuple of rows_cap rows (scales in
    the layout of S(rows_cap)).  `out`: an existing 4-tuple to fill (pad rows keep what they held)."""
    o8, o4, s8, s4 = x
    _req_width("moe_gather_i4", o_outliers_1=o8, o_norms_1=o4, f16_outlier_scales_2=s8, f16_norm_scales_2=s4, dest_row_4=dest_row)
    _req_cuda(o8, o4, s8, s4, dest_row)
    t, k = dest_row.shape
    h = o4.size(1) * 2 + 128
    if o8.shape != (t, 128) or o4.size(0) != t:
        raise RuntimeError("moe_gather_i4: the tuple must hold one row per token of dest_row")
    out = out if out is not None else _quant_outputs(int(rows_cap), h, o8.device)
    with torch.cuda.device(o8.device):
        _lib.check(_lib.lib().atom_moe_gather_i4(o8.data_ptr(), o4.data_ptr(), s8.data_ptr(), s4.data_ptr(), t, h, k, dest_row.data_ptr(),
                                                 int(rows_cap), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(),
                                                 _stream(o8)), "moe_gather_i4")
    return out


def _grouped_args(what, x, w4, s4, w8, s8, tiles, token_tile):
    o8, o4, xs8, xs4 = x
    _req_width(what, a_1=o4, b_1=w4, f16_a_scale_2=xs4, f16_b_scale_2=s4, a_keeper_1=o8, b_keeper_1=w8, f16_a_keeper_scale_2=xs8,
               f16_b_keeper_scale_2=s8, tiles_4=tiles)
    _req_cuda(o4, w4, xs4, s4, o8, w8, xs8, s8, tiles)
    rows_cap, k = o8.size(0), o4.size(1) * 2 + 128
    if w4.dim() != 3 or w8.dim() != 3 or w4.shape[:2] != w8.shape[:2] or w4.size(2) * 2 + 128 != k or \
            s4.shape != (w4.size(0), k // 128 - 1, w4.size(1)) or s8.shape != w4.shape[:2]:
        raise RuntimeError(f"{what}: weights must be stacked [E, N, ...] with scales [E, K/128-1, N] and [E, N]")
    if rows_cap != tiles.size(0) * int(token_tile):
        raise RuntimeError(f"{what}: the permuted activations must have tiles x token_tile rows")
    return rows_cap, k


def dense_layer_gemm_i4_gateup_act_grouped(x, w13_int4, w13_scale, w13_int8, w13_keeper_scale, tiles, token_tile):
    """EXTENSION: the gate/up projections + SiLU(gate) * up + quantisation of every expert in one launch over the permuted
    activation tuple `x` (moe_gather_i4) and the tile table (moe_plan).  w13_* are stacked [E, 2I, ...] (gate rows, then up rows,
    per expert).  Returns the activation tuple of the down projection (rows_cap rows; pad rows unwritten)."""
    rows_cap, k = _grouped_args("dense_layer_gemm_i4_gateup_act_grouped", x, w13_int4, w13_scale, w13_int8, w13_keeper_scale, tiles,
                                token_tile)
    e, n2 = w13_int4.shape[:2]
    out = _quant_outputs(rows_cap, n2 // 2, x[0].device)
    with torch.cuda.device(x[0].device):
        _lib.check(_lib.lib().atom_gemm_i4_gateup_act_grouped(x[1].data_ptr(), w13_int4.data_ptr(), x[3].data_ptr(), w13_scale.data_ptr(),
                                                              x[0].data_ptr(), w13_int8.data_ptr(), x[2].data_ptr(),
                                                              w13_keeper_scale.data_ptr(), out[0].data_ptr(), out[1].data_ptr(),
                                                              out[2].data_ptr(), out[3].data_ptr(), tiles.data_ptr(), tiles.size(0),
                                                              int(token_tile), rows_cap, e, n2 // 2, k, _stream(x[0])),
                   "dense_layer_gemm_i4_gateup_act_grouped")
    return out


def dense_layer_gemm_i4_fp16_grouped(x, w2_int4, w2_scale, w2_int8, w2_keeper_scale, tiles, token_tile):
    """EXTENSION: the down projection of every expert in one launch; w2_* stacked [E, H, ...].  Returns f16 [rows_cap, H]."""
    rows_cap, k = _grouped_args("dense_layer_gemm_i4_fp16_grouped", x, w2_int4, w2_scale, w2_int8, w2_keeper_scale, tiles, token_tile)
    e, n = w2_int4.shape[:2]
    d = torch.empty((rows_cap, n), dtype=torch.float16, device=x[0].device)
    with torch.cuda.device(x[0].device):
        _lib.check(_lib.lib().atom_gemm_i4_o16_grouped(x[1].data_ptr(), w2_int4.data_ptr(), x[3].data_ptr(), w2_scale.data_ptr(),
                                                       x[0].data_ptr(), w2_int8.data_ptr(), x[2].data_ptr(), w2_keeper_scale.data_ptr(),
                                                       d.data_ptr(), tiles.data_ptr(), tiles.size(0), int(token_tile), rows_cap, e, n, k,
                                                       _stream(x[0])), "dense_layer_gemm_i4_fp16_grouped")
    return d


def moe_combine_f16(y, topk_ids, topk_weights, dest_row):
    """EXTENSION: out f16 [T,H] = the experts' outputs weighted and summed per token in ascending expert order (FP16 products
    and adds from +0.0), bit for bit the index_add_ loop of the simulator."""
    _req_width("moe_combine_f16", f16_y_2=y, topk_ids_4=topk_ids, f16_topk_weights_2=topk_weights, dest_row_4=dest_row)
    _req_cuda(y, topk_ids, topk_weights, dest_row)
    t, k = topk_ids.shape
    if topk_weights.shape != (t, k) or dest_row.shape != (t, k):
        raise RuntimeError("moe_combine_f16: topk_ids, topk_weights and dest_row must all be [T, k]")
    out = torch.empty((t, y.size(1)), dtype=torch.float16, device=y.device)
    with torch.cuda.device(y.device):
        _lib.check(_lib.lib().atom_moe_combine_f16(y.data_ptr(), topk_ids.data_ptr(), topk_weights.data_ptr(), dest_row.data_ptr(), t,
                                                   y.size(1), k, out.data_ptr(), _stream(y)), "moe_combine_f16")
    return out


def _sample_param(name, v, b, dtype, device, check):
    """One per-row parameter of sample_tokens: a CUDA tensor of `b` elements (values read on the device), or a host sequence /
    scalar that is checked here and copied."""
    if isinstance(v, torch.Tensor):
        _req_cuda(v)
        want = torch.int64 if dtype in (torch.int64, torch.uint64) else dtype
        if v.dtype != want and not (want == torch.int64 and v.dtype == torch.uint64):
            raise RuntimeError(f"atom_b200.ops.sample_tokens: `{name}` must be {want}, got {v.dtype}")
        shape = (b, 2) if name == "keys" else (b,)
        if tuple(v.shape) != shape:
            raise RuntimeError(f"atom_b200.ops.sample_tokens: `{name}` must have shape {shape}, got {tuple(v.shape)}")
        if v.device != device:
            raise RuntimeError(f"atom_b200.ops.sample_tokens: `{name}` must be on {device}")
        return v
    import numpy as np
    if dtype in (torch.int64, torch.uint64):                    # 64-bit words: any integer in [0, 2^64)
        ints = np.array(v, dtype=object).reshape(-1)
        if not all(isinstance(x, (int, np.integer)) and 0 <= int(x) < 1 << 64 for x in ints):
            raise RuntimeError(f"atom_b200.ops.sample_tokens: `{name}` must hold integers in [0, 2^64)")
        a = np.array([int(x) for x in ints], dtype=np.uint64).view(np.int64)
        shape = (b, 2) if name == "keys" else (b,)
        if a.size != int(np.prod(shape)):
            raise RuntimeError(f"atom_b200.ops.sample_tokens: `{name}` must have {shape} entries, got {a.size}")
        return torch.from_numpy(a.reshape(shape)).to(device)
    a = np.broadcast_to(np.asarray(v, dtype=np.float64), (b,)) if np.ndim(v) == 0 else np.asarray(v, dtype=np.float64)
    if a.shape != (b,):
        raise RuntimeError(f"atom_b200.ops.sample_tokens: `{name}` must have {b} entries, got shape {a.shape}")
    bad = check(a)
    if bad.any():
        raise RuntimeError(f"atom_b200.ops.sample_tokens: `{name}` out of range at row {int(np.argmax(bad))}: {a[np.argmax(bad)]!r}")
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(device)


SAMPLE_TOP_N_MAX = 20


def penalty_table(slots, vocab, device):
    """EXTENSION: a zeroed penalty table for `slots` requests over a `vocab`-token vocabulary, for sample_tokens' penalties:
    int16 [slots, ld] holding the u16 entries of atom_sample_ex_f16 (bit 15: the token is in the request's prompt; bits 0-14:
    how often the request has generated it, saturating at 0x7FFF), ld = vocab rounded up to a multiple of 8."""
    if int(slots) < 1 or int(vocab) < 1:
        raise RuntimeError(f"atom_b200.ops.penalty_table: need slots >= 1 and vocab >= 1, got {slots}, {vocab}")
    return torch.zeros((int(slots), (int(vocab) + 7) // 8 * 8), dtype=torch.int16, device=device)


def _check_table(table):
    if not (isinstance(table, torch.Tensor) and table.is_cuda):
        raise RuntimeError("atom_b200.ops: all tensors must live on a CUDA device (there is no CPU path)")
    if table.dtype not in (torch.int16, torch.uint16) or table.dim() != 2 or table.stride(1) != 1 or table.stride(0) % 8 or \
            table.data_ptr() % 16:
        raise RuntimeError("atom_b200.ops: a penalty table is 16-bit [slots, ld] with unit stride along ld, a row pitch that is a "
                           "multiple of 8 and a 16-byte aligned base (ops.penalty_table)")


def init_penalty_slot(table, slot, prompt):
    """EXTENSION: set up `slot` of a penalty table for a new request in one launch: zero its row and mark every token of `prompt`
    (all the request's prompt, a shared system prompt included) as a prompt token.  prompt: token ids, a host sequence (checked
    to lie in [0, ld)) or an int32 CUDA tensor (ids outside it are ignored)."""
    _check_table(table)
    if not 0 <= int(slot) < table.size(0):
        raise RuntimeError(f"atom_b200.ops.init_penalty_slot: slot {slot} outside [0, {table.size(0)})")
    if isinstance(prompt, torch.Tensor):
        _req_cuda(prompt)
        if prompt.dtype != torch.int32 or prompt.dim() != 1 or not prompt.is_contiguous():
            raise RuntimeError("atom_b200.ops.init_penalty_slot: a prompt tensor must be contiguous int32 [n]")
        ids = prompt
    else:
        import numpy as np
        a = np.asarray(prompt, dtype=np.int64).reshape(-1)
        if a.size and (a.min() < 0 or a.max() >= table.size(1)):
            raise RuntimeError(f"atom_b200.ops.init_penalty_slot: prompt ids must lie in [0, {table.size(1)})")
        ids = torch.from_numpy(a.astype(np.int32)).to(table.device)
    with torch.cuda.device(table.device):
        _lib.check(_lib.lib().atom_sample_slot_init(table.data_ptr(), table.stride(0), table.size(1), int(slot),
                                                    ids.data_ptr() if ids.numel() else None, ids.numel(), _stream(table)),
                   "init_penalty_slot")


def _neutral(v, value):
    import numpy as np
    return not isinstance(v, torch.Tensor) and bool(np.all(np.asarray(v, dtype=np.float64) == value))


def _sample_slots(slots, b, table, device):
    if isinstance(slots, torch.Tensor):
        _req_cuda(slots)
        if slots.dtype != torch.int32 or tuple(slots.shape) != (b,) or slots.device != device:
            raise RuntimeError(f"atom_b200.ops.sample_tokens: `slots` must be int32 [{b}] on {device}")
        return slots
    import numpy as np
    a = np.asarray(slots, dtype=np.int64).reshape(-1)
    if a.shape != (b,) or (a < -1).any() or (a >= table.size(0)).any():
        raise RuntimeError(f"atom_b200.ops.sample_tokens: `slots` must hold {b} entries in [-1, {table.size(0)})")
    used = a[a >= 0]
    if len(np.unique(used)) != len(used):
        raise RuntimeError("atom_b200.ops.sample_tokens: the rows of one call must use distinct slots")
    return torch.from_numpy(a.astype(np.int32)).to(device)


def sample_tokens(logits, temperature, top_k, top_p, keys, counters, *, min_p=0.0, repetition_penalty=1.0, frequency_penalty=0.0,
                  presence_penalty=0.0, penalty_table=None, slots=None, logprobs=None, drafts=None):
    """EXTENSION: one token id per row of f16 logits [B, V] (rows may have any pitch), int32 [B].  Per row: temperature
    (0 = argmax), top_k (0 = off, on the raw logits), top_p (1 = off), Philox key (key0, key1) and counter; the semantics are
    atom_sample_f16's (include/atom_b200.h, DESIGN section 5.6).  Each parameter is a CUDA tensor with one entry per row (keys:
    [B, 2]; keys and counters int64 holding the uint64 bit patterns) whose values are read on the device -- so a captured graph
    replays with new ones -- or a host sequence or scalar, which is validated (T finite and >= 0, top_k >= 0, top_p in (0, 1])
    and copied.  Rows with NaN / +inf logits, only -inf logits, or out-of-range device parameters give -1.

    The keyword options (atom_sample_ex_f16; at their defaults the call and its result are exactly the above), each per row like
    the parameters:
      min_p in [0, 1] (0 = off); repetition_penalty > 0 (1 = off), frequency_penalty and presence_penalty finite (0 = off),
      which need penalty_table (ops.penalty_table) and slots (int32 [B], -1 = no state, distinct in one call): the kernel
      penalises each row's logits by its slot's history and records the drawn token in that slot;
      logprobs = n in [0, 20]: also return, per row, the log-probability of the chosen token (float32 [B]) and the first n
      tokens of the order on the penalised logits with theirs (int32 / float32 [B, n]), a log-softmax at temperature 1.
    With logprobs the result is (tokens, logprob, top_ids, top_logprobs).

    drafts (atom_sample_draft_f16; speculative decoding): one candidate token per row, an int32 CUDA tensor [B] or a host sequence
    (-1 = none).  A row accepts its candidate d with probability W_d / Z (its kept weight over the kept total: rejection
    sampling with a point-mass proposal) and otherwise draws from the kept set without d, so every token keeps the probability
    the sampler gives it (DESIGN section 5.7).  Greedy rows return the argmax whatever d is; rows without a candidate are exactly
    the call without drafts; a candidate outside [-1, V) in a device tensor gives -1.  Not with penalties.  None: exactly the
    call above."""
    if not (isinstance(logits, torch.Tensor) and logits.is_cuda):
        raise RuntimeError("atom_b200.ops: all tensors must live on a CUDA device (there is no CPU path)")
    if logits.dtype != torch.float16 or logits.dim() != 2 or logits.stride(1) != 1:
        raise RuntimeError("atom_b200.ops.sample_tokens: logits must be float16 [B, V] with unit stride along V")
    b, v = logits.shape
    dev = logits.device
    import numpy as np
    t = _sample_param("temperature", temperature, b, torch.float32, dev, lambda a: ~np.isfinite(a) | (a < 0))
    k = _sample_param("top_k", top_k, b, torch.int32, dev, lambda a: (a < 0) | (a != np.floor(a)) | (a >= 1 << 31))
    p = _sample_param("top_p", top_p, b, torch.float32, dev, lambda a: ~((a > 0) & (a <= 1)))
    key = _sample_param("keys", keys, b, torch.int64, dev, None)
    ctr = _sample_param("counters", counters, b, torch.int64, dev, None)
    pen = penalty_table is not None
    if not pen and (slots is not None or not (_neutral(repetition_penalty, 1) and _neutral(frequency_penalty, 0) and
                                              _neutral(presence_penalty, 0))):
        raise RuntimeError("atom_b200.ops.sample_tokens: penalties need a penalty_table and slots")
    if logprobs is not None and not (isinstance(logprobs, (int, np.integer)) and 0 <= int(logprobs) <= SAMPLE_TOP_N_MAX):
        raise RuntimeError(f"atom_b200.ops.sample_tokens: logprobs must be an integer in [0, {SAMPLE_TOP_N_MAX}], got {logprobs!r}")
    if drafts is not None:
        if pen or slots is not None:
            raise RuntimeError("atom_b200.ops.sample_tokens: drafts cannot be combined with penalties")
        return _sample_draft(logits, t, k, p, key, ctr, min_p, logprobs, drafts)
    if pen or logprobs is not None or not _neutral(min_p, 0):
        return _sample_ex(logits, t, k, p, key, ctr, min_p, repetition_penalty, frequency_penalty, presence_penalty, penalty_table,
                          slots, logprobs)
    out = torch.empty((b,), dtype=torch.int32, device=dev)
    if b == 0:
        return out
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().atom_sample_f16(logits.data_ptr(), logits.stride(0) if b > 1 else v, b, v, t.data_ptr(), k.data_ptr(),
                                              p.data_ptr(), key.data_ptr(), ctr.data_ptr(), out.data_ptr(), _stream(logits)),
                   "sample_tokens")
    return out


def _sample_ex(logits, t, k, p, key, ctr, min_p, rep, freq, pres, table, slots, logprobs):
    import numpy as np
    b, v = logits.shape
    dev = logits.device
    m = None if _neutral(min_p, 0) else _sample_param("min_p", min_p, b, torch.float32, dev, lambda a: ~((a >= 0) & (a <= 1)))
    pen = table is not None
    if pen:
        _check_table(table)
        if table.device != dev or table.size(1) < v:
            raise RuntimeError(f"atom_b200.ops.sample_tokens: penalty_table must be on {dev} with at least {v} columns")
        if slots is None:
            raise RuntimeError("atom_b200.ops.sample_tokens: penalty_table needs slots")
        sl = _sample_slots(slots, b, table, dev)
        r = _sample_param("repetition_penalty", rep, b, torch.float32, dev, lambda a: ~np.isfinite(a) | (a <= 0))
        f = _sample_param("frequency_penalty", freq, b, torch.float32, dev, lambda a: ~np.isfinite(a))
        q = _sample_param("presence_penalty", pres, b, torch.float32, dev, lambda a: ~np.isfinite(a))
    n = 0 if logprobs is None else int(logprobs)
    out = torch.empty((b,), dtype=torch.int32, device=dev)
    lp = torch.empty((b,), dtype=torch.float32, device=dev) if logprobs is not None else None
    top_ids = torch.empty((b, n), dtype=torch.int32, device=dev)
    top_lp = torch.empty((b, n), dtype=torch.float32, device=dev)
    if b:
        ptr = lambda x: None if x is None else x.data_ptr()      # noqa: E731
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().atom_sample_ex_f16(
                logits.data_ptr(), logits.stride(0) if b > 1 else v, b, v, t.data_ptr(), k.data_ptr(), p.data_ptr(), key.data_ptr(),
                ctr.data_ptr(), ptr(m), ptr(r) if pen else None, ptr(f) if pen else None, ptr(q) if pen else None,
                ptr(sl) if pen else None, ptr(table) if pen else None, table.stride(0) if pen else 0, out.data_ptr(), ptr(lp), n,
                top_ids.data_ptr() if n else None, top_lp.data_ptr() if n else None, _stream(logits)), "sample_tokens")
    return out if logprobs is None else (out, lp, top_ids, top_lp)


def _sample_draft(logits, t, k, p, key, ctr, min_p, logprobs, drafts):
    import numpy as np
    b, v = logits.shape
    dev = logits.device
    if isinstance(drafts, torch.Tensor):
        _req_cuda(drafts)
        if drafts.dtype != torch.int32 or tuple(drafts.shape) != (b,) or drafts.device != dev:
            raise RuntimeError(f"atom_b200.ops.sample_tokens: `drafts` must be int32 [{b}] on {dev}")
        d = drafts
    else:
        a = np.asarray(drafts, dtype=np.int64).reshape(-1)
        if a.shape != (b,) or (a < -1).any() or (a >= v).any():
            raise RuntimeError(f"atom_b200.ops.sample_tokens: `drafts` must hold {b} entries in [-1, {v})")
        d = torch.from_numpy(a.astype(np.int32)).to(dev)
    m = None if _neutral(min_p, 0) else _sample_param("min_p", min_p, b, torch.float32, dev, lambda a: ~((a >= 0) & (a <= 1)))
    n = 0 if logprobs is None else int(logprobs)
    out = torch.empty((b,), dtype=torch.int32, device=dev)
    lp = torch.empty((b,), dtype=torch.float32, device=dev) if logprobs is not None else None
    top_ids = torch.empty((b, n), dtype=torch.int32, device=dev)
    top_lp = torch.empty((b, n), dtype=torch.float32, device=dev)
    if b:
        ptr = lambda x: None if x is None else x.data_ptr()      # noqa: E731
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().atom_sample_draft_f16(
                logits.data_ptr(), logits.stride(0) if b > 1 else v, b, v, t.data_ptr(), k.data_ptr(), p.data_ptr(), key.data_ptr(),
                ctr.data_ptr(), ptr(m), out.data_ptr(), ptr(lp), n, top_ids.data_ptr() if n else None,
                top_lp.data_ptr() if n else None, d.data_ptr(), _stream(logits)), "sample_tokens")
    return out if logprobs is None else (out, lp, top_ids, top_lp)


SPEC_MAX_DRAFT = 7
SPEC_MAX_NGRAM = 16


def spec_history(slots, cap, device):
    """EXTENSION (speculative decoding): zeroed token histories for `slots` sequences of up to `cap` tokens each, for
    spec_commit_propose: (history int32 [slots, cap], lengths int32 [slots])."""
    if int(slots) < 1 or int(cap) < 1 or int(cap) >= 1 << 31:
        raise RuntimeError(f"atom_b200.ops.spec_history: need slots >= 1 and cap in [1, 2^31), got {slots}, {cap}")
    return (torch.zeros((int(slots), int(cap)), dtype=torch.int32, device=device),
            torch.zeros((int(slots),), dtype=torch.int32, device=device))


def spec_init_slot(history, lengths, slot, context):
    """EXTENSION: set slot `slot` of a token history to `context` (a request's whole context: a shared system prompt, then its
    own prompt), by a plain device copy."""
    if not 0 <= int(slot) < history.size(0) or len(context) > history.size(1):
        raise RuntimeError(f"atom_b200.ops.spec_init_slot: slot {slot} outside [0, {history.size(0)}) or a context of "
                           f"{len(context)} tokens past cap {history.size(1)}")
    n = len(context)
    if n:
        history[int(slot), :n].copy_(torch.tensor(list(context), dtype=torch.int32))
    lengths[int(slot)].fill_(n)


def spec_commit_propose(tokens, cands, row_indptr, slots, history, lengths, out, num_draft, ngram_min, ngram_max):
    """EXTENSION (atom_spec_commit_propose; DESIGN section 5.8): after a (verify) sampling step, per sequence i owning rows
    row_indptr[i] .. row_indptr[i+1] of `tokens` (the sampler's output) and `cands` (the candidates it was given, -1: none):
    commit the accepted tokens to its history slot slots[i] and propose up to num_draft drafts by prompt lookup (the longest
    n-gram in [ngram_min, ngram_max] whose latest earlier occurrence in the history matches its tail).  All int32 CUDA tensors;
    tokens and cands [R], row_indptr [B+1], slots [B], history / lengths as spec_history makes them, out [B, 2 * num_draft + 3]
    receives (emitted, draft_len, tokens [num_draft + 1], drafts [num_draft]), padded with -1.  Allocates nothing, so a CUDA
    graph may capture it.  slots given as a host sequence are checked to lie in range and be distinct."""
    k, nmin, nmax = int(num_draft), int(ngram_min), int(ngram_max)
    if not (1 <= k <= SPEC_MAX_DRAFT and 1 <= nmin <= nmax <= SPEC_MAX_NGRAM):
        raise RuntimeError(f"atom_b200.ops.spec_commit_propose: need 1 <= num_draft <= {SPEC_MAX_DRAFT} and "
                           f"1 <= ngram_min <= ngram_max <= {SPEC_MAX_NGRAM}, got {k}, {nmin}, {nmax}")
    _req_cuda(tokens, cands, row_indptr, history, lengths, out)
    b = row_indptr.numel() - 1
    nslots, cap = history.shape
    if b < 1 or any(x.dtype != torch.int32 or not x.is_contiguous() for x in (tokens, cands, row_indptr, history, lengths, out)):
        raise RuntimeError("atom_b200.ops.spec_commit_propose: all tensors must be contiguous int32, with at least one sequence")
    if tokens.shape != cands.shape or tuple(lengths.shape) != (nslots,) or tuple(out.shape) != (b, 2 * k + 3):
        raise RuntimeError(f"atom_b200.ops.spec_commit_propose: tokens and cands [R], lengths [{nslots}], out [{b}, {2 * k + 3}]")
    if cap < k + 1:
        raise RuntimeError(f"atom_b200.ops.spec_commit_propose: cap={cap} must hold at least num_draft + 1 tokens")
    if not isinstance(slots, torch.Tensor):
        import numpy as np
        a = np.asarray(slots, dtype=np.int64).reshape(-1)
        if a.shape != (b,) or (a < 0).any() or (a >= nslots).any() or len(np.unique(a)) != b:
            raise RuntimeError(f"atom_b200.ops.spec_commit_propose: `slots` must hold {b} distinct entries in [0, {nslots})")
        slots = torch.from_numpy(a.astype(np.int32)).to(history.device)
    elif slots.dtype != torch.int32 or tuple(slots.shape) != (b,) or not slots.is_cuda:
        raise RuntimeError(f"atom_b200.ops.spec_commit_propose: `slots` must be int32 [{b}]")
    with torch.cuda.device(history.device):
        _lib.check(_lib.lib().atom_spec_commit_propose(tokens.data_ptr(), cands.data_ptr(), row_indptr.data_ptr(), slots.data_ptr(), b,
                                                       history.data_ptr(), lengths.data_ptr(), nslots, cap, k, nmin, nmax,
                                                       out.data_ptr(), _stream(history)), "spec_commit_propose")
    return out


BEAM_MAX_WIDTH = 8
BEAM_MAX_STOP = 8
_BEAM_LIST = BEAM_MAX_WIDTH + BEAM_MAX_STOP


def beam_out(batch, width, device):
    """A packed output buffer for beam_select: int32 [6 * batch * width]."""
    return torch.empty(6 * int(batch) * int(width), dtype=torch.int32, device=device)


def split_beam_out(out, batch, width):
    """The four views of a packed beam_select buffer (a CUDA tensor or a host array): live [B, W, 2], live_key [B, W] (float32),
    fin [B, W, 2], fin_key [B, W] (float32)."""
    n = int(batch) * int(width)
    if isinstance(out, torch.Tensor):
        f32 = lambda x: x.view(torch.float32)      # noqa: E731
    else:
        import numpy as np
        f32 = lambda x: x.view(np.float32)         # noqa: E731
    return (out[:2 * n].reshape(batch, width, 2), f32(out[2 * n:3 * n]).reshape(batch, width),
            out[3 * n:5 * n].reshape(batch, width, 2), f32(out[5 * n:6 * n]).reshape(batch, width))


def beam_select(logits, row_indptr, sums, width, stop_ids=(), *, out=None, workspace=None):
    """EXTENSION (atom_beam_select_f16; DESIGN section 5.9): one beam-search step.  logits float16 [R, V] (unit stride along V),
    row_indptr int32 [B + 1] (request i owns rows row_indptr[i] .. row_indptr[i+1]; zero rows pads), sums float32 [R] (each row's
    beam's running sum), all on one CUDA device; width W in [1, 8]; stop_ids at most 8 host ids in [0, V).  Returns (live [B, W, 2]
    of (row, token), live_key [B, W], fin [B, W, 2], fin_key [B, W]), padded with -1: each request's live beams and the stop
    candidates of rank < W, in order (include/atom_b200.h).  out (beam_out) and workspace (uint8 >= R * 192 bytes, 16-byte
    aligned) may be given, so that a CUDA graph captures no allocation; the four tensors are then views of out."""
    w = int(width)
    stops = [int(t) for t in stop_ids]
    if not 1 <= w <= BEAM_MAX_WIDTH:
        raise RuntimeError(f"atom_b200.ops.beam_select: width must be in [1, {BEAM_MAX_WIDTH}], got {width}")
    _req_cuda(row_indptr, sums)
    if not (isinstance(logits, torch.Tensor) and logits.is_cuda and logits.dtype == torch.float16 and logits.dim() == 2
            and logits.stride(1) == 1):
        raise RuntimeError("atom_b200.ops.beam_select: logits must be float16 [R, V] on a CUDA device with unit stride along V")
    r, v = logits.shape
    b = row_indptr.numel() - 1
    dev = logits.device
    if row_indptr.dtype != torch.int32 or row_indptr.dim() != 1 or b < 1 or row_indptr.device != dev:
        raise RuntimeError(f"atom_b200.ops.beam_select: row_indptr must be int32 [B + 1] with B >= 1 on {dev}")
    if sums.dtype != torch.float32 or tuple(sums.shape) != (r,) or sums.device != dev:
        raise RuntimeError(f"atom_b200.ops.beam_select: sums must be float32 [{r}] on {dev}")
    if len(stops) > BEAM_MAX_STOP or len(set(stops)) != len(stops) or any(not 0 <= t < v for t in stops) or len(stops) >= v:
        raise RuntimeError(f"atom_b200.ops.beam_select: stop_ids must be at most {BEAM_MAX_STOP} distinct ids in [0, {v}), fewer "
                           f"than the vocabulary, got {stop_ids!r}")
    if out is None:
        out = beam_out(b, w, dev)
    elif out.dtype != torch.int32 or out.numel() != 6 * b * w or not out.is_contiguous() or out.device != dev:
        raise RuntimeError(f"atom_b200.ops.beam_select: out must be contiguous int32 [{6 * b * w}] on {dev}")
    if workspace is None:
        workspace = torch.empty(max(1, r) * _BEAM_LIST * 12, dtype=torch.uint8, device=dev)
    elif workspace.numel() * workspace.element_size() < r * _BEAM_LIST * 12 or not workspace.is_contiguous() or workspace.device != dev:
        raise RuntimeError(f"atom_b200.ops.beam_select: workspace must hold {r * _BEAM_LIST * 12} contiguous bytes on {dev}")
    live, live_key, fin, fin_key = split_beam_out(out, b, w)
    import ctypes
    arr = (ctypes.c_int * max(1, len(stops)))(*stops)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().atom_beam_select_f16(logits.data_ptr(), logits.stride(0) if r > 1 else v, r, v, row_indptr.data_ptr(), b,
                                                   sums.data_ptr(), arr, len(stops), w, workspace.data_ptr(), live.data_ptr(),
                                                   live_key.data_ptr(), fin.data_ptr(), fin_key.data_ptr(), _stream(logits)),
                   "beam_select")
    return live, live_key, fin, fin_key


def copy_kv_pages(pool, src, dst, slots):
    """EXTENSION (atom_kv_copy_pages_i4; DESIGN section 5.9): in one launch, copy the first slots[p] token slots of page src[p] to
    page dst[p] in every layer, K/V and head block of pool.buf and pool.param (a kvcache.KvPoolInt4, or anything with those two
    tensors).  src, dst, slots: int32 CUDA tensors [n] (read on the device, so a CUDA graph replays with new pairs; src < 0 is
    padding), or host sequences, which are checked: src != dst, pages in range, slots in [1, page size]."""
    buf, param = pool.buf, pool.param
    _req_cuda(buf, param)
    pages, layers, two, heads, P, half = buf.shape
    if buf.dtype != torch.uint8 or half != 64 or two != 2 or tuple(param.shape) != (pages, layers, 2, heads, P, 2) or \
            param.dtype != torch.float16:
        raise RuntimeError("atom_b200.ops.copy_kv_pages: pool.buf must be uint8 [pages, L, 2, H, P, 64] and pool.param float16 "
                           "[pages, L, 2, H, P, 2]")
    dev = buf.device
    pairs = []
    for name, x in (("src", src), ("dst", dst), ("slots", slots)):
        if isinstance(x, torch.Tensor):
            _req_cuda(x)
            if x.dtype != torch.int32 or x.dim() != 1 or x.device != dev:
                raise RuntimeError(f"atom_b200.ops.copy_kv_pages: `{name}` must be int32 [n] on {dev}")
            pairs.append(x)
        else:
            pairs.append(list(x))
    n = len(pairs[0])
    if any(len(x) != n for x in pairs):
        raise RuntimeError("atom_b200.ops.copy_kv_pages: src, dst and slots must have one entry per pair")
    if not isinstance(pairs[0], torch.Tensor) and not any(isinstance(x, torch.Tensor) for x in pairs):
        for s, d, k in zip(*pairs):
            if s >= 0 and (s == d or not 0 <= d < pages or s >= pages or not 1 <= k <= P):
                raise RuntimeError(f"atom_b200.ops.copy_kv_pages: pair ({s}, {d}, {k}) needs src != dst, pages in [0, {pages}) "
                                   f"and slots in [1, {P}]")
    if n == 0:
        return
    pairs = [x if isinstance(x, torch.Tensor) else torch.tensor(x, dtype=torch.int32).to(dev) for x in pairs]
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().atom_kv_copy_pages_i4(buf.data_ptr(), param.data_ptr(), pages, layers, heads, P, pairs[0].data_ptr(),
                                                    pairs[1].data_ptr(), pairs[2].data_ptr(), n, _stream(buf)), "copy_kv_pages")
