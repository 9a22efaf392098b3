"""Tensor parallelism for the W4A4 layers (BASELINE config #5: Llama-65B over 8 GPUs).  NEW functionality: the reference
has no NCCL / torch.distributed code at all (SURVEY.md section 0.3), so there is nothing to be drop-in with; the layout
follows Megatron: one process per GPU, column-parallel q/k/v/gate/up (no communication), row-parallel o_proj/down_proj
followed by ONE all-reduce (NCCL over NVLink/NVSwitch) per column->row pair -- two per decoder layer.

Row-parallel quantisation is shard-local: a rank's K-slice is a complete W4A4 operand of its own (its own reorder
permutation, INT4 groups and 128-channel INT8 keeper), so activations never have to be gathered:
    y = all_reduce( gemm_i4(quantise(x_local[:, perm_r]), W_r) )
Slices are cut on 128-channel group boundaries; uneven splits are allowed (22016 / 8 = 21.5 groups -> 22 / 21 groups).
"""
from typing import List, Optional

import torch
import torch.distributed as dist
from torch import nn

from . import ops
from .llama import LinearInt4, fuse_linear_rows


def split_sizes(total: int, world: int, quantum: int = 128, minimum: int = 256) -> List[int]:
    """Cut `total` channels into `world` contiguous slices that are multiples of `quantum`, as even as possible
    (larger slices first).  Every slice must hold at least one INT4 group plus the keeper (>= 256)."""
    if total % quantum:
        raise ValueError(f"{total} is not a multiple of {quantum}")
    units = total // quantum
    base, extra = divmod(units, world)
    sizes = [(base + (1 if r < extra else 0)) * quantum for r in range(world)]
    if min(sizes) < minimum:
        raise ValueError(f"cannot split {total} channels over {world} ranks: slice of {min(sizes)} < {minimum}")
    return sizes


def slice_range(sizes: List[int], rank: int):
    beg = sum(sizes[:rank])
    return beg, beg + sizes[rank]


class ColumnParallelLinearInt4(LinearInt4):
    """Output channels [n0, n1) of a LinearInt4.  Input: the replicated quantised activation 4-tuple."""

    def __init__(self, in_features, out_features, out_dtype, rank, world, quantum=128):
        self.full_out = out_features
        self.sizes = split_sizes(out_features, world, quantum, minimum=quantum)
        self.n0, self.n1 = slice_range(self.sizes, rank)
        super().__init__(in_features, self.n1 - self.n0, out_dtype)

    @torch.no_grad()
    def load_full(self, full: LinearInt4):
        self.weight_int4.copy_(full.weight_int4[self.n0:self.n1])
        self.weight_int8.copy_(full.weight_int8[self.n0:self.n1])
        g = full.scale_int4.shape[0]
        flat = full.scale_int4.reshape(-1)[: g * full.out_features].view(g, full.out_features)   # kernels address [G][N]
        mine = self.scale_int4.reshape(-1)[: g * self.out_features].view(g, self.out_features)
        mine.copy_(flat[:, self.n0:self.n1])
        self.scale_int8[: self.out_features].copy_(full.scale_int8[self.n0:self.n1])
        return self


class RowParallelLinearInt4(nn.Module):
    """Input channels [k0, k1) of a linear layer as a self-contained W4A4 operand + all-reduce of the partial outputs."""

    def __init__(self, in_features, out_features, rank, world, group: Optional[dist.ProcessGroup] = None, gemm_fn=None,
                 allreduce=None):
        super().__init__()
        self.sizes = split_sizes(in_features, world)
        self.k0, self.k1 = slice_range(self.sizes, rank)
        self.local = LinearInt4(self.k1 - self.k0, out_features, out_dtype="fp16")
        self.world, self.group = world, group
        self.gemm_fn = gemm_fn
        self.allreduce = allreduce       # comm.PushAllReduce / NcclAllReduce; None = plain dist.all_reduce

    def can_push(self, batch):
        """Fused all-reduce (GEMM epilogue pushes, the following add+RMSNorm reduces): push kernel, decode batch, wide rows."""
        return (self.world > 1 and self.gemm_fn is None and getattr(self.allreduce, "handle", None) is not None
                and getattr(self.allreduce, "fuse", False) and batch <= 64
                and self.local.out_features % 1024 == 0 and batch * self.local.out_features <= self.allreduce.slot)

    def forward_push(self, local_tuple):
        """The GEMM only; its partial goes straight into every rank's receive buffer.  The caller must hand the returned
        ops.PendingAllReduce to LlamaRMSNormInt4.forward_add before anything else uses this all-reduce object."""
        outlier, norms, outlier_scales, norm_scales = local_tuple
        return ops.dense_layer_gemm_i4_fp16_push(norms, self.local.weight_int4, norm_scales, self.local.scale_int4, outlier,
                                                 self.local.weight_int8, outlier_scales, self.local.scale_int8, self.allreduce.handle)

    def forward(self, local_tuple):
        outlier, norms, outlier_scales, norm_scales = local_tuple
        f = self.gemm_fn or ops.dense_layer_gemm_i4_fp16
        y = f(norms, self.local.weight_int4, norm_scales, self.local.scale_int4, outlier, self.local.weight_int8,
              outlier_scales, self.local.scale_int8)
        if self.world > 1:                   # the one collective of the column->row pair
            if self.allreduce is not None:
                y = self.allreduce(y)
            else:
                dist.all_reduce(y, op=dist.ReduceOp.SUM, group=self.group)
        return y


class TPLlamaDecoderLayer(nn.Module):
    """One Llama decoder layer over `world` ranks: heads and MLP channels are sharded, hidden states replicated.
    forward(hidden, decode_kv) runs a decode step (one token per sequence); KV cache pools are per rank (local KV heads:
    with grouped-query attention a rank holds num_key_value_heads / world of them and their query heads)."""

    def __init__(self, config, layer_idx, rank, world, group=None, allreduce=None):
        super().__init__()
        from .llama import LlamaRMSNormInt4
        h, nh = config.hidden_size, config.num_attention_heads
        if nh % world:
            raise ValueError("num_attention_heads must be divisible by the tensor-parallel size")
        nkv = getattr(config, "num_key_value_heads", None) or nh
        if nkv % world:      # KV heads are sharded with the query heads of their groups; they are not replicated
            raise ValueError("num_key_value_heads must be divisible by the tensor-parallel size")
        self.rank, self.world, self.layer_idx = rank, world, layer_idx
        self.local_heads, self.local_kv_heads = nh // world, nkv // world
        self.rope_theta = float(getattr(config, "rope_theta", 10000.0))
        hl, hkvl = self.local_heads * 128, self.local_kv_heads * 128
        self.q_proj = LinearInt4(h, hl, "fp16")
        self.k_proj = LinearInt4(h, hkvl, "int4")
        self.v_proj = LinearInt4(h, hkvl, "int4")
        self.o_proj = RowParallelLinearInt4(h, h, rank, world, group, allreduce=allreduce)
        assert self.o_proj.k1 - self.o_proj.k0 == hl, "head slices and o_proj K-slices must coincide"
        self.inter_sizes = split_sizes(config.intermediate_size, world)
        il = self.inter_sizes[rank]
        self.gate_proj = LinearInt4(h, il, "fp16")
        self.up_proj = LinearInt4(h, il, "fp16")
        self.down_proj = RowParallelLinearInt4(config.intermediate_size, h, rank, world, group, allreduce=allreduce)
        self.input_layernorm = LlamaRMSNormInt4(h, eps=config.rms_norm_eps)
        self.post_attention_layernorm = LlamaRMSNormInt4(h, eps=config.rms_norm_eps)
        self.attn_reorder_index = nn.Parameter(torch.randperm(hl, dtype=torch.int16), requires_grad=False)   # shard-local

    def init_random(self, seed=0):
        i = 0
        for m in self.modules():
            if isinstance(m, LinearInt4):
                m.init_random(seed * 64 + self.rank * 8 + i)
                i += 1
        if self.q_proj.weight_int4.is_cuda:
            self.fuse()
        return self

    def fuse(self):
        """Fused decode launches (ops.dense_layer_gemm_i4_qkv / _gateup_act) on this rank's shards."""
        self._qkv = fuse_linear_rows([self.q_proj, self.k_proj, self.v_proj])
        self._gu = fuse_linear_rows([self.gate_proj, self.up_proj])
        return self

    def forward(self, hidden_states, decode_kv):
        hidden_states, pending = self.forward_chain(hidden_states, None, decode_kv, last=True)
        return hidden_states

    def forward_chain(self, hidden_states, pending, decode_kv, last=False):
        """One decode step.  `pending`: the previous layer's down projection whose all-reduce has not been formed yet (it is, together
        with the residual add, inside this layer's input norm launch).  Returns (hidden_states, pending'): with last=False and a
        push-capable all-reduce the down projection of this layer is returned pending, otherwise it is reduced and added here."""
        b = hidden_states.shape[0]
        if pending is not None:
            hidden_states, x = self.input_layernorm.forward_add(pending, hidden_states)
        else:
            x = self.input_layernorm(hidden_states)
        fused = getattr(self, "_qkv", None) is not None and b <= 64
        if fused:
            w4, s4, w8, s8 = self._qkv
            kv_rows = None if self.local_kv_heads == self.local_heads else self.local_kv_heads * 128
            q, (k, ks), (v, vs) = ops.dense_layer_gemm_i4_qkv(x[1], w4, x[3], s4, x[0], w8, x[2], s8, kv_rows=kv_rows)
            q = q.view(b, self.local_heads, 128)
        else:
            q = self.q_proj(x).view(b, self.local_heads, 128)
            k, ks = self.k_proj(x)
            v, vs = self.v_proj(x)
        ops.append_kv_i4(decode_kv, k.view(b, self.local_kv_heads, 64), v.view(b, self.local_kv_heads, 64),
                         ks.view(b, self.local_kv_heads, 2), vs.view(b, self.local_kv_heads, 2), self.layer_idx)
        attn = ops.batch_decode_i4(q, decode_kv, self.layer_idx, rope_theta=self.rope_theta).view(b, self.local_heads * 128)
        o_in = ops.reorder_fp16_i4(attn, self.attn_reorder_index)
        o = self.o_proj.forward_push(o_in) if self.o_proj.can_push(b) else self.o_proj(o_in)                  # all-reduce #1
        hidden_states, x = self.post_attention_layernorm.forward_add(o, hidden_states)                        # residual add (+ reduce) folded into the norm
        if fused:
            w4, s4, w8, s8 = self._gu
            act = ops.dense_layer_gemm_i4_gateup_act(x[1], w4, x[3], s4, x[0], w8, x[2], s8)
        else:
            act = ops.activate_fp16_i4(self.gate_proj(x), self.up_proj(x))
        if not last and self.down_proj.can_push(b):
            return hidden_states, self.down_proj.forward_push(act)                                           # all-reduce #2, formed by the next layer's norm
        return hidden_states + self.down_proj(act), None                                                     # all-reduce #2
