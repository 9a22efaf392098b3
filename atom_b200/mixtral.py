"""Real-INT4 Mixtral decoder layer on the CUDA kernels: the attention is llama.LlamaAttention (grouped-query, RoPE base from the
config), the MLP is a sparse mixture of experts -- FP router, top-k routing, the experts' W4A4 GEMMs as two grouped launches,
weighted combine (csrc/moe_kernels.cuh).

Conventions (modelutils.reorder_model_mixtral): every expert shares expert 0's channel orders, so post_attention_layernorm's
quantised output is the input of EVERY expert and only its rows are permuted; the router (`gate`) is never quantised and reads
the FP16 normalised row in the same reordered order.  Expert operands are stacked over the experts, gate (w1) and up (w3) row
concatenated per expert:
    w13_int4 u8 [E, 2I, (H-128)/2]  w13_int8 i8 [E, 2I, 128]  w13_scale f16 [E, H/128-1, 2I]  w13_keeper_scale f16 [E, 2I]
    w2_int4  u8 [E, H, (I-128)/2]   w2_int8  i8 [E, H, 128]   w2_scale  f16 [E, I/128-1, H]   w2_keeper_scale  f16 [E, H]
    router_weight f16 [E, H]
"""
import math
from dataclasses import dataclass

import torch
from torch import nn

from . import ops
from .cat_tensor import BatchLenInfo
from .llama import LlamaAttention, LlamaRMSNormInt4


@dataclass
class MixtralConfig:
    """Mixtral-8x7B by default; HuggingFace field names."""
    hidden_size: int = 4096
    intermediate_size: int = 14336
    num_attention_heads: int = 32
    num_key_value_heads: int = 8
    num_hidden_layers: int = 32
    num_local_experts: int = 8
    num_experts_per_tok: int = 2
    rms_norm_eps: float = 1e-5
    rope_theta: float = 1e6
    vocab_size: int = 32000
    pad_token_id: int = 0


class SparseMoeInt4(nn.Module):
    """The sparse MoE block.  forward(hidden_sum, x) takes the residual sum and its quantised post-attention norm (the pair
    LlamaRMSNormInt4.forward_add returns) and returns the FP16 MoE delta of the residual stream.  `norm` is the layer's
    post_attention_layernorm: the router normalises the residual sum with its weight, index and eps."""

    def __init__(self, config, norm: LlamaRMSNormInt4):
        super().__init__()
        h, i = config.hidden_size, config.intermediate_size
        e, k = config.num_local_experts, config.num_experts_per_tok
        if not (1 <= e <= 64 and 1 <= k <= min(e, 8)):
            raise ValueError(f"{e} experts, top-{k}: the MoE kernels serve up to 64 experts and top-k <= min(experts, 8)")
        if h % 128 or i % 128 or h < 256 or i < 256:
            raise ValueError("hidden_size and intermediate_size must be multiples of 128, at least 256")
        self.hidden_size, self.intermediate_size, self.num_experts, self.top_k = h, i, e, k
        self._norm = [norm]                  # shared with the decoder layer, not a child module (no second state_dict entry)
        p = lambda *shape, dtype: nn.Parameter(torch.empty(*shape, dtype=dtype), requires_grad=False)  # noqa: E731
        self.router_weight = p(e, h, dtype=torch.float16)
        self.w13_int4 = p(e, 2 * i, (h - 128) // 2, dtype=torch.uint8)
        self.w13_int8 = p(e, 2 * i, 128, dtype=torch.int8)
        self.w13_scale = p(e, h // 128 - 1, 2 * i, dtype=torch.float16)
        self.w13_keeper_scale = p(e, 2 * i, dtype=torch.float16)
        self.w2_int4 = p(e, h, (i - 128) // 2, dtype=torch.uint8)
        self.w2_int8 = p(e, h, 128, dtype=torch.int8)
        self.w2_scale = p(e, i // 128 - 1, h, dtype=torch.float16)
        self.w2_keeper_scale = p(e, h, dtype=torch.float16)

    @property
    def norm(self):
        return self._norm[0]

    @torch.no_grad()
    def init_random(self, seed=0):
        """Random-quantised experts and a random router (the magnitudes of LinearInt4.init_random)."""
        dev = self.w13_int4.device
        g = torch.Generator(device=dev).manual_seed(seed)
        for w4, w8, s4, s8, k in ((self.w13_int4, self.w13_int8, self.w13_scale, self.w13_keeper_scale, self.hidden_size),
                                  (self.w2_int4, self.w2_int8, self.w2_scale, self.w2_keeper_scale, self.intermediate_size)):
            w4.copy_(torch.randint(0, 256, w4.shape, dtype=torch.uint8, device=dev, generator=g))
            w8.copy_(torch.randint(-128, 128, w8.shape, dtype=torch.int8, device=dev, generator=g))
            s4.copy_((0.02 / 7 / math.sqrt(k) * 8) * (1 + torch.rand(s4.shape, device=dev, generator=g)))
            s8.copy_((0.02 / 127 / math.sqrt(k) * 8) * (1 + torch.rand(s8.shape, device=dev, generator=g)))
        self.router_weight.copy_(torch.randn(self.router_weight.shape, device=dev, generator=g) / math.sqrt(self.hidden_size))
        return self

    def route(self, hidden_sum, router_logits=False):
        n = self.norm
        return ops.moe_route_f16(hidden_sum, n.weight, n.reorder_index, n.variance_epsilon, self.router_weight, self.top_k,
                                 router_logits=router_logits)

    def forward(self, hidden_sum, x):
        ids, w = self.route(hidden_sum)
        return self.experts(x, ids, w)

    def experts(self, x, topk_ids, topk_weights):
        """The expert path for a given routing: plan, gather, grouped gate/up+act, grouped down, combine."""
        bn, tiles_max, rows_cap = ops.moe_tiles(topk_ids.size(0), self.num_experts, self.top_k)
        dest, tiles = ops.moe_plan(topk_ids, self.num_experts, bn, tiles_max)
        xp = ops.moe_gather_i4(x, dest, rows_cap)
        act = ops.dense_layer_gemm_i4_gateup_act_grouped(xp, self.w13_int4, self.w13_scale, self.w13_int8, self.w13_keeper_scale, tiles, bn)
        y = ops.dense_layer_gemm_i4_fp16_grouped(act, self.w2_int4, self.w2_scale, self.w2_int8, self.w2_keeper_scale, tiles, bn)
        return ops.moe_combine_f16(y, topk_ids, topk_weights, dest)


class MixtralDecoderLayer(nn.Module):
    """LlamaDecoderLayer with the MLP replaced by SparseMoeInt4: same forward / forward_residual contract."""

    def __init__(self, config, layer_idx: int):
        super().__init__()
        self.hidden_size = config.hidden_size
        self.self_attn = LlamaAttention(config=config, layer_idx=layer_idx)
        self.input_layernorm = LlamaRMSNormInt4(config.hidden_size, eps=config.rms_norm_eps)
        self.post_attention_layernorm = LlamaRMSNormInt4(config.hidden_size, eps=config.rms_norm_eps)
        self.block_sparse_moe = SparseMoeInt4(config, self.post_attention_layernorm)

    def init_random(self, seed=0):
        from .llama import LinearInt4
        for i, m in enumerate(mod for mod in self.self_attn.modules() if isinstance(mod, LinearInt4)):
            m.init_random(seed * 16 + i)
        self.block_sparse_moe.init_random(seed * 16 + 8)
        if self.self_attn.q_proj.weight_int4.is_cuda:
            self.fuse()
        return self

    def fuse(self):
        self.self_attn.fuse()
        return self

    def forward(self, hidden_states, blen: BatchLenInfo, prefill_kv, decode_kv) -> torch.Tensor:
        hidden_states, delta = self.forward_residual(hidden_states, None, blen, prefill_kv, decode_kv)
        return hidden_states + delta

    def forward_residual(self, residual, delta, blen: BatchLenInfo, prefill_kv, decode_kv):
        """As LlamaDecoderLayer.forward_residual; the returned delta is the MoE block's output."""
        if delta is None:
            x = self.input_layernorm(residual)
        else:
            residual, x = self.input_layernorm.forward_add(delta, residual)
        attn = self.self_attn(x, blen, prefill_kv, decode_kv)
        residual, x = self.post_attention_layernorm.forward_add(attn, residual)
        return residual, self.block_sparse_moe(residual, x)
