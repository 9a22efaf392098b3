"""Simulated (model/) layer -> real-INT4 serving layer (e2e/).  No reference equivalent: the reference's e2e harness runs
random INT4 weights (e2e/README.md) and its accuracy simulator never leaves FP16; this module is the missing bridge, so
a layer calibrated with the model/ surface (QLlamaDecoderLayer, QMixtralDecoderLayer) can be served by the sm_90a kernels -- multi-head or
grouped-query attention (Llama-2-70B, Llama-3 shapes: fewer k/v rows, a KV cache of KV heads), with the layer's RoPE base.

Operand conventions are the kernels' (include/atom_b200.h; e2e/punica-atom/punica/models/llama.py:35-58):
  weight_int4 u8 [out, (in-128)/2]   reordered input channel 2j in the low nibble of byte j
  weight_int8 i8 [out, 128]          the last 128 reordered input channels (the keeper)
  scale_int4 f16 [in/128-1, S(out)]  allocated like the reference, but READ as flat [group][out] (pitch `out`)
  scale_int8 f16 [S(out)]
"""
import torch

from . import ops
from .llama import LinearInt4, LlamaConfig, LlamaDecoderLayer


@torch.no_grad()
def fill_linear_int4(dst: LinearInt4, q):
    """Copy a QLinearLayer's real-INT4 operands into a LinearInt4 (the simulated layer is left untouched)."""
    op = q.int4_operands()
    out_f, in_f = dst.out_features, dst.in_features
    assert tuple(op["weight_int4"].shape) == (out_f, (in_f - 128) // 2), (op["weight_int4"].shape, out_f, in_f)
    dst.weight_int4.copy_(op["weight_int4"])
    dst.weight_int8.copy_(op["weight_int8"])
    dst.scale_int4.zero_()
    dst.scale_int8.zero_()
    # the kernels address B scales as flat [group][out] (pitch = out); LinearInt4 merely over-allocates rows of S(out)
    dst.scale_int4.view(-1)[: op["scale_int4"].numel()].copy_(op["scale_int4"].reshape(-1))
    dst.scale_int8[:out_f].copy_(op["scale_int8"])
    return dst


def _index_i16(idx, n):
    if idx is None:
        return torch.arange(n, dtype=torch.int16)
    assert idx.numel() == n and n <= 32768
    return idx.to(torch.int16).cpu()


def _orig_norm(n):
    """The FP RMSNorm a simulated norm wraps (QLlamaRMSNorm.originalNorm, QMixtralRMSNorm.originalRMSNorm)."""
    return n.originalNorm if hasattr(n, "originalNorm") else n.originalRMSNorm


def _attention_config(qlayer):
    """(attention module, config fields of the served layer) shared by the Llama and the Mixtral export."""
    at = qlayer.self_attn
    if at.num_heads % at.num_key_value_heads or at.num_heads // at.num_key_value_heads not in (1, 2, 4, 8):
        raise ValueError(f"{at.num_heads} query heads over {at.num_key_value_heads} KV heads: the INT4 paged-KV decode kernel serves "
                         f"1, 2, 4 or 8 query heads per KV head")
    assert at.head_dim == 128, "head_dim must be 128 (KV quantisation group)"
    theta = getattr(at, "rope_theta", None) or getattr(getattr(at, "config", None), "rope_theta", None) or 10000.0
    norm = _orig_norm(qlayer.input_layernorm)
    return at, dict(hidden_size=at.hidden_size, num_attention_heads=at.num_heads, num_hidden_layers=1,
                    rms_norm_eps=float(getattr(norm, "variance_epsilon", getattr(norm, "eps", 1e-6))),
                    rope_theta=float(theta))


def _fill_attention_and_norms(layer, qlayer, at):
    hidden = at.hidden_size
    for name in ("q_proj", "k_proj", "v_proj", "o_proj"):
        fill_linear_int4(getattr(layer.self_attn, name), getattr(at, name))
    for dst, src in ((layer.input_layernorm, qlayer.input_layernorm), (layer.post_attention_layernorm, qlayer.post_attention_layernorm)):
        dst.weight.copy_(_orig_norm(src).weight.detach().to(torch.float16))
        dst.reorder_index.copy_(_index_i16(src.reorder_index, hidden))
    layer.self_attn.reorder_index.copy_(_index_i16(at.reorder_index, hidden))


@torch.no_grad()
def int4_decoder_layer(qlayer, device="cuda", layer_idx=0):
    """QLlamaDecoderLayer -> atom_b200.llama.LlamaDecoderLayer with identical quantised weights and reorder indices.
    Multi-head or grouped-query attention (num_heads / num_key_value_heads in {1, 2, 4, 8}: the group sizes the INT4 paged-KV
    decode kernel serves), head_dim 128; the layer's RoPE base (`rope_theta` of the attention module or its config, default 1e4)
    is carried into the exported config."""
    at, fields = _attention_config(qlayer)
    inter = qlayer.mlp.gate_proj.weight.shape[0]
    cfg = LlamaConfig(intermediate_size=inter, num_key_value_heads=None if at.num_key_value_heads == at.num_heads else int(at.num_key_value_heads),
                      **fields)
    layer = LlamaDecoderLayer(cfg, layer_idx)
    _fill_attention_and_norms(layer, qlayer, at)
    for name in ("gate_proj", "up_proj", "down_proj"):
        fill_linear_int4(getattr(layer.mlp, name), getattr(qlayer.mlp, name))
    return layer.to(device) if device is not None else layer


@torch.no_grad()
def int4_mixtral_decoder_layer(qlayer, device="cuda", layer_idx=0):
    """QMixtralDecoderLayer -> atom_b200.mixtral.MixtralDecoderLayer.  Attention and norms as int4_decoder_layer; every expert's
    w1 / w3 (gate / up) operands go into its slice of the stacked w13 tensors (gate rows first), w2 into w2; the router weight
    (already in post_attention_layernorm's channel order) becomes an FP16 [E, H] matrix."""
    from .mixtral import MixtralConfig, MixtralDecoderLayer
    at, fields = _attention_config(qlayer)
    moe = qlayer.block_sparse_moe
    inter = moe.experts[0].w1.weight.shape[0]
    cfg = MixtralConfig(intermediate_size=inter, num_key_value_heads=int(at.num_key_value_heads), num_local_experts=int(moe.num_experts),
                        num_experts_per_tok=int(moe.top_k), **fields)
    layer = MixtralDecoderLayer(cfg, layer_idx)
    _fill_attention_and_norms(layer, qlayer, at)
    dst = layer.block_sparse_moe
    for e, ex in enumerate(moe.experts):
        ops13 = [ex.w1.int4_operands(), ex.w3.int4_operands()]
        dst.w13_int4[e].copy_(torch.cat([o["weight_int4"] for o in ops13], 0))
        dst.w13_int8[e].copy_(torch.cat([o["weight_int8"] for o in ops13], 0))
        dst.w13_scale[e].copy_(torch.cat([o["scale_int4"] for o in ops13], 1))
        dst.w13_keeper_scale[e].copy_(torch.cat([o["scale_int8"] for o in ops13], 0))
        o2 = ex.w2.int4_operands()
        dst.w2_int4[e].copy_(o2["weight_int4"])
        dst.w2_int8[e].copy_(o2["weight_int8"])
        dst.w2_scale[e].copy_(o2["scale_int4"])
        dst.w2_keeper_scale[e].copy_(o2["scale_int8"])
    dst.router_weight.copy_(moe.gate.weight.detach().to(torch.float16))
    return layer.to(device) if device is not None else layer
