"""Simulated (model/) layer -> real-INT4 serving layer (e2e/).  No reference equivalent: the reference's e2e harness runs
random INT4 weights (e2e/README.md) and its accuracy simulator never leaves FP16; this module is the missing bridge, so
a layer calibrated with the model/ surface (QLlamaDecoderLayer) can be served by the sm_90a kernels.

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


@torch.no_grad()
def int4_decoder_layer(qlayer, device="cuda", layer_idx=0):
    """QLlamaDecoderLayer -> atom_b200.llama.LlamaDecoderLayer with identical quantised weights and reorder indices.
    MHA only (num_key_value_heads == num_heads), head_dim 128 -- the shapes the INT4 KV kernels support."""
    at = qlayer.self_attn
    assert at.num_key_value_heads == at.num_heads, "the INT4 paged-KV kernels are MHA (as the reference's)"
    assert at.head_dim == 128, "head_dim must be 128 (KV quantisation group)"
    hidden = at.hidden_size
    inter = qlayer.mlp.gate_proj.weight.shape[0]
    norm = qlayer.input_layernorm.originalNorm
    cfg = LlamaConfig(hidden_size=hidden, intermediate_size=inter, num_attention_heads=at.num_heads, num_hidden_layers=1,
                      rms_norm_eps=float(getattr(norm, "variance_epsilon", getattr(norm, "eps", 1e-6))))
    layer = LlamaDecoderLayer(cfg, layer_idx)
    for name in ("q_proj", "k_proj", "v_proj", "o_proj"):
        fill_linear_int4(getattr(layer.self_attn, name), getattr(at, name))
    for name in ("gate_proj", "up_proj", "down_proj"):
        fill_linear_int4(getattr(layer.mlp, name), getattr(qlayer.mlp, name))
    for dst, src in ((layer.input_layernorm, qlayer.input_layernorm), (layer.post_attention_layernorm, qlayer.post_attention_layernorm)):
        dst.weight.copy_(src.originalNorm.weight.detach().to(torch.float16))
        dst.reorder_index.copy_(_index_i16(src.reorder_index, hidden))
    layer.self_attn.reorder_index.copy_(_index_i16(at.reorder_index, hidden))
    return layer.to(device) if device is not None else layer
