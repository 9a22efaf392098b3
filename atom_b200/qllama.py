"""QLlamaDecoderLayer and friends -- the operator surface of /root/reference/model/qLlamaLayer.py:53-350.

This is the *accuracy-simulation* side of the hot path (SURVEY.md section 8(a), last row): FP16/FP32 tensors whose values
are snapped to the INT4/INT8 grids by Quantizer modules placed exactly where the real kernels quantise
(after each RMSNorm, before o_proj, before down_proj, K before RoPE, V before P.V).  modelutils_llama.py drives it through
attribute names, so the names are the interface:

    layer.input_layernorm / post_attention_layernorm : QLlamaRMSNorm  (.originalNorm, .act_quant, .reorder_index)
    layer.self_attn : QLlamaAttention (.q_proj .k_proj .v_proj .o_proj : QLinearLayer, .act_quant .k_quant .v_quant, .reorder_index)
    layer.mlp       : QLlamaMLP       (.gate_proj .up_proj .down_proj : QLinearLayer, .act_quant)

The wrapped "original" layer only has to expose HF-Llama attribute names (q_proj ... down_proj, the two norms, and either
the per-module sizes or a `.config` carrying them), so a transformers LlamaDecoderLayer of any vintage or the
ToyLlamaDecoderLayer below (used by the CPU tests -- there is no network for checkpoints) both work.

`QLlamaDecoderLayer.to_int4()` is the bridge the reference does not have: it turns the simulated layer into the real
INT4 serving layer (atom_b200.llama.LlamaDecoderLayer: fused norm+quantise, W4A4 wgmma GEMMs, INT4 paged KV).
"""
import math
from typing import Optional, Tuple

import torch
from torch import nn

from .qlinear import QLinearLayer
from .quant import Quantizer


def _cfg(obj, name, default=None):
    """Attribute from the module itself (transformers <= 4.3x) or from its config (newer releases)."""
    if hasattr(obj, name):
        return getattr(obj, name)
    cfg = getattr(obj, "config", None)
    alias = {"hidden_size": "hidden_size", "num_heads": "num_attention_heads", "num_key_value_heads": "num_key_value_heads",
             "max_position_embeddings": "max_position_embeddings", "rope_theta": "rope_theta", "attention_dropout": "attention_dropout"}
    if cfg is not None and hasattr(cfg, alias.get(name, name)):
        return getattr(cfg, alias.get(name, name))
    if default is not None:
        return default
    raise AttributeError(f"{type(obj).__name__} has neither .{name} nor .config.{alias.get(name, name)}")


def rope_cos_sin(position_ids, head_dim, theta, dtype):
    """cos/sin [bsz, seq, head_dim] in the rotate-half convention (LlamaRotaryEmbedding)."""
    inv = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float32, device=position_ids.device) / head_dim))
    ang = position_ids[..., None].float() * inv
    emb = torch.cat((ang, ang), dim=-1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def apply_rotary_pos_emb(q, k, cos, sin):
    cos, sin = cos.unsqueeze(1), sin.unsqueeze(1)
    return q * cos + rotate_half(q) * sin, k * cos + rotate_half(k) * sin


def repeat_kv(x, n_rep):
    if n_rep == 1:
        return x
    b, h, s, d = x.shape
    return x[:, :, None].expand(b, h, n_rep, s, d).reshape(b, h * n_rep, s, d)


def quantised_attention(mod, hidden_states, attention_mask, position_ids, past_key_value, output_attentions, use_cache):
    """The attention data flow shared by QLlamaAttention and QMixtralAttention (qLlamaLayer.py:228-310,
    qMixtralLayer.py:141-235): K is snapped to the INT4 grid *before* RoPE (the paged cache stores pre-RoPE K and
    the decode kernel rotates on load), V before P.V, the head-concatenated output is reordered and quantised for
    o_proj.  `past_key_value` is the legacy (key, value) tuple."""
    bsz, q_len, _ = hidden_states.shape
    q = mod.q_proj(hidden_states).view(bsz, q_len, mod.num_heads, mod.head_dim).transpose(1, 2)
    k = mod.k_proj(hidden_states).view(bsz, q_len, mod.num_key_value_heads, mod.head_dim).transpose(1, 2)
    v = mod.v_proj(hidden_states).view(bsz, q_len, mod.num_key_value_heads, mod.head_dim).transpose(1, 2)
    past = 0 if past_key_value is None else past_key_value[0].shape[-2]
    kv_len = q_len + past
    if mod.q_kv_cache:
        k = mod.k_quant(k)
    if position_ids is None:
        position_ids = torch.arange(past, kv_len, device=hidden_states.device)[None].expand(bsz, -1)
    if mod.rotary_emb is not None:
        cos, sin = mod.rotary_emb(v, position_ids)
    else:
        cos, sin = rope_cos_sin(position_ids, mod.head_dim, mod.rope_theta, q.dtype)
    q, k = apply_rotary_pos_emb(q, k, cos, sin)
    if past_key_value is not None:
        k = torch.cat([past_key_value[0], k], dim=2)
        v = torch.cat([past_key_value[1], v], dim=2)
    present = (k, v) if use_cache else None
    k = repeat_kv(k, mod.num_key_value_groups)
    v = repeat_kv(v, mod.num_key_value_groups)
    w = torch.matmul(q, k.transpose(2, 3)) / math.sqrt(mod.head_dim)
    if attention_mask is not None:
        if attention_mask.size() != (bsz, 1, q_len, kv_len):
            raise ValueError(f"Attention mask should be of size {(bsz, 1, q_len, kv_len)}, but is {attention_mask.size()}")
        w = w + attention_mask
    elif q_len > 1:                       # no mask given: causal, as every caller of a decoder layer means
        causal = torch.full((q_len, kv_len), float("-inf"), device=w.device, dtype=w.dtype).triu(1 + past)
        w = w + causal
    w = nn.functional.softmax(w, dim=-1, dtype=torch.float32).to(q.dtype)
    if mod.q_kv_cache:
        v = mod.v_quant(v)
    o = torch.matmul(w, v).transpose(1, 2).contiguous().reshape(bsz, q_len, mod.num_heads * mod.head_dim)
    if mod.reorder_index is not None:
        o = torch.index_select(o, 2, mod.reorder_index)
    o = mod.o_proj(mod.act_quant(o))
    return o, (w if output_attentions else None), present


class QLlamaRMSNorm(nn.Module):
    """qLlamaLayer.py:129-158: norm -> channel reorder -> activation quantise (the FP restatement of rmsnorm_fp16_i4)."""

    def __init__(self, originalNorm, args):
        super().__init__()
        self.originalNorm = originalNorm
        self.act_quant = Quantizer(args=args)
        self.register_buffer("reorder_index", None)
        self.args = args

    @torch.no_grad()
    def forward(self, hidden_states):
        result = self.originalNorm(hidden_states)
        if self.reorder_index is not None:
            assert result.shape[-1] == self.reorder_index.shape[0]
            result = torch.index_select(result, result.dim() - 1, self.reorder_index)
        if self.args.abits < 16:
            result = self.act_quant(result)
        return result


class QLlamaAttention(nn.Module):
    def __init__(self, originalAttn, args):
        super().__init__()
        self.abits = args.abits
        self.q_kv_cache = args.kv_cache
        self.config = getattr(originalAttn, "config", None)
        self.hidden_size = _cfg(originalAttn, "hidden_size")
        self.num_heads = _cfg(originalAttn, "num_heads")
        self.head_dim = self.hidden_size // self.num_heads
        self.num_key_value_heads = _cfg(originalAttn, "num_key_value_heads", self.num_heads)
        self.num_key_value_groups = self.num_heads // self.num_key_value_heads
        self.max_position_embeddings = _cfg(originalAttn, "max_position_embeddings", 4096)
        self.rope_theta = _cfg(originalAttn, "rope_theta", 10000.0)
        if self.head_dim * self.num_heads != self.hidden_size:
            raise ValueError(f"hidden_size must be divisible by num_heads (got `hidden_size`: {self.hidden_size}"
                             f" and `num_heads`: {self.num_heads}).")
        self.q_proj = QLinearLayer(originalAttn.q_proj, args)
        self.k_proj = QLinearLayer(originalAttn.k_proj, args)
        self.v_proj = QLinearLayer(originalAttn.v_proj, args)
        self.o_proj = QLinearLayer(originalAttn.o_proj, args)
        self.rotary_emb = getattr(originalAttn, "rotary_emb", None)
        self.act_quant = Quantizer(args=args)
        self.v_quant = Quantizer(args=args)
        self.k_quant = Quantizer(args=args)
        self.register_buffer("reorder_index", None)

    @torch.no_grad()
    def forward(self, hidden_states, attention_mask=None, position_ids=None, past_key_value=None, output_attentions=False,
                use_cache=False):
        return quantised_attention(self, hidden_states, attention_mask, position_ids, past_key_value, output_attentions, use_cache)


class QLlamaMLP(nn.Module):
    def __init__(self, originalMLP, args):
        super().__init__()
        self.gate_proj = QLinearLayer(originalMLP.gate_proj, args)
        self.down_proj = QLinearLayer(originalMLP.down_proj, args)
        self.up_proj = QLinearLayer(originalMLP.up_proj, args)
        self.act_fn = originalMLP.act_fn
        self.act_quant = Quantizer(args=args)

    @torch.no_grad()
    def forward(self, x):
        return self.down_proj(self.act_quant(self.act_fn(self.gate_proj(x)) * self.up_proj(x)))


class QLlamaDecoderLayer(nn.Module):
    def __init__(self, originalLayer, args):
        super().__init__()
        self.args = args
        self.hidden_size = _cfg(originalLayer, "hidden_size", originalLayer.self_attn.q_proj.weight.shape[1])
        self.self_attn = QLlamaAttention(originalLayer.self_attn, args)
        self.mlp = QLlamaMLP(originalLayer.mlp, args)
        self.input_layernorm = QLlamaRMSNorm(originalLayer.input_layernorm, args)
        self.post_attention_layernorm = QLlamaRMSNorm(originalLayer.post_attention_layernorm, args)

    @torch.no_grad()
    def forward(self, hidden_states, attention_mask=None, position_ids=None, past_key_value=None, output_attentions=False,
                use_cache=False, cache_position=None, padding_mask=None, **_):
        residual = hidden_states
        hidden_states, attn_w, present = self.self_attn(self.input_layernorm(hidden_states), attention_mask, position_ids,
                                                        past_key_value, output_attentions, use_cache)
        hidden_states = residual + hidden_states
        hidden_states = hidden_states + self.mlp(self.post_attention_layernorm(hidden_states))
        outputs = (hidden_states,)
        if output_attentions:
            outputs += (attn_w,)
        if use_cache:
            outputs += (present,)
        return outputs

    @torch.no_grad()
    def to_int4(self, device="cuda"):
        """Real-INT4 serving layer from this simulated one (no reference equivalent: e2e/ runs random weights).

        Every QLinearLayer must still hold (or have saved, via quant()) its reordered FP weight.  Mapping:
          input_layernorm.reorder_index            -> LlamaRMSNormInt4.reorder_index (q/k/v input order)
          self_attn.reorder_index                  -> the reorder_fp16_i4 before o_proj
          mlp: the reference folds down_proj's input order into gate/up's *output* order, so nothing is carried.
        """
        from .export import int4_decoder_layer
        return int4_decoder_layer(self, device)


# ------------------------------------------------------------------------------------------------ test stand-ins
class ToyRMSNorm(nn.Module):
    def __init__(self, hidden, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(1.0 + 0.1 * torch.randn(hidden))
        self.variance_epsilon = eps

    def forward(self, x):
        v = x.float().pow(2).mean(-1, keepdim=True)
        return (self.weight * (x.float() * torch.rsqrt(v + self.variance_epsilon))).to(x.dtype)


class _ToyAttention(nn.Module):
    def __init__(self, hidden, heads, kv_heads=None, rope_theta=10000.0):
        super().__init__()
        kv_heads = kv_heads or heads
        self.hidden_size, self.num_heads, self.num_key_value_heads = hidden, heads, kv_heads
        self.head_dim = hidden // heads
        self.num_key_value_groups = heads // kv_heads
        self.max_position_embeddings, self.rope_theta = 4096, rope_theta
        self.attention_dropout, self.layer_idx = 0.0, 0
        self.q_proj = nn.Linear(hidden, hidden, bias=False)
        self.k_proj = nn.Linear(hidden, kv_heads * self.head_dim, bias=False)
        self.v_proj = nn.Linear(hidden, kv_heads * self.head_dim, bias=False)
        self.o_proj = nn.Linear(hidden, hidden, bias=False)
        self.rotary_emb = None
        self.q_kv_cache, self.reorder_index = False, None
        self.act_quant = self.k_quant = self.v_quant = lambda t: t


class _ToyMLP(nn.Module):
    def __init__(self, hidden, inter):
        super().__init__()
        self.gate_proj = nn.Linear(hidden, inter, bias=False)
        self.up_proj = nn.Linear(hidden, inter, bias=False)
        self.down_proj = nn.Linear(inter, hidden, bias=False)
        self.act_fn = nn.SiLU()

    def forward(self, x):
        return self.down_proj(self.act_fn(self.gate_proj(x)) * self.up_proj(x))


class ToyLlamaDecoderLayer(nn.Module):
    """Random-weight FP Llama decoder layer with HF attribute names (head_dim = hidden/heads, 128 for the KV quantiser)."""

    def __init__(self, hidden=256, inter=512, heads=2, kv_heads=None):
        super().__init__()
        self.hidden_size = hidden
        self.self_attn = _ToyAttention(hidden, heads, kv_heads)
        self.mlp = _ToyMLP(hidden, inter)
        self.input_layernorm = ToyRMSNorm(hidden)
        self.post_attention_layernorm = ToyRMSNorm(hidden)

    @torch.no_grad()
    def forward(self, x, attention_mask=None, position_ids=None):
        a, _, _ = quantised_attention(self.self_attn, self.input_layernorm(x), attention_mask, position_ids, None, False, False)
        x = x + a
        return (x + self.mlp(self.post_attention_layernorm(x)),)
