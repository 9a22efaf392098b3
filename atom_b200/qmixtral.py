"""QMixtralDecoderLayer and friends -- the operator surface of /root/reference/model/qMixtralLayer.py:58-446.

Same simulation as qllama.py with the Mixtral differences the reference has:
  * the norms do NOT quantise (QMixtralRMSNorm has no act_quant); the decoder layer's own `act_quant` runs after
    input_layernorm (qMixtralLayer.py:411-413) and the MoE block's `act_quant` runs *after* the router, so the
    router (`gate`, a QLinearLayer with enable_quant=False) always sees un-quantised activations (:289, :306-311);
  * each expert is w1/w3 (gate/up) -> act_quant -> w2 (down);
  * quantisers default to the identity lambda and are assigned by the driver (modelutils_mixtral.py), not configure()d.
Top-k routing is evaluated expert by expert with index_add_, like the HF block the reference wraps.
"""
import torch
import torch.nn.functional as F
from torch import nn

from .qlinear import QLinearLayer
from .qllama import ToyRMSNorm, _cfg, _ToyAttention, quantised_attention


def _identity(x):
    return x


class QMixtralRMSNorm(nn.Module):
    def __init__(self, originalRMSNorm, args):
        super().__init__()
        self.originalRMSNorm = originalRMSNorm
        self.register_buffer("reorder_index", None)
        self.args = args

    @torch.no_grad()
    def forward(self, hidden_states):
        result = self.originalRMSNorm(hidden_states)
        if self.reorder_index is not None:
            assert result.shape[-1] == self.reorder_index.shape[0]
            result = torch.index_select(result, result.dim() - 1, self.reorder_index)
        return result


class QMixtralAttention(nn.Module):
    def __init__(self, originalAttn, args):
        super().__init__()
        self.config = getattr(originalAttn, "config", None)
        self.layer_idx = getattr(originalAttn, "layer_idx", None)
        self.hidden_size = _cfg(originalAttn, "hidden_size")
        self.num_heads = _cfg(originalAttn, "num_heads")
        self.head_dim = getattr(originalAttn, "head_dim", self.hidden_size // self.num_heads)
        self.num_key_value_heads = _cfg(originalAttn, "num_key_value_heads", self.num_heads)
        self.num_key_value_groups = self.num_heads // self.num_key_value_heads
        self.max_position_embeddings = _cfg(originalAttn, "max_position_embeddings", 32768)
        self.rope_theta = _cfg(originalAttn, "rope_theta", 1e6)
        self.is_causal = True
        self.attention_dropout = _cfg(originalAttn, "attention_dropout", 0.0)
        self.register_buffer("reorder_index", None)
        if self.head_dim * self.num_heads != self.hidden_size:
            raise ValueError(f"hidden_size must be divisible by num_heads (got `hidden_size`: {self.hidden_size}"
                             f" and `num_heads`: {self.num_heads}).")
        self.q_proj = QLinearLayer(originalAttn.q_proj, args)
        self.k_proj = QLinearLayer(originalAttn.k_proj, args)
        self.v_proj = QLinearLayer(originalAttn.v_proj, args)
        self.o_proj = QLinearLayer(originalAttn.o_proj, args)
        self.rotary_emb = getattr(originalAttn, "rotary_emb", None)
        self.act_quant = _identity
        self.k_quant = _identity
        self.v_quant = _identity
        self.q_kv_cache = args.kv_cache

    @torch.no_grad()
    def forward(self, hidden_states, attention_mask=None, position_ids=None, past_key_value=None, output_attentions=False,
                use_cache=False, **_):
        return quantised_attention(self, hidden_states, attention_mask, position_ids, past_key_value, output_attentions, use_cache)


class QMixtralBlockSparseTop2MLP(nn.Module):
    def __init__(self, originalTop2MLP, args):
        super().__init__()
        self.ffn_dim = originalTop2MLP.ffn_dim
        self.ffm_dim = self.ffn_dim                       # the reference's spelling (qMixtralLayer.py:244)
        self.hidden_dim = originalTop2MLP.hidden_dim
        self.w1 = QLinearLayer(originalTop2MLP.w1, args)
        self.w2 = QLinearLayer(originalTop2MLP.w2, args)
        self.w3 = QLinearLayer(originalTop2MLP.w3, args)
        self.act_fn = originalTop2MLP.act_fn
        self.act_quant = _identity

    @torch.no_grad()
    def forward(self, hidden_states):
        return self.w2(self.act_quant(self.act_fn(self.w1(hidden_states)) * self.w3(hidden_states)))

    def quant(self):
        self.w1.quant()
        self.w2.quant()
        self.w3.quant()


class QMixtralSparseMoeBlock(nn.Module):
    def __init__(self, originalMoeBlock, args):
        super().__init__()
        self.hidden_dim = originalMoeBlock.hidden_dim
        self.ffn_dim = originalMoeBlock.ffn_dim
        self.num_experts = originalMoeBlock.num_experts
        self.top_k = originalMoeBlock.top_k
        self.args = args
        self.act_quant = _identity
        self.gate = QLinearLayer(originalMoeBlock.gate, args, enable_quant=False)
        self.experts = nn.ModuleList([QMixtralBlockSparseTop2MLP(originalMoeBlock.experts[i], args) for i in range(self.num_experts)])

    @torch.no_grad()
    def forward(self, hidden_states):
        bsz, seq, hidden = hidden_states.shape
        x = hidden_states.reshape(-1, hidden)
        router_logits = self.gate(x)                      # FP router on un-quantised activations
        if self.args.abits < 16:
            x = self.act_quant(x)
        p = F.softmax(router_logits, dim=1, dtype=torch.float)
        p, chosen = torch.topk(p, self.top_k, dim=-1)
        p = (p / p.sum(dim=-1, keepdim=True)).to(x.dtype)
        out = torch.zeros_like(x)
        for e in range(self.num_experts):
            tok, slot = torch.where(chosen == e)
            if tok.numel() == 0:
                continue
            out.index_add_(0, tok, (self.experts[e](x[tok]) * p[tok, slot, None]).to(x.dtype))
        return out.reshape(bsz, seq, hidden), router_logits


class QMixtralDecoderLayer(nn.Module):
    def __init__(self, originalLayer, args):
        super().__init__()
        self.args = args
        self.hidden_size = _cfg(originalLayer, "hidden_size", originalLayer.self_attn.q_proj.weight.shape[1])
        self.act_quant = _identity
        self.self_attn = QMixtralAttention(originalLayer.self_attn, args)
        self.block_sparse_moe = QMixtralSparseMoeBlock(originalLayer.block_sparse_moe, args)
        self.input_layernorm = QMixtralRMSNorm(originalLayer.input_layernorm, args)
        self.post_attention_layernorm = QMixtralRMSNorm(originalLayer.post_attention_layernorm, args)

    @torch.no_grad()
    def forward(self, hidden_states, attention_mask=None, position_ids=None, past_key_value=None, output_attentions=False,
                output_router_logits=False, use_cache=False, cache_position=None, **_):
        residual = hidden_states
        hidden_states = self.input_layernorm(hidden_states)
        if self.args.abits < 16:
            hidden_states = self.act_quant(hidden_states)
        hidden_states, attn_w, present = self.self_attn(hidden_states, attention_mask, position_ids, past_key_value,
                                                        output_attentions, use_cache)
        hidden_states = residual + hidden_states
        moe, router_logits = self.block_sparse_moe(self.post_attention_layernorm(hidden_states))
        hidden_states = hidden_states + moe
        outputs = (hidden_states,)
        if output_attentions:
            outputs += (attn_w,)
        if use_cache:
            outputs += (present,)
        if output_router_logits:
            outputs += (router_logits,)
        return outputs

    @torch.no_grad()
    def to_int4(self, device="cuda"):
        """Real-INT4 serving layer (atom_b200.mixtral.MixtralDecoderLayer) from this simulated one; every QLinearLayer must still
        hold (or have saved, via quant()) its reordered FP weight.  See export.int4_mixtral_decoder_layer."""
        from .export import int4_mixtral_decoder_layer
        return int4_mixtral_decoder_layer(self, device)


# ------------------------------------------------------------------------------------------------ test stand-ins
class _ToyExpert(nn.Module):
    def __init__(self, hidden, inter):
        super().__init__()
        self.ffn_dim, self.hidden_dim = inter, hidden
        self.w1 = nn.Linear(hidden, inter, bias=False)
        self.w2 = nn.Linear(inter, hidden, bias=False)
        self.w3 = nn.Linear(hidden, inter, bias=False)
        self.act_fn = nn.SiLU()

    def forward(self, x):
        return self.w2(self.act_fn(self.w1(x)) * self.w3(x))


class _ToyMoe(nn.Module):
    def __init__(self, hidden, inter, experts, top_k):
        super().__init__()
        self.hidden_dim, self.ffn_dim, self.num_experts, self.top_k = hidden, inter, experts, top_k
        self.gate = nn.Linear(hidden, experts, bias=False)
        self.experts = nn.ModuleList([_ToyExpert(hidden, inter) for _ in range(experts)])

    def forward(self, hs):
        """Dense float restatement: every expert on every token, weighted by the renormalised top-k softmax."""
        b, s, h = hs.shape
        x = hs.reshape(-1, h)
        p = F.softmax(self.gate(x), dim=1, dtype=torch.float)
        top, idx = torch.topk(p, self.top_k, dim=-1)
        wts = torch.zeros_like(p).scatter_(1, idx, top / top.sum(-1, keepdim=True))
        out = sum(self.experts[e](x) * wts[:, e:e + 1] for e in range(self.num_experts))
        return out.reshape(b, s, h)


class ToyMixtralDecoderLayer(nn.Module):
    def __init__(self, hidden=256, inter=256, heads=2, kv_heads=1, experts=4, top_k=2):
        super().__init__()
        self.hidden_size = hidden
        self.self_attn = _ToyAttention(hidden, heads, kv_heads, rope_theta=1e6)
        self.block_sparse_moe = _ToyMoe(hidden, inter, experts, top_k)
        self.input_layernorm = ToyRMSNorm(hidden)
        self.post_attention_layernorm = ToyRMSNorm(hidden)

    @torch.no_grad()
    def forward(self, x, attention_mask=None, position_ids=None):
        a, _, _ = quantised_attention(self.self_attn, self.input_layernorm(x), attention_mask, position_ids, None, False, False)
        x = x + a
        return (x + self.block_sparse_moe(self.post_attention_layernorm(x)),)
