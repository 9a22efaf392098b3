"""Real-INT4 Llama layers on the CUDA kernels -- the operator surface of
/root/reference/e2e/punica-atom/punica/models/llama.py:35-364 (LinearInt4, LlamaMLP, LlamaAttention, LlamaRMSNormInt4,
LlamaDecoderLayer, LlamaModel, LlamaForCausalLM): same constructor arguments, parameter names / shapes and
forward(hidden_states, blen, prefill_kv, decode_kv) contract, so the reference's bench_textgen harness can drive it.

Differences (documented in DESIGN.md):
  * hidden / intermediate sizes are free multiples of 128 (reference kernels: 4096 / 11008 only);
  * prefill attention uses the K/V that were just quantised into the cache (dequantised, causal SDPA with RoPE); the
    reference feeds torch.randn K/V there ("HACK", llama.py:171-174);
  * no HuggingFace dependency: any object with hidden_size / intermediate_size / num_attention_heads /
    num_hidden_layers / rms_norm_eps / vocab_size works as `config` (LlamaConfig does).
"""
import math
from dataclasses import dataclass
from typing import Optional

import torch
from torch import nn

from . import ops
from .cat_tensor import BatchLenInfo
from .kvcache import BatchedKvCacheInt4


@dataclass
class LlamaConfig:
    hidden_size: int = 4096
    intermediate_size: int = 11008
    num_attention_heads: int = 32
    num_hidden_layers: int = 32
    rms_norm_eps: float = 1e-6
    vocab_size: int = 32000
    pad_token_id: int = 0
    num_key_value_heads: Optional[int] = None      # None = multi-head attention (one KV head per query head)
    rope_theta: float = 10000.0


def rotate_half(x):
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2:]
    return torch.cat((-x2, x1), dim=-1)


def rotary_pos_emb(q, k, beg, theta=10000):
    """llama.py:18-32 (`theta`: the RoPE base, 1e4 there)"""
    bsz, nhead, seqlen, dim = q.shape
    inv_freq = 1.0 / (theta ** (torch.arange(0, dim, 2, device=q.device).float() / dim))
    t = torch.arange(beg, beg + seqlen, device=q.device, dtype=torch.float32)
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)[None, None]
    cos, sin = emb.cos(), emb.sin()
    return ((q.float() * cos) + (rotate_half(q.float()) * sin)).to(q.dtype), ((k.float() * cos) + (rotate_half(k.float()) * sin)).to(k.dtype)


class LinearInt4(nn.Module):
    """llama.py:35-68.  weight_int4 u8 [out, (in-128)/2], weight_int8 i8 [out, 128], scale_int4 f16 [in/128-1, S(out)],
    scale_int8 f16 [S(out)] -- allocated like the reference; the kernels read scale_int4 as a flat [group][out] array
    (pitch `out`, so only the first (in/128-1)*out halves are live) and the first `out` halves of scale_int8."""

    def __init__(self, in_features, out_features, out_dtype, bias=False):
        super().__init__()
        assert bias is False
        self.in_features, self.out_features, self.out_dtype = in_features, out_features, out_dtype
        gs = 128
        self.weight_int4 = nn.Parameter(torch.empty(out_features, (in_features - gs) // 2, dtype=torch.uint8), requires_grad=False)
        self.weight_int8 = nn.Parameter(torch.empty(out_features, gs, dtype=torch.int8), requires_grad=False)
        self.scale_int4 = nn.Parameter(torch.empty((in_features // gs - 1, ops.scale_size(out_features)), dtype=torch.float16), requires_grad=False)
        self.scale_int8 = nn.Parameter(torch.empty(ops.scale_size(out_features), dtype=torch.float16), requires_grad=False)
        self.register_parameter("bias", None)

    @torch.no_grad()
    def init_random(self, seed=0):
        """Random-quantised weights of this shape (the e2e harness runs on random INT4 weights, e2e/README.md:9)."""
        g = torch.Generator(device=self.weight_int4.device).manual_seed(seed)
        dev = self.weight_int4.device
        self.weight_int4.copy_(torch.randint(0, 256, self.weight_int4.shape, dtype=torch.uint8, device=dev, generator=g))
        self.weight_int8.copy_(torch.randint(-128, 128, self.weight_int8.shape, dtype=torch.int8, device=dev, generator=g))
        k = self.in_features
        self.scale_int4.copy_((0.02 / 7 / math.sqrt(k) * 8) * (1 + torch.rand(self.scale_int4.shape, device=dev, generator=g)))
        self.scale_int8.copy_((0.02 / 127 / math.sqrt(k) * 8) * (1 + torch.rand(self.scale_int8.shape, device=dev, generator=g)))
        return self

    def forward(self, input, flags=ops.GEMM_AUTO):
        outlier, norms, outlier_scales, norm_scales = input
        f = {"int4": ops.dense_layer_gemm_i4_o4, "fp16": ops.dense_layer_gemm_i4_fp16}[self.out_dtype]
        return f(norms, self.weight_int4, norm_scales, self.scale_int4, outlier, self.weight_int8, outlier_scales, self.scale_int8,
                 flags=flags)


@torch.no_grad()
def fuse_linear_rows(layers):
    """Row-concatenate LinearInt4 layers that share their input (q/k/v or gate/up) for the fused decode launches
    (ops.dense_layer_gemm_i4_qkv / _gateup_act).  The big tensors are shared, not duplicated: every layer's weight_int4 /
    weight_int8 becomes a row-slice VIEW of the fused tensor; only the (small) scales exist twice, because a slice of the
    fused [G, sum N] scale matrix has the wrong pitch for the single-projection kernels."""
    k = layers[0].in_features
    g = k // 128 - 1
    assert all(l.in_features == k for l in layers)
    w4 = torch.cat([l.weight_int4.data for l in layers], 0).contiguous()
    w8 = torch.cat([l.weight_int8.data for l in layers], 0).contiguous()
    s4 = torch.cat([l.scale_int4.data.reshape(-1)[: g * l.out_features].view(g, l.out_features) for l in layers], 1).contiguous()
    s8 = torch.cat([l.scale_int8.data[: l.out_features] for l in layers], 0).contiguous()
    r = 0
    for l in layers:
        l.weight_int4 = nn.Parameter(w4[r:r + l.out_features], requires_grad=False)
        l.weight_int8 = nn.Parameter(w8[r:r + l.out_features], requires_grad=False)
        r += l.out_features
    return w4, s4, w8, s8


def _capturing():
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


def run_concurrently(layers, x):
    """Decode-sized batches: the GEMMs that share one input (q/k/v, gate/up) are independent and each too small to fill
    the GPU, so they run side by side on forked streams, un-split along K (a 4096-channel projection is then 32 CTAs);
    the fork/join is captured into CUDA graphs like any other dependency.  Larger batches run one after the other."""
    if x[0].shape[0] > 64 or len(layers) == 1:
        return [l(x) for l in layers]
    cur = torch.cuda.current_stream()
    ev = torch.cuda.Event()
    ev.record(cur)
    outs = [None] * len(layers)
    side = [torch.cuda.Stream(device=x[0].device) for _ in layers[1:]]
    for st in side:
        st.wait_event(ev)
    outs[0] = layers[0](x, flags=ops.GEMM_NO_SPLITK)
    for i, st in enumerate(side):
        with torch.cuda.stream(st):
            outs[i + 1] = layers[i + 1](x, flags=ops.GEMM_NO_SPLITK)
    for i, st in enumerate(side):
        cur.wait_stream(st)
        for t in (outs[i + 1] if isinstance(outs[i + 1], tuple) else (outs[i + 1],)):
            t.record_stream(cur)
    return outs


class LlamaMLP(nn.Module):
    """llama.py:71-87"""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.hidden_size, self.intermediate_size = config.hidden_size, config.intermediate_size
        self.gate_proj = LinearInt4(self.hidden_size, self.intermediate_size, out_dtype="fp16")
        self.up_proj = LinearInt4(self.hidden_size, self.intermediate_size, out_dtype="fp16")
        self.down_proj = LinearInt4(self.intermediate_size, self.hidden_size, out_dtype="fp16")
        self._gu = None        # fused [gate; up] operands, built by fuse()

    def fuse(self):
        """One launch for gate_proj + up_proj + SiLU*mul + quantise on decode batches (call after the weights are loaded)."""
        self._gu = fuse_linear_rows([self.gate_proj, self.up_proj])
        return self

    def forward(self, x):
        if x[1].shape[0] <= 64 and self._gu is None and not _capturing():
            self.fuse()
        if x[1].shape[0] <= 64 and self._gu is not None:
            outlier, norms, outlier_scales, norm_scales = x
            w4, s4, w8, s8 = self._gu
            return self.down_proj(ops.dense_layer_gemm_i4_gateup_act(norms, w4, norm_scales, s4, outlier, w8, outlier_scales, s8))
        gate, up = run_concurrently([self.gate_proj, self.up_proj], x)
        return self.down_proj(ops.activate_fp16_i4(gate, up))


def _dequant_o4(d, d_scale, num_heads):
    """(u8 [T, H*64], f16 [T, H*2]) -> f16 [T, H, 128]: x = nibble * scale - zero (quantization.cuh:76)."""
    t = d.shape[0]
    d = d.view(t, num_heads, 64)
    lo, hi = (d & 0xF).float(), (d >> 4).float()
    x = torch.stack((lo, hi), dim=-1).view(t, num_heads, 128)
    p = d_scale.view(t, num_heads, 2).float()
    return (x * p[..., :1] - p[..., 1:]).half()


class LlamaAttention(nn.Module):
    """llama.py:90-232"""

    def __init__(self, config, layer_idx: int):
        super().__init__()
        self.config = config
        self.hidden_size, self.num_heads = config.hidden_size, config.num_attention_heads
        self.head_dim = self.hidden_size // self.num_heads
        self._scale = 1 / math.sqrt(self.head_dim)
        self.layer_idx = layer_idx
        if self.head_dim * self.num_heads != self.hidden_size:
            raise ValueError(f"hidden_size must be divisible by num_heads (got `hidden_size`: {self.hidden_size}"
                             f" and `num_heads`: {self.num_heads}).")
        # grouped-query attention: fewer KV heads than query heads (Llama-2-70B, Llama-3, Mixtral); None = multi-head
        self.num_kv_heads = getattr(config, "num_key_value_heads", None) or self.num_heads
        self.rope_theta = float(getattr(config, "rope_theta", 10000.0))
        if self.num_heads % self.num_kv_heads:
            raise ValueError(f"num_attention_heads ({self.num_heads}) must be a multiple of num_key_value_heads ({self.num_kv_heads})")
        h = self.num_heads * self.head_dim
        hkv = self.num_kv_heads * self.head_dim
        self.q_proj = LinearInt4(self.hidden_size, h, out_dtype="fp16")
        self.k_proj = LinearInt4(self.hidden_size, hkv, out_dtype="int4")
        self.v_proj = LinearInt4(self.hidden_size, hkv, out_dtype="int4")
        self.o_proj = LinearInt4(h, self.hidden_size, out_dtype="fp16")
        self.reorder_index = nn.Parameter(torch.randperm(self.hidden_size, dtype=torch.int16), requires_grad=False)
        self._qkv = None       # fused [q; k; v] operands, built by fuse()

    def fuse(self):
        """One launch for the q, k and v projections (call after the weights are loaded)."""
        self._qkv = fuse_linear_rows([self.q_proj, self.k_proj, self.v_proj])
        return self

    def forward(self, hidden_states, blen: BatchLenInfo, prefill_kv, decode_kv) -> torch.Tensor:
        nvtx = torch.cuda.nvtx
        nvtx.range_push("qkv_proj")
        if self._qkv is None and not _capturing():
            self.fuse()
        if self._qkv is not None:
            outlier, norms, outlier_scales, norm_scales = hidden_states
            w4, s4, w8, s8 = self._qkv
            kv_rows = None if self.num_kv_heads == self.num_heads else self.num_kv_heads * self.head_dim
            q_proj, k_proj, v_proj = ops.dense_layer_gemm_i4_qkv(norms, w4, norm_scales, s4, outlier, w8, outlier_scales, s8,
                                                                 kv_rows=kv_rows)
        else:
            q_proj, k_proj, v_proj = run_concurrently([self.q_proj, self.k_proj, self.v_proj], hidden_states)
        nvtx.range_pop()
        stack = []
        nq, nh, hd = self.num_heads, self.num_kv_heads, self.head_dim      # nh: heads of k / v and of the cache
        if len(blen.prefills) > 0:
            nvtx.range_push("init_kv")
            assert prefill_kv is not None
            ops.init_kv_i4(prefill_kv, k_proj[0][:blen.doff].view(-1, nh, hd // 2), v_proj[0][:blen.doff].view(-1, nh, hd // 2),
                           k_proj[1][:blen.doff].view(-1, nh, hd // 128 * 2), v_proj[1][:blen.doff].view(-1, nh, hd // 128 * 2),
                           blen.indptr, self.layer_idx)
            nvtx.range_pop()
            nvtx.range_push("prefill_attention")
            stack.append(ops.prefill_attention_i4(q_proj[:blen.doff], k_proj[0][:blen.doff], k_proj[1][:blen.doff],
                                                  v_proj[0][:blen.doff], v_proj[1][:blen.doff], blen.indptr, seqlens=list(blen.prefills),
                                                  rope_theta=self.rope_theta))
            nvtx.range_pop()
        if blen.decode > 0:
            q = q_proj[blen.doff:].view(blen.decode, nq, hd)
            k = k_proj[0][blen.doff:].view(blen.decode, nh, hd // 2)
            v = v_proj[0][blen.doff:].view(blen.decode, nh, hd // 2)
            ks = k_proj[1][blen.doff:].view(blen.decode, nh, hd // 128 * 2)
            vs = v_proj[1][blen.doff:].view(blen.decode, nh, hd // 128 * 2)
            nvtx.range_push("append_kv")
            assert decode_kv is not None
            ops.append_kv_i4(decode_kv, k.contiguous(), v.contiguous(), ks.contiguous(), vs.contiguous(), self.layer_idx)
            nvtx.range_pop()
            nvtx.range_push("batch_decode")
            stack.append(ops.batch_decode_i4(q.contiguous(), decode_kv, self.layer_idx, rope_theta=self.rope_theta)
                         .view(blen.decode, self.hidden_size))
            nvtx.range_pop()
        attn = stack[0] if len(stack) == 1 else torch.cat(stack, dim=0)
        nvtx.range_push("o_proj")
        out = self.o_proj(ops.reorder_fp16_i4(attn.contiguous(), self.reorder_index))
        nvtx.range_pop()
        return out


class LlamaRMSNormInt4(nn.Module):
    """llama.py:235-245"""

    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size, dtype=torch.float16))
        self.variance_epsilon = eps
        self.reorder_index = nn.Parameter(torch.randperm(hidden_size, dtype=torch.int16), requires_grad=False)

    def forward(self, hidden_states):
        return ops.rmsnorm_fp16_i4(hidden_states, self.weight, self.reorder_index, self.variance_epsilon)

    def forward_add(self, hidden_states, residual):
        """(residual + hidden_states, norm+quantise of that sum) in one launch.  hidden_states may be an ops.PendingAllReduce
        (tensor parallelism): the all-reduce is then formed inside the same launch."""
        if isinstance(hidden_states, ops.PendingAllReduce):
            return ops.reduce_add_rmsnorm_fp16_i4(hidden_states, residual, self.weight, self.reorder_index, self.variance_epsilon)
        return ops.add_rmsnorm_fp16_i4(hidden_states, residual, self.weight, self.reorder_index, self.variance_epsilon)


class LlamaDecoderLayer(nn.Module):
    """llama.py:248-292"""

    def __init__(self, config, layer_idx: int):
        super().__init__()
        self.hidden_size = config.hidden_size
        self.self_attn = LlamaAttention(config=config, layer_idx=layer_idx)
        self.mlp = LlamaMLP(config)
        self.input_layernorm = LlamaRMSNormInt4(config.hidden_size, eps=config.rms_norm_eps)
        self.post_attention_layernorm = LlamaRMSNormInt4(config.hidden_size, eps=config.rms_norm_eps)

    def init_random(self, seed=0):
        for i, m in enumerate(mod for mod in self.modules() if isinstance(mod, LinearInt4)):
            m.init_random(seed * 16 + i)
        if self.self_attn.q_proj.weight_int4.is_cuda:
            self.fuse()
        return self

    def fuse(self):
        """Build the fused q/k/v and gate/up operands (weights already on the GPU)."""
        self.self_attn.fuse()
        self.mlp.fuse()
        return self

    def forward(self, hidden_states, blen: BatchLenInfo, prefill_kv, decode_kv) -> torch.Tensor:
        hidden_states, delta = self.forward_residual(hidden_states, None, blen, prefill_kv, decode_kv)
        return hidden_states + delta

    def forward_residual(self, residual, delta, blen: BatchLenInfo, prefill_kv, decode_kv):
        """The layer on a (residual, delta) pair whose sum is the hidden state: every `residual + x` of the reference's layer
        (llama.py:266-292) is folded into the RMSNorm+quantise launch that follows it (ops.add_rmsnorm_fp16_i4), including
        the one that closes the PREVIOUS layer.  Returns the pair for the next layer; LlamaModel adds the last one."""
        if delta is None:
            x = self.input_layernorm(residual)
        else:
            residual, x = self.input_layernorm.forward_add(delta, residual)
        attn = self.self_attn(x, blen, prefill_kv, decode_kv)
        residual, x = self.post_attention_layernorm.forward_add(attn, residual)
        return residual, self.mlp(x)


class LlamaRMSNorm(nn.Module):
    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size, dtype=torch.float16))
        self.variance_epsilon = eps

    def forward(self, x):
        v = x.float().pow(2).mean(-1, keepdim=True)
        return (x.float() * torch.rsqrt(v + self.variance_epsilon)).to(x.dtype) * self.weight


class LlamaModel(nn.Module):
    """llama.py:311-343 (every layer gets its own layer_idx; the reference reuses index 0 "for memory")."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size, getattr(config, "pad_token_id", None))
        self.layers = nn.ModuleList([LlamaDecoderLayer(config, i) for i in range(config.num_hidden_layers)])
        self.norm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)

    def forward(self, input_ids, blen, prefill_kv, decode_kv):
        h, delta = self.embed_tokens(input_ids), None
        for layer in self.layers:
            h, delta = layer.forward_residual(h, delta, blen, prefill_kv, decode_kv)
        return self.norm(h + delta if delta is not None else h)


class LlamaForCausalLM(nn.Module):
    """llama.py:346-364"""

    def __init__(self, config):
        super().__init__()
        self.model = LlamaModel(config)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)

    def forward(self, input_ids, blen, prefill_kv, decode_kv):
        hidden_states = self.model(input_ids, blen, prefill_kv, decode_kv)
        return self.lm_head(hidden_states), hidden_states
