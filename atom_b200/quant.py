"""Quantisation math of the accuracy simulator -- the function surface of /root/reference/model/quant.py
(quantize_tensor :119-183, quantize_tensor_channel_group :69-107, quantize_activation_wrapper :188-231,
quantize_attn_{k,v}_wrapper :234-257, Quantizer :259-304), integer uniform-affine path only (FP4 / FP8 / exponential
formats are out of scope, DESIGN.md section 7).

In addition to the fake-quant ("quantise then dequantise") functions the reference has, `quantize_weight_int` returns the
INTEGER codes and scales themselves: that is what `QLinearLayer.pack()` turns into the real-INT4 operands of the
GEMM -- the bridge between model/ and e2e/ that the reference lacks.
"""
from functools import partial

import torch
from torch import nn


def _affine_params(w2d, n_bits, sym, clip_ratio):
    """Per-row (scale, zero, qmin, qmax) of a 2-D tensor [rows, group] (quant.py:141-178)."""
    if sym:
        qmax, qmin = 2 ** (n_bits - 1) - 1, -(2 ** (n_bits - 1))
        amax = w2d.abs().amax(dim=-1, keepdim=True).clamp(min=1e-5)
        if clip_ratio < 1.0:
            amax = amax * clip_ratio
        scale = amax / qmax
        zero = torch.zeros_like(scale)
    else:
        qmax, qmin = 2 ** n_bits - 1, 0
        hi, lo = w2d.amax(dim=-1, keepdim=True), w2d.amin(dim=-1, keepdim=True)
        if clip_ratio < 1.0:
            hi, lo = hi * clip_ratio, lo * clip_ratio
        scale = (hi - lo).clamp(min=1e-5) / qmax
        zero = torch.round(-lo / scale).clamp_(min=qmin, max=qmax)
    return scale, zero, qmin, qmax


@torch.no_grad()
def quantize_tensor(w, n_bits, group_size, tiling, sym, clip_ratio=1.0, exponential=False, quant_type="int"):
    """Fake-quantise `w` in groups of `group_size` along the last dim (0 = whole rows).  torch.round = half-to-even."""
    assert tiling == 0 and not exponential and quant_type == "int", "only the uniform INT path is supported"
    assert n_bits < 16
    shape = w.shape
    w2 = w.squeeze()
    w2 = w2.reshape(-1, group_size) if group_size > 0 else w2.reshape(-1, w2.shape[-1])
    scale, zero, qmin, qmax = _affine_params(w2, n_bits, sym, clip_ratio)
    return ((torch.clamp(torch.round(w2 / scale) + zero, qmin, qmax) - zero) * scale).reshape(shape)


@torch.no_grad()
def quantize_weight_int(W, n_bits, group_size, sym, channel_group=1, clip_ratio=1.0):
    """Integer codes and scales of a weight [out, in]: groups of `group_size` input channels, `channel_group` adjacent
    output rows sharing one scale (quant.py:80-105).  Returns (q int8 [out, in], scale fp32 [in/group, out])."""
    assert sym, "weights are symmetric in the W4A4 recipe"
    out_f, in_f = W.shape
    g = in_f // group_size
    blocks = W.reshape(out_f // channel_group, channel_group, g, group_size).permute(2, 0, 1, 3)   # [g, out/cg, cg, gs]
    flat = blocks.reshape(g, out_f // channel_group, channel_group * group_size)
    scale, _, qmin, qmax = _affine_params(flat.reshape(-1, channel_group * group_size), n_bits, True, clip_ratio)
    scale = scale.reshape(g, out_f // channel_group, 1)
    q = torch.clamp(torch.round(flat / scale), qmin, qmax)
    q = q.reshape(g, out_f // channel_group, channel_group, group_size).permute(1, 2, 0, 3).reshape(out_f, in_f)
    return q.to(torch.int8), scale.reshape(g, out_f // channel_group).repeat_interleave(channel_group, dim=1)


@torch.no_grad()
def quantize_tensor_channel_group(W, n_bits, group_size, tiling, sym, channel_group=1, clip_ratio=1.0, exponential=False, quant_type="int"):
    assert W.is_contiguous() and n_bits < 16
    if group_size == 0:
        return quantize_tensor(W, n_bits=n_bits, group_size=0, tiling=tiling, sym=sym, exponential=exponential)
    assert W.shape[-1] % group_size == 0
    if sym:
        q, scale = quantize_weight_int(W, n_bits, group_size, True, channel_group, clip_ratio)
        g = W.shape[1] // group_size
        return (q.reshape(W.shape[0], g, group_size).to(W.dtype) * scale.t().reshape(W.shape[0], g, 1).to(W.dtype)).reshape(W.shape).contiguous()
    out = W.clone()
    for c0 in range(0, W.shape[1], group_size):
        blk = W[:, c0:c0 + group_size]
        if channel_group > 1:
            blk = blk.reshape(W.shape[0] // channel_group, -1)
        out[:, c0:c0 + group_size] = quantize_tensor(blk.contiguous(), n_bits, 0, tiling, sym, clip_ratio).reshape(-1, group_size)
    return out.contiguous()


@torch.no_grad()
def quantize_activation_wrapper(x, args):
    """quant.py:188-231: last `keeper` channels INT8 per row, everything else INT-abits per group."""
    if args.abits >= 16:
        return x
    shape = x.shape
    x = x.view(-1, shape[-1])
    assert args.act_group_size == 0 or shape[-1] % args.act_group_size == 0
    if args.keeper > 0:
        saved = x[:, -args.keeper:].clone().contiguous()
        if args.keeper_precision == 3:
            saved = quantize_tensor(saved, n_bits=8, group_size=0, tiling=0, sym=True)
        elif args.keeper_precision != 0:
            raise NotImplementedError("FP8 keepers (keeper_precision 1/2) are outside the W4A4 INT path")
        x[:, -args.keeper:] = 0
    x = quantize_tensor(x, n_bits=args.abits, group_size=args.act_group_size, tiling=args.tiling, sym=args.a_sym, clip_ratio=args.a_clip_ratio)
    if args.keeper > 0:
        x[:, -args.keeper:] = saved
    return x.view(shape)


@torch.no_grad()
def _quantize_attn_wrapper(w, args):
    assert w.shape[-1] == 128, "KV Cache Quantization is per head granularity."
    shape = w.shape
    w = quantize_tensor(w.reshape(-1, 128), n_bits=args.abits, group_size=0, tiling=0, sym=False, clip_ratio=args.kv_clip_ratio)
    return w.view(shape)


quantize_attn_v_wrapper = _quantize_attn_wrapper
quantize_attn_k_wrapper = _quantize_attn_wrapper


class Quantizer(nn.Module):
    """quant.py:259-304 (dynamic path; static scales keep the reference's asserts)."""

    def __init__(self, args) -> None:
        super().__init__()
        self.register_buffer("scales", None)
        self.args = args
        self.act_quant = lambda x: x

    @torch.no_grad()
    def forward(self, hidden_states):
        if self.args.static is False or self.scales is None:
            return self.act_quant(hidden_states)
        shape = hidden_states.shape
        assert self.args.a_sym is True, "Only support statically symmetric quantization"
        hs = hidden_states.view(-1, shape[-1])
        sel = hs[:, self.args.keeper:].clone()
        if self.args.act_group_size > 0:
            sel = sel.reshape(-1, self.args.act_group_size)
        assert self.scales.numel() == sel.shape[-2], "Scales and selected states must have the same dimension"
        sel = torch.clamp(torch.round(sel / self.scales), self.q_min, self.q_max) * self.scales
        hs[:, self.args.keeper:] = sel.reshape(-1, shape[-1] - self.args.keeper)
        return hs.view(shape)

    def configure(self, func, scales):
        if self.args.static is False:
            self.act_quant = func
            return
        assert scales is not None, "Scales is None"
        self.register_buffer("scales", scales)
        self.q_min, self.q_max = -(2 ** (self.args.abits - 1)), 2 ** (self.args.abits - 1) - 1
        self.act_quant = func


def make_act_quant(args):
    return partial(quantize_activation_wrapper, args=args)
