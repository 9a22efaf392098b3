"""QLinearLayer -- the surface of /root/reference/model/qLinearLayer.py:16-86 (constructor, buffers `weight`/`bias`, `args`,
`.quant()`, `.reorder()`, `.to()`, `.forward()`), plus the step the reference lacks: `.pack()` converts the quantised
weight into the real-INT4 operands of the W4A4 GEMM, after which `forward()` runs
    reorder_fp16_i4 (dynamic per-group activation quantise)  ->  dense_layer_gemm_i4_fp16
on the GPU instead of F.linear on fake-quantised FP16 weights.

Layout after pack() (= LinearInt4's parameters, e2e/punica-atom/punica/models/llama.py:44-58):
    weight_int4 u8 [out, (in-128)/2]   two INT4 per byte, input channel 2j in the low nibble
    weight_int8 i8 [out, 128]          the keeper (last 128 reordered input channels)
    scale_int4 f16 [in/128-1, out]     per (group, output channel); adjacent channels share it (weight_channel_group=2)
    scale_int8 f16 [out]
"""
import torch
import torch.nn as nn

from . import ops
from .quant import quantize_tensor, quantize_tensor_channel_group, quantize_weight_int


def find_qlinear_layers(module, name=""):
    if type(module) == QLinearLayer:
        if module.enable_quant:
            return {name: module}
    res = {}
    for n1, child in module.named_children():
        res.update(find_qlinear_layers(child, name=name + "." + n1 if name != "" else n1))
    return res


class QLinearLayer(nn.Module):
    def __init__(self, originalLayer: nn.Linear, args, enable_quant: bool = True):
        super().__init__()
        self.args = args
        self.register_buffer("weight", originalLayer.weight)
        self.enable_quant = enable_quant
        if originalLayer.bias is not None:
            self.register_buffer("bias", originalLayer.bias)
        else:
            self.bias = None
        self.packed = False
        self._w_unquantized = None
        self._quantized = False

    @torch.no_grad()
    def forward(self, x):
        if not self.packed:
            return torch.functional.F.linear(x, self.weight, self.bias)
        shape = x.shape
        x2 = x.reshape(-1, shape[-1]).to(torch.float16).contiguous()
        outlier, norms, outlier_scales, norm_scales = ops.reorder_fp16_i4(x2, self.identity_index)
        y = ops.dense_layer_gemm_i4_fp16(norms.view(torch.uint8), self.weight_int4, norm_scales, self.scale_int4, outlier,
                                         self.weight_int8, outlier_scales, self.scale_int8)
        if self.bias is not None:
            y = y + self.bias.to(y.dtype)
        return y.reshape(*shape[:-1], y.shape[-1])

    def to(self, *args, **kwargs):
        super(QLinearLayer, self).to(*args, **kwargs)
        self.weight = self.weight.to(*args, **kwargs)
        return self

    @torch.no_grad()
    def quant(self):
        """qLinearLayer.py:42-77: INT8 per-row keeper on the last `keeper` input channels, grouped INT4 elsewhere."""
        a = self.args
        if a.wbits >= 16:
            return
        if getattr(a, "keeper_precision", 0) not in (0, 3):
            raise NotImplementedError("FP8 keepers are outside the W4A4 INT path")
        # The FP weight is only needed again by int4_operands() / pack() / to_int4(); keeping it doubles the simulator's
        # weight memory (+130 GB for Llama-65B), so it is opt-in: args.keep_fp_for_export, freed again by pack().
        self._w_unquantized = self.weight.clone() if getattr(a, "keep_fp_for_export", False) else None
        self._quantized = True
        if a.keeper > 0:
            saved = self.weight[:, -a.keeper:].clone().contiguous()
            if a.keeper_precision == 3:
                saved = quantize_tensor(saved, n_bits=8, group_size=0, tiling=0, sym=True, exponential=False)
            self.weight[:, -a.keeper:] = 0
        self.weight = quantize_tensor_channel_group(self.weight.clone(), n_bits=a.wbits, exponential=a.exponential, sym=a.w_sym,
                                                    group_size=a.weight_group_size, channel_group=a.weight_channel_group,
                                                    clip_ratio=a.w_clip_ratio, tiling=a.tiling, quant_type=a.quant_type)
        if a.keeper > 0:
            self.weight[:, -a.keeper:] = saved
        return

    def reorder(self, in_reorder_index, out_reorder_index=None):
        if self.args.reorder is True:
            in_reorder_index = in_reorder_index.to(self.weight.device)
            self.weight = torch.index_select(self.weight, 1, in_reorder_index)
            if out_reorder_index is not None:
                self.weight = torch.index_select(self.weight, 0, out_reorder_index.to(self.weight.device))
        return

    @torch.no_grad()
    def int4_operands(self):
        """Real-INT4 GEMM operands (CPU tensors) of the (reordered, un-fake-quantised if available) weight, without
        changing the layer.  Requires the W4A4 recipe: wbits=4, symmetric, weight_group_size=128, keeper=128 (INT8)."""
        a = self.args
        assert a.wbits == 4 and a.w_sym and a.weight_group_size == 128 and a.keeper == 128 and a.weight_channel_group == 2, "pack() implements the W4A4/g128/keeper128 recipe"
        if getattr(self, "_quantized", False) and self._w_unquantized is None:
            raise RuntimeError("QLinearLayer was fake-quantised without args.keep_fp_for_export=True: the FP weight needed to "
                               "derive real INT4 operands is gone (call pack()/to_int4() before quant(), or set the flag)")
        w = (self._w_unquantized if self._w_unquantized is not None else self.weight).float().cpu()
        out_f, in_f = w.shape
        assert in_f % 128 == 0 and in_f >= 256 and out_f % 8 == 0
        keep = w[:, -128:].contiguous()
        body = w[:, :-128].contiguous()
        # keeper: INT8 per output row; body: INT4 per (group, channel pair); same arithmetic as quant()
        # The GEMM (like the reference's, Dense_layer_gemm_i4_o16.cuh:404-434) reads EVERY weight scale -- the keeper's
        # too -- from column n&~1 for activation rows with m%16 < 8 and from n|1 otherwise, so scales must be shared by
        # adjacent output channels to be applied correctly: the INT4 body is (weight_channel_group = 2), and the
        # keeper is exported with one INT8 scale per channel pair for the same reason.
        ks = keep.abs().amax(dim=-1, keepdim=True).clamp(min=1e-5) / 127
        ks = ks.view(out_f // 2, 2).amax(dim=1, keepdim=True).repeat_interleave(2, dim=0)
        kq = torch.clamp(torch.round(keep / ks), -128, 127).to(torch.int8)
        # quant() quantises the body with the keeper columns zeroed: the last group is all zero there and lives in the
        # keeper instead, so only the first in/128-1 groups are packed
        q, scale = quantize_weight_int(body, 4, 128, True, a.weight_channel_group, a.w_clip_ratio)
        qi = q.to(torch.int16)
        packed = ((qi[:, 0::2] & 0xF) | ((qi[:, 1::2] & 0xF) << 4)).to(torch.uint8)
        return {"weight_int4": packed.contiguous(), "weight_int8": kq.contiguous(),
                "scale_int4": scale.to(torch.float16).contiguous(), "scale_int8": ks.reshape(-1).to(torch.float16).contiguous()}

    @torch.no_grad()
    def pack(self, device=None):
        """Switch this layer to the real-INT4 kernels: registers int4_operands() as buffers on `device`; forward() then
        runs reorder_fp16_i4 + dense_layer_gemm_i4_fp16 (CUDA only)."""
        dev = device if device is not None else self.weight.device
        for k, v in self.int4_operands().items():
            self.register_buffer(k, v.to(dev))
        self.register_buffer("identity_index", torch.arange(self.weight.shape[1], dtype=torch.int16, device=dev))
        self.packed = True
        self._w_unquantized = None          # the saved FP copy has served its purpose
        return self
