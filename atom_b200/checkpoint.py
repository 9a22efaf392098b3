"""On-disk format for real-INT4 models (SURVEY.md section 8(f) row 2; no reference counterpart -- the reference's e2e path
only ever runs random weights and its simulator never leaves FP16).

One `.safetensors` file holding the module's state_dict verbatim -- for every LinearInt4 the four kernel operands
(`weight_int4` u8, `weight_int8` i8, `scale_int4` f16, `scale_int8` f16, shapes as punica/models/llama.py:44-58), the fp16
norm weights, the int16 reorder indices, and for a full model the embedding / lm_head -- plus a JSON header in the file
metadata: format tag, the LlamaConfig fields and which class was saved (files written before `num_key_value_heads` /
`rope_theta` joined the config lack them and load with the defaults: multi-head attention, base 1e4).  Loading rebuilds the module on the meta device
and assigns the tensors (no random init, no second copy), so a 65B shard loads at file-read speed.
"""
import dataclasses
import json

import torch

from .llama import LlamaConfig, LlamaDecoderLayer, LlamaForCausalLM

FORMAT = "atom_b200.int4.v1"
_KINDS = {"LlamaDecoderLayer": LlamaDecoderLayer, "LlamaForCausalLM": LlamaForCausalLM}


def _config_of(module) -> LlamaConfig:
    if isinstance(module, LlamaForCausalLM):
        c = module.model.config
    else:
        at = module.self_attn
        c = LlamaConfig(hidden_size=at.hidden_size, intermediate_size=module.mlp.intermediate_size,
                        num_attention_heads=at.num_heads, num_hidden_layers=1,
                        rms_norm_eps=module.input_layernorm.variance_epsilon,
                        num_key_value_heads=None if at.num_kv_heads == at.num_heads else at.num_kv_heads,
                        rope_theta=at.rope_theta)
    fields = {f.name for f in dataclasses.fields(LlamaConfig)}
    return LlamaConfig(**{k: getattr(c, k) for k in fields if hasattr(c, k)})


def save_int4(module, path: str, extra: dict = None) -> None:
    """Write a LlamaDecoderLayer or LlamaForCausalLM (real-INT4 operands) to `path`."""
    from safetensors.torch import save_file
    kind = type(module).__name__
    if kind not in _KINDS:
        raise TypeError(f"save_int4: unsupported module {kind}")
    meta = {"format": FORMAT, "kind": kind, "config": json.dumps(dataclasses.asdict(_config_of(module))),
            "layer_idx": str(getattr(getattr(module, "self_attn", None), "layer_idx", 0)),
            "extra": json.dumps(extra or {})}
    tensors = {k: v.detach().cpu().contiguous() for k, v in module.state_dict().items()}
    save_file(tensors, path, metadata=meta)


def load_int4(path: str, device="cuda"):
    """Rebuild the saved module on `device`.  Returns (module, extra)."""
    from safetensors import safe_open
    with safe_open(path, framework="pt", device="cpu") as f:
        meta = f.metadata() or {}
        if meta.get("format") != FORMAT:
            raise ValueError(f"{path}: not an {FORMAT} file (format tag {meta.get('format')!r})")
        tensors = {k: f.get_tensor(k) for k in f.keys()}
    cfg = LlamaConfig(**json.loads(meta["config"]))
    cls = _KINDS[meta["kind"]]
    with torch.device("meta"):
        module = cls(cfg, int(meta["layer_idx"])) if cls is LlamaDecoderLayer else cls(cfg)
    missing = set(module.state_dict().keys()) ^ set(tensors.keys())
    if missing:
        raise ValueError(f"{path}: tensor names do not match the {meta['kind']} layout: {sorted(missing)[:6]} ...")
    for k, ref in module.state_dict().items():
        if tuple(ref.shape) != tuple(tensors[k].shape) or ref.dtype != tensors[k].dtype:
            raise ValueError(f"{path}: {k} is {tuple(tensors[k].shape)} {tensors[k].dtype}, expected {tuple(ref.shape)} {ref.dtype}")
    module.load_state_dict({k: v.to(device) for k, v in tensors.items()}, assign=True)
    return module, json.loads(meta.get("extra", "{}"))
