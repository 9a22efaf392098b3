"""CPU suite: the host side of grouped-query attention (fewer KV heads than query heads) on the INT4 paged-KV path -- the
oracle the GPU tests compare against, config defaults, KV pool shapes, checkpoint metadata, tensor-parallel head split.
No kernel is launched (there is no GPU here)."""
import dataclasses
import json

import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import gqa_oracle as GO


def _cache(rng, pages, L, hkv, P):
    data = rng.integers(0, 256, (pages, L, 2, hkv, P, 64), dtype=np.uint8)
    param = np.stack([rng.uniform(0.01, 0.05, (pages, L, 2, hkv, P)), rng.uniform(0, 0.4, (pages, L, 2, hkv, P))], -1).astype(np.float16)
    return data, param


@pytest.mark.parametrize("hq,hkv", [(4, 2), (8, 1), (4, 4)])
def test_gqa_oracle_equals_mha_oracle_on_head_repeated_cache(hq, hkv):
    rng = np.random.default_rng(hq * 16 + hkv)
    P, L, g = 16, 2, hq // hkv
    data, param = _cache(rng, 7, L, hkv, P)
    indptr, indices, last = np.array([0, 3, 4, 7], np.int32), np.array([5, 1, 3, 0, 2, 6, 4], np.int32), np.array([8, 1, 16], np.int32)
    q = rng.standard_normal((3, hq, 128)).astype(np.float16)
    got = GO.batch_decode_gqa_i4(q, data, param, indptr, indices, last, 1)
    rd, rp = GO.repeat_heads(data, param, g)
    ref = O.batch_decode_i4(q, rd, rp, indptr, indices, last, 1)
    assert np.array_equal(got.view(np.uint16), ref.view(np.uint16))
    # the base matters: another theta moves the result (guards against the argument being dropped on the way down)
    other = GO.batch_decode_gqa_i4(q, data, param, indptr, indices, last, 1, theta=5e5)
    assert np.abs(other.astype(np.float32) - got.astype(np.float32)).max() > 1e-3


def test_config_defaults_are_multi_head_and_base_1e4():
    from atom_b200 import textgen as tg
    from atom_b200.llama import LlamaAttention, LlamaConfig
    c = LlamaConfig()
    assert c.num_key_value_heads is None and c.rope_theta == 10000.0
    with torch.device("meta"):
        at = LlamaAttention(LlamaConfig(hidden_size=512, num_attention_heads=4), 0)
        assert at.num_kv_heads == 4 and at.rope_theta == 10000.0 and at.k_proj.out_features == 512

        class Duck:                                         # a config object that predates the two fields
            hidden_size, num_attention_heads = 512, 4
        assert LlamaAttention(Duck(), 0).num_kv_heads == 4
        gq = LlamaAttention(LlamaConfig(hidden_size=1024, num_attention_heads=8, num_key_value_heads=2, rope_theta=5e5), 0)
    assert (gq.q_proj.out_features, gq.k_proj.out_features, gq.v_proj.out_features, gq.o_proj.in_features) == (1024, 256, 256, 1024)
    assert gq.rope_theta == 5e5
    with pytest.raises(ValueError):
        LlamaAttention(LlamaConfig(hidden_size=1024, num_attention_heads=8, num_key_value_heads=3), 0)
    m7 = tg.MODEL_CFGS["7b"]
    assert m7.num_kv_heads is None and m7.kv_heads == 32 and m7.rope_theta == 10000.0
    m70, l3 = tg.MODEL_CFGS["70b"], tg.MODEL_CFGS["llama3-8b"]
    assert (m70.num_layers, m70.num_heads, m70.kv_heads, m70.hidden_size, m70.intermediate_size) == (80, 64, 8, 8192, 28672)
    assert (l3.num_layers, l3.num_heads, l3.kv_heads, l3.hidden_size, l3.intermediate_size, l3.rope_theta) == (32, 32, 8, 4096, 14336, 5e5)


def test_kv_pool_of_a_gqa_config_holds_kv_heads():
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvPoolInt4
    mc = tg.MODEL_CFGS["llama3-8b"]
    pool = KvPoolInt4(2, mc.kv_heads, mc.hidden_size // mc.num_heads, capacity=5, block_len=32, device=torch.device("cpu"))
    assert pool.buf.shape == (5, 2, 2, 8, 32, 64) and pool.param.shape == (5, 2, 2, 8, 32, 2)


def test_rope_table_is_keyed_by_base():
    from atom_b200 import ops
    from atom_b200.llama import rotary_pos_emb
    dev = torch.device("cpu")
    t4, t5 = ops.rope_table(10, dev), ops.rope_table(10, dev, theta=5e5)
    assert t4 is ops.rope_table(10, dev, theta=10000.0) and t5 is ops.rope_table(10, dev, theta=5e5) and t4 is not t5
    assert torch.equal(t4[:, 0], t5[:, 0]) and not torch.allclose(t4[:, 1:], t5[:, 1:])
    x = torch.randn(1, 2, 10, 128)
    a, _ = rotary_pos_emb(x, x, 0, theta=5e5)
    ref = torch.cat((x[..., :64] * t5[:10, :, 0] - x[..., 64:] * t5[:10, :, 1], x[..., 64:] * t5[:10, :, 0] + x[..., :64] * t5[:10, :, 1]), -1)
    assert torch.allclose(a, ref, atol=1e-6)
    assert torch.equal(rotary_pos_emb(x, x, 3)[0], rotary_pos_emb(x, x, 3, theta=10000)[0])


def test_checkpoint_carries_kv_heads_and_base_and_old_files_default(tmp_path):
    from safetensors import safe_open
    from safetensors.torch import save_file
    from atom_b200.checkpoint import FORMAT, load_int4, save_int4
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaDecoderLayer
    cfg = LlamaConfig(hidden_size=512, intermediate_size=512, num_attention_heads=4, num_hidden_layers=1, num_key_value_heads=2, rope_theta=1e6)
    layer = LlamaDecoderLayer(cfg, 0)
    for i, lin in enumerate(x for x in layer.modules() if isinstance(x, LinearInt4)):
        lin.init_random(i)
    path = str(tmp_path / "gqa.safetensors")
    save_int4(layer, path)
    back, _ = load_int4(path, device="cpu")
    assert back.self_attn.num_kv_heads == 2 and back.self_attn.rope_theta == 1e6 and back.self_attn.k_proj.out_features == 256
    assert all(torch.equal(a, b) for a, b in zip(layer.state_dict().values(), back.state_dict().values()))
    # a file written before the two fields existed: same format tag, header without them -> multi-head, base 1e4
    mha = LlamaDecoderLayer(LlamaConfig(hidden_size=512, intermediate_size=512, num_attention_heads=4, num_hidden_layers=1), 0)
    for i, lin in enumerate(x for x in mha.modules() if isinstance(x, LinearInt4)):
        lin.init_random(i)
    new = str(tmp_path / "mha.safetensors")
    save_int4(mha, new)
    with safe_open(new, framework="pt", device="cpu") as f:
        meta = dict(f.metadata())
        tensors = {k: f.get_tensor(k) for k in f.keys()}
    header = json.loads(meta["config"])
    assert header["num_key_value_heads"] is None and header["rope_theta"] == 10000.0 and meta["format"] == FORMAT
    del header["num_key_value_heads"], header["rope_theta"]
    meta["config"] = json.dumps(header)
    old = str(tmp_path / "old.safetensors")
    save_file(tensors, old, metadata=meta)
    back, _ = load_int4(old, device="cpu")
    assert back.self_attn.num_kv_heads == 4 and back.self_attn.rope_theta == 10000.0


def test_export_accepts_gqa_layer_and_carries_base():
    from atom_b200 import modelutils
    from atom_b200.export import int4_decoder_layer
    from atom_b200.qllama import ToyLlamaDecoderLayer
    from tests.test_export_cpu import _args
    torch.manual_seed(0)
    layers = [ToyLlamaDecoderLayer(512, 512, 4, kv_heads=1)]
    layers[0].self_attn.rope_theta = 5e5
    a = _args()
    a.reorder = False
    modelutils.quantize_model_llama(layers, a)
    modelutils.add_act_quant_wrapper_llama(layers, a)
    real = int4_decoder_layer(layers[0], device=None)
    at = real.self_attn
    assert (at.num_heads, at.num_kv_heads, at.rope_theta) == (4, 1, 5e5)
    assert at.k_proj.weight_int4.shape == (128, (512 - 128) // 2) and at.q_proj.weight_int4.shape == (512, (512 - 128) // 2)
    assert dataclasses.asdict(at.config)["num_key_value_heads"] == 1


def test_tp_layer_shards_kv_heads_and_refuses_a_bad_split():
    from atom_b200.llama import LlamaConfig
    from atom_b200.tp import TPLlamaDecoderLayer
    cfg = LlamaConfig(hidden_size=2048, intermediate_size=2048, num_attention_heads=16, num_hidden_layers=1, num_key_value_heads=2)
    with torch.device("meta"):
        l = TPLlamaDecoderLayer(cfg, 0, rank=1, world=2)
        assert (l.local_heads, l.local_kv_heads) == (8, 1)
        assert (l.q_proj.out_features, l.k_proj.out_features, l.v_proj.out_features) == (1024, 128, 128)
        with pytest.raises(ValueError, match="num_key_value_heads"):
            TPLlamaDecoderLayer(cfg, 0, rank=0, world=4)
        mha = TPLlamaDecoderLayer(LlamaConfig(hidden_size=2048, intermediate_size=2048, num_attention_heads=16, num_hidden_layers=1), 0, 0, 4)
        assert (mha.local_heads, mha.local_kv_heads, mha.rope_theta) == (4, 4, 10000.0)
