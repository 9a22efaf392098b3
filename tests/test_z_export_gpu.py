"""GPU suite (-m gpu), sorted last on purpose: a layer calibrated with the model/ surface (QLlamaDecoderLayer: reorder ->
RTN quantise -> activation quantisers), exported with .to_int4(), must give on the sm_90a kernels what the oracle's
restatement of the kernel chain gives on the same exported operands, and stay within quantisation noise of the simulator."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests.test_export_cpu import _build, _gemm, _input, _np

pytestmark = pytest.mark.gpu


def test_exported_mlp_branch_on_kernels_matches_oracle_chain_and_simulator():
    q, a = _build(hidden=512, inter=1024, heads=4, seed=5)
    real = q.to_int4("cuda:0")
    x = _input(9, 512, 7)
    n = real.post_attention_layernorm
    got = real.mlp(n(x.cuda())).float().cpu().numpy()
    cpu = real.cpu()
    h = O.rmsnorm_fp16_i4(_np(x), _np(cpu.post_attention_layernorm.weight), _np(cpu.post_attention_layernorm.reorder_index),
                          n.variance_epsilon)
    gate, up = _gemm(h, cpu.mlp.gate_proj), _gemm(h, cpu.mlp.up_proj)
    ref = _gemm(O.activate_fp16_i4(gate, up), cpu.mlp.down_proj).astype(np.float32)
    # kernels vs oracle chain: every stage is bit-exact or within one quantisation LSB on isolated elements
    assert np.abs(got - ref).max() <= 0.03 * np.abs(ref).max()
    sim = _np(q.mlp(q.post_attention_layernorm(x.float()[None]))[0])
    assert np.abs(got - sim).max() <= 0.20 * np.abs(sim).max()     # oracle chain vs simulator is 8 % here (CPU-checked)
