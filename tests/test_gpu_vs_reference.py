"""GPU parity suite, part 2 (-m gpu): our kernels against the REFERENCE'S OWN CUDA kernels.

The reference's torch-extension sources, compiled unmodified for sm_90a into oracle/_ref/libatom_ref.so (oracle/Makefile; the
INT4 mma.sync is emulated by ptxas on the INT8 pipe), were run on an H100 on the seeded inputs of every case below and their
outputs recorded in tests/golden/ref_kernels_h100.npz: small outputs in full, large ones as a SHA-256 digest of their bytes.
Outputs are compared bit for bit -- this is the strongest available statement of drop-in parity, because the reference ships
no golden vectors for its GEMM or decode kernels (SURVEY.md 8c).

To record again (after changing a case), build oracle/_ref where the reference tree is present and run this file on an H100
with ATOM_RECORD_REF=<output .npz>: every case then runs the reference kernel live, compares against it and stores it."""
import atexit
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle import ref_gpu as R

pytestmark = pytest.mark.gpu

_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_kernels_h100.npz")
_RECORD = os.environ.get("ATOM_RECORD_REF")
_FULL_BYTES = 16 * 1024          # outputs up to this size are stored in full
_recorded = {}
_golden = None


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _bytes(t):
    return np.ascontiguousarray(t.contiguous().cpu().numpy()).view(np.uint8).reshape(-1)


def _digest(u8):
    return np.frombuffer(hashlib.sha256(u8.tobytes()).digest(), dtype=np.uint8)


def _reference(key, live, full=False):
    """The reference kernel's outputs for case `key`, each as (bytes or None, digest).  `live` runs the kernel (recording only)."""
    global _golden
    if _RECORD:
        if not _recorded:
            atexit.register(lambda: np.savez_compressed(_RECORD, **_recorded))
        outs = []
        for i, t in enumerate(live()):
            u8 = _bytes(t)
            _recorded[f"{key}/{i}/sha256"] = _digest(u8)
            if full or u8.nbytes <= _FULL_BYTES:
                _recorded[f"{key}/{i}/bytes"] = u8
            outs.append((u8 if (full or u8.nbytes <= _FULL_BYTES) else None, _digest(u8)))
        return outs
    if _golden is None:
        _golden = np.load(_GOLDEN)
    n = sum(1 for k in _golden.files if k.startswith(key + "/") and k.endswith("/sha256"))
    assert n > 0, f"no recorded reference output for {key}"
    return [(_golden[f"{key}/{i}/bytes"] if f"{key}/{i}/bytes" in _golden.files else None, _golden[f"{key}/{i}/sha256"]) for i in range(n)]


def _same(ours, ref):
    u8 = _bytes(ours)
    return np.array_equal(u8, ref[0]) if ref[0] is not None else np.array_equal(_digest(u8), ref[1])


def _as(ref, dtype, shape):
    return ref[0].view(dtype).reshape(shape)


def _quant_parts(out, m):
    idx = torch.tensor([O.scale_index(r) + 2 * j for r in range(m) for j in range(4)], device="cuda:0")
    return [out[0], out[1], out[2][idx], out[3][:, idx]]


def _cmp_quant(ours, ref, m):
    ours = _quant_parts(ours, m)
    assert _same(ours[0], ref[0]), "INT8 outliers differ"
    assert _same(ours[1], ref[1]), "packed INT4 differs"
    assert _same(ours[2], ref[2]) and _same(ours[3], ref[3]), "scales differ"


@pytest.mark.parametrize("m", [1, 7, 16, 100, 1024])
def test_reorder_equals_reference_kernel(m):
    from atom_b200 import ops
    rng = np.random.default_rng(m)
    x = T((rng.standard_normal((m, 4096)) * 2).astype(np.float16)); idx = T(rng.permutation(4096).astype(np.int16))
    _cmp_quant(ops.reorder_fp16_i4(x, idx), _reference(f"reorder/{m}", lambda: _quant_parts(R.reorder_fp16_i4(x, idx), m)), m)


@pytest.mark.parametrize("m", [1, 7, 16, 100, 1024])
def test_rmsnorm_equals_reference_kernel(m):
    from atom_b200 import ops
    rng = np.random.default_rng(m + 1)
    x = T((rng.standard_normal((m, 4096)) * 2).astype(np.float16)); idx = T(rng.permutation(4096).astype(np.int16))
    w = T((1 + 0.2 * rng.standard_normal(4096)).astype(np.float16))
    _cmp_quant(ops.rmsnorm_fp16_i4(x, w, idx, 1e-5), _reference(f"rmsnorm/{m}", lambda: _quant_parts(R.rmsnorm_fp16_i4(x, w, idx, 1e-5), m)), m)


@pytest.mark.parametrize("m", [1, 7, 16, 100])
def test_activate_equals_reference_kernel(m):
    from atom_b200 import ops
    rng = np.random.default_rng(m + 2)
    a = T((rng.standard_normal((m, 11008)) * 2).astype(np.float16)); b = T((rng.standard_normal((m, 11008)) * 2).astype(np.float16))
    _cmp_quant(ops.activate_fp16_i4(a, b), _reference(f"activate/{m}", lambda: _quant_parts(R.activate_fp16_i4(a, b), m)), m)


@pytest.mark.parametrize("m,n,k,flags", [(16, 4096, 4096, 1), (7, 4096, 4096, 1), (128, 4096, 4096, 1), (128, 4096, 4096, 2), (1000, 4096, 4096, 0),
                                         (4096, 4096, 4096, 0), (16, 11008, 4096, 1), (33, 4096, 11008, 1), (300, 4096, 11008, 0),
                                         # Llama-13B (config #4) and Llama-65B TP-8 (config #5) projection shapes, decode batch 32
                                         (32, 5120, 5120, 1), (32, 13824, 5120, 1), (32, 5120, 13824, 1), (32, 1024, 8192, 1),
                                         (32, 8192, 2816, 1), (32, 8192, 2688, 1), (64, 8192, 1024, 1),
                                         # prefill: the 7B MLP up-projection and config #3's 16 x 2048 tokens
                                         (4096, 11008, 4096, 0), (32768, 4096, 4096, 0),
                                         # the same prefill shapes forced through each of the two prefill kernels
                                         (4096, 4096, 4096, 512), (4096, 4096, 4096, 1024), (1000, 11008, 4096, 512)])
def test_gemm_o16_equals_reference_kernel(m, n, k, flags):
    from atom_b200 import ops
    t = [T(x) for x in O.make_gemm_inputs(m, n, k, seed=m + n + k, pair_shared=(m % 2 == 0))]
    ours = ops.dense_layer_gemm_i4_fp16(*t, flags=flags)
    ref = _reference(f"gemm_o16/{m}-{n}-{k}", lambda: [R.gemm_i4_o16(*t)])[0]
    assert _same(ours, ref), f"fp16 outputs differ from the reference kernel's ({ours.numel()} values)"


def test_gemm_o16_splitk_within_one_ulp_of_reference_kernel():
    from atom_b200 import ops
    t = [T(x) for x in O.make_gemm_inputs(16, 4096, 4096, seed=3)]
    ours = ops.dense_layer_gemm_i4_fp16(*t, flags=0).float()
    # the un-split result is the reference's bit for bit (checked here by digest), so it stands in for it below
    nosplit = ops.dense_layer_gemm_i4_fp16(*t, flags=1)
    assert _same(nosplit, _reference("gemm_o16_splitk", lambda: [R.gemm_i4_o16(*t)])[0])
    ref = nosplit.float()
    assert torch.allclose(ours, ref, rtol=1e-3, atol=1e-3 * ref.abs().mean().item())
    assert (ours != ref).float().mean().item() < 0.02


@pytest.mark.parametrize("m,flags", [(16, 1), (16, 0), (33, 0), (100, 0), (1000, 0)])      # flags 0 = the default dispatch (o4 never splits K)
def test_gemm_o4_equals_reference_kernel(m, flags):
    from atom_b200 import ops
    t = [T(x) for x in O.make_gemm_inputs(m, 4096, 4096, seed=m)]
    d, ds = ops.dense_layer_gemm_i4_o4(*t, flags=flags)
    rd, rds = _reference(f"gemm_o4/{m}", lambda: R.gemm_i4_o4(*t))
    assert _same(ds, rds), "o4 (scale, zero) differ"
    assert _same(d, rd), "o4 packed values differ"


def test_batch_decode_at_least_as_close_to_the_oracle_as_the_reference_kernel():
    """Both kernels approximate transcendentals (the reference: __powf / __sincosf per element; ours: a rotation table and
    packed FP16 dequantisation), so neither is the other's bit pattern.  Judge both against the CPU oracle (float math,
    decode.cuh:480-689 restated): ours must meet rtol = atol = 5e-4 and must not be further from it than the reference is."""
    from atom_b200 import ops
    from tests.test_gpu_parity import _kv_fixture, _KV
    rng = np.random.default_rng(0xabc)
    B, H, P, L = 7, 32, 16, 3
    lens = rng.integers(1, 500, B).tolist()
    data, param, indptr, indices, last = _kv_fixture(rng, B, H, P, L, lens)
    kv = _KV(data, param, indptr, indices, last)
    qn = rng.standard_normal((B, H, 128)).astype(np.float16)
    q = T(qn)
    for layer in range(L):
        ours = ops.batch_decode_i4(q, kv, layer).float().cpu().numpy()
        ref = _reference(f"batch_decode/{layer}", lambda: [R.batch_decode_i4(q, kv.data, kv.param, kv.indptr, kv.indicies, kv.last_page_offset, layer)], full=True)[0]
        ref = _as(ref, np.float16, (B, H, 128)).astype(np.float32)
        orc = O.batch_decode_i4(qn, data, param, indptr, indices, last, layer).astype(np.float32)
        e_ours = (np.abs(ours - orc) - 5e-4 * np.abs(orc)).max()
        e_ref = (np.abs(ref - orc) - 5e-4 * np.abs(orc)).max()
        assert e_ours <= 5e-4, f"layer {layer}: ours exceeds 5e-4 by {e_ours:.2e} (reference kernel: {e_ref:.2e})"
        assert np.abs(ours - orc).max() <= max(np.abs(ref - orc).max() * 1.5, 2e-4), (np.abs(ours - orc).max(), np.abs(ref - orc).max())


def test_append_kv_equals_reference_kernel():
    from atom_b200 import ops
    from tests.test_gpu_parity import _kv_fixture, _KV
    rng = np.random.default_rng(9)
    B, H, P, L = 4, 32, 16, 2
    lens = [1, 16, 17, 300]
    data, param, indptr, indices, last = _kv_fixture(rng, B, H, P, L, lens)
    k = T(rng.integers(0, 256, (B, H, 64), dtype=np.uint8)); v = T(rng.integers(0, 256, (B, H, 64), dtype=np.uint8))
    kp = T(rng.random((B, H, 2)).astype(np.float16)); vp = T(rng.random((B, H, 2)).astype(np.float16))
    a = _KV(data, param, indptr, indices, last)
    ops.append_kv_i4(a, k, v, kp, vp, 1)

    def live():
        b = _KV(data, param, indptr, indices, last)
        R.append_kv_i4(b.data, b.param, b.indptr, b.indicies, b.last_page_offset, k, v, kp, vp, 1)
        return [b.data, b.param]
    rdata, rparam = _reference("append_kv", live)
    assert _same(a.data, rdata) and _same(a.param, rparam)
