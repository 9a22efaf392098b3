"""The push all-reduce kernel (csrc/comm_kernels.cuh) on ONE GPU: with world == 1 the "peer" table holds the local buffer,
so the full protocol runs (push into slot [e % 3][0], reset of the previous buffer to the sentinel, poll, FP32 reduction,
call counter) and the result must equal the input bit for bit (-0.0 arrives as +0.0) -- eagerly, with sizes that grow and
shrink between calls and leave CTAs without work, and across CUDA-graph replays (the buffer rotation is driven by the
device-side counter).  The N >= 2 behaviour is covered by tools/tp_check.py under torchrun
(several GPUs) and the host logic by tests/test_tp_gloo.py."""
import pytest
import torch

from atom_b200 import _lib

pytestmark = pytest.mark.gpu


def _setup(slot, dev):
    buf = torch.full((3 * 1 * slot,), -32768, dtype=torch.int16, device=dev)  # [3][world=1][slot] of 0x8000 (FP16 -0.0)
    state = torch.zeros(_lib.lib().atom_allreduce_state_words(), dtype=torch.int32, device=dev)
    bufs = torch.tensor([buf.data_ptr()], dtype=torch.int64, device=dev)
    return buf, state, bufs


def _call(x, out, st, slot):
    buf, state, bufs = st
    _lib.check(_lib.lib().atom_allreduce_push_f16(x.data_ptr(), out.data_ptr(), bufs.data_ptr(), state.data_ptr(),
                                                  x.numel(), slot, 0, 1, torch.cuda.current_stream().cuda_stream), "allreduce_push_f16")


def test_world1_identity_and_epochs():
    dev = torch.device("cuda", 0)
    slot = 32 * 8192
    st = _setup(slot, dev)
    for it, n in enumerate([8, 64, 4096, 32 * 5120, slot, 2048, slot, 8, slot]):
        torch.manual_seed(it)
        x = (torch.randn(n, device=dev) * 5).half()
        x[::7] = -0.0                                           # the sentinel pattern as payload: must arrive as +0.0
        x[3::11] = 0.0
        out = torch.full_like(x, 7.0)
        _call(x, out, st, slot)
        torch.cuda.synchronize()
        assert torch.equal(out, x), f"call {it} (numel {n})"   # (-0.0 == +0.0 under torch.equal)
        assert not (out.view(torch.int16) == -32768).any(), "-0.0 must be delivered as +0.0"
    assert int(st[1][0]) == 9 and int(st[1][1]) == 0           # nine completed calls, ticket counter back at zero
    torch.cuda.synchronize()
    # after the last call only the buffer it used holds payload; the one before it has been reset
    b3 = st[0].view(3, slot)
    assert (b3[(9 + 2) % 3] == -32768).all()


def test_world1_graph_replay():
    dev = torch.device("cuda", 0)
    slot = 16 * 4096
    st = _setup(slot, dev)
    x = torch.zeros(slot, dtype=torch.float16, device=dev)
    outs = [torch.empty_like(x) for _ in range(3)]
    s = torch.cuda.Stream(dev)
    with torch.cuda.stream(s):
        _call(x, outs[0], st, slot)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            _call(x, outs[0], st, slot)            # three chained all-reduces per replay: odd count, so the parity of the
            _call(outs[0], outs[1], st, slot)      # first call alternates between replays
            _call(outs[1], outs[2], st, slot)
        for rep in range(5):
            torch.manual_seed(100 + rep)
            x.copy_((torch.randn(slot, device=dev) * 3).half())
            g.replay()
            s.synchronize()
            assert torch.equal(outs[2], x), f"replay {rep}"


def test_argument_validation():
    dev = torch.device("cuda", 0)
    st = _setup(1024, dev)
    x = torch.zeros(1024 + 8, dtype=torch.float16, device=dev)
    with pytest.raises(RuntimeError):
        _call(x, torch.empty_like(x), st, 1024)      # numel > slot
    y = torch.zeros(12, dtype=torch.float16, device=dev)
    with pytest.raises(RuntimeError):
        _call(y, torch.empty_like(y), st, 1024)      # numel % 8 != 0


def test_world1_fused_gemm_push_and_reducing_rmsnorm():
    """The fused pair (row-parallel GEMM pushes from its epilogue, add+RMSNorm+quantise reduces while it loads) against the unfused
    sequence GEMM -> add_rmsnorm on one GPU (world == 1: the sum has one term, so everything is bit-identical), over several calls
    (buffer rotation), interleaved with stand-alone all-reduces on the same buffers, eagerly and from a CUDA graph."""
    import numpy as np
    from atom_b200 import ops
    from oracle import oracle as O
    dev = torch.device("cuda", 0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    slot = 64 * 4096
    st = _setup(slot, dev)
    h = ops.ArHandle(st[2].data_ptr(), st[1], slot, 0, 1)
    for it, (m, n, k) in enumerate([(16, 4096, 1024), (32, 4096, 512), (7, 2048, 1024), (64, 1024, 512), (16, 4096, 4096)]):
        t = [T(x) for x in O.make_gemm_inputs(m, n, k, seed=900 + it)]
        rng = np.random.default_rng(it)
        res = T((rng.standard_normal((m, n)) * 2).astype(np.float16))
        w = T((1 + 0.2 * rng.standard_normal(n)).astype(np.float16))
        idx = T(rng.permutation(n).astype(np.int16))
        torch.cuda.synchronize()
        flags = 1 | 4                                  # no split-K, decode kernel: the association of the reference
        d = ops.dense_layer_gemm_i4_fp16(*t, flags=flags)
        s_ref, q_ref = ops.add_rmsnorm_fp16_i4(d, res, w, idx, 1e-5)
        pend = ops.dense_layer_gemm_i4_fp16_push(*t, h, flags=flags)
        s, q = ops.reduce_add_rmsnorm_fp16_i4(pend, res, w, idx, 1e-5)
        torch.cuda.synchronize()
        assert torch.equal(s, s_ref), f"case {it}: sum differs"
        for a, b in zip(q[:2], q_ref[:2]):
            assert torch.equal(a, b), f"case {it}: quantised operand differs"
        if it % 2 == 1:                                # a stand-alone all-reduce in between: same counter, same buffers
            x = (torch.randn(4096, device=dev) * 3).half()
            out = torch.empty_like(x)
            _call(x, out, st, slot)
            torch.cuda.synchronize()
            assert torch.equal(out, x)
    # split-K path (default dispatch) + graph replay: three fused pairs per replay
    t = [T(x) for x in O.make_gemm_inputs(16, 4096, 4096, seed=77)]
    res = torch.zeros(16, 4096, dtype=torch.float16, device=dev)
    w = torch.ones(4096, dtype=torch.float16, device=dev)
    idx = torch.arange(4096, dtype=torch.int16, device=dev)
    torch.cuda.synchronize()
    d = ops.dense_layer_gemm_i4_fp16(*t)               # auto: split-K, deterministic
    s_ref, q_ref = ops.add_rmsnorm_fp16_i4(d, res, w, idx, 1e-5)
    sstream = torch.cuda.Stream(dev)
    with torch.cuda.stream(sstream):
        ops.reduce_add_rmsnorm_fp16_i4(ops.dense_layer_gemm_i4_fp16_push(*t, h), res, w, idx, 1e-5)
        sstream.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=sstream):
            outs = [ops.reduce_add_rmsnorm_fp16_i4(ops.dense_layer_gemm_i4_fp16_push(*t, h), res, w, idx, 1e-5) for _ in range(3)]
        for rep in range(4):
            g.replay()
            sstream.synchronize()
            for s, q in outs:
                assert torch.equal(s, s_ref) and torch.equal(q[1], q_ref[1]), f"replay {rep}"
