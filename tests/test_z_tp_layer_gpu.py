"""GPU suite (-m gpu): the tensor-parallel decode layer (atom_b200/tp.py) with 1, 2, 4 and 8 ranks emulated on one GPU, every kernel
call of every rank checked against tests/tp_ref64.py.

Each rank is a Python thread; every kernel of every rank goes to ONE CUDA stream (PDL off).  A rank's all-reduce object holds an
ops.ArHandle over W receive buffers and W state blocks on the one GPU (as test_push_multi_rank_on_one_gpu builds them), so the push
GEMM and the reducing add+RMSNorm are the real kernels; reduce_add_rmsnorm_fp16_i4 first waits at a host barrier of the ranks, so
every rank's push GEMM is queued ahead of every rank's reduce and no polling kernel waits on work queued behind it.  The stand-alone
all-reduce (batches > 64, hidden % 1024 != 0, fuse off) is the rank-order FP32 sum in torch after the same barrier; the one-shot
all-reduce kernel is never launched at world > 1 here, its poll would wait on kernels queued after it."""
import numpy as np
import pytest
import torch

from tests import layer_ref64 as R
from tests import tp_ref64 as T

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
TOY_BATCHES = (16, 64, 65, 3, 33)          # push, push at the 64-row limit, stand-alone, push, push: the written extent shrinks and grows


def _config(hidden, inter, heads, kv_heads=None, theta=1e4):
    from atom_b200.llama import LlamaConfig
    return LlamaConfig(hidden_size=hidden, intermediate_size=inter, num_attention_heads=heads, num_key_value_heads=kv_heads,
                       num_hidden_layers=2, rope_theta=theta)


class Ranks:
    """`world` emulated ranks of a chain of `layers` TPLlamaDecoderLayers, each rank on its own KV pool of sequences `lens`."""

    def __init__(self, monkeypatch, cfg, world, lens, P=16, fuse=True, layers=2, row_cap=1 << 27, check=True, seed=1):
        from atom_b200 import _lib, ops
        from atom_b200.kvcache import KvCacheInt4, KvPoolInt4
        self.world, self.check = world, check
        self.rdv = T.Rendezvous(world, timeout=120)
        real = ops.reduce_add_rmsnorm_fp16_i4

        def reduce_after_every_push(pending, residual, weight, reorder_index, eps):
            self.rdv.wait()
            return real(pending, residual, weight, reorder_index, eps)
        self.rec = T.TPRecorder(world, {"reduce_add_rmsnorm_fp16_i4": reduce_after_every_push}).install(monkeypatch)
        slot = 64 * cfg.hidden_size                  # a batch of 65 cannot push
        self.bufs = [torch.full((3 * world * slot,), -32768, dtype=torch.int16, device=DEV) for _ in range(world)]
        self.table = torch.tensor([b.data_ptr() for b in self.bufs], dtype=torch.int64, device=DEV)
        self.states = [torch.zeros(_lib.lib().atom_allreduce_state_words(), dtype=torch.int32, device=DEV) for _ in range(world)]
        ars = [None] * world
        if world > 1:
            ars = [T.EmulatedAllReduce(r, self.rdv, self.rec, ops.ArHandle(self.table.data_ptr(), self.states[r], slot, r, world), slot,
                                       fuse) for r in range(world)]
        self.ranks = T.make_ranks(cfg, world, layers, DEV, ars, seed=seed)
        hkv = self.ranks[0][0].local_kv_heads
        pages = sum(-(-(n + 8) // P) for n in lens) + 2
        self.pools, self.seqs = [], []
        for r in range(world):
            pool = KvPoolInt4(layers, hkv, 128, pages, P, DEV)
            g = torch.Generator(device=DEV).manual_seed(100 * seed + r)
            pool.buf.copy_(torch.randint(0, 256, pool.buf.shape, dtype=torch.uint8, device=DEV, generator=g))
            pool.param[..., 0].uniform_(0.01, 0.05, generator=g)
            pool.param[..., 1].uniform_(0.0, 0.4, generator=g)
            self.pools.append(pool)
            self.seqs.append([KvCacheInt4(pool, n) for n in lens])
        self.ref = T.TPRef(self.ranks, P, fuse, slot, row_cap) if check else None
        self.rng = np.random.default_rng(seed)
        self.stream = torch.cuda.Stream(DEV)

    def step(self, b):
        """One decode step of the first b sequences on every rank; checked against the reference.  Returns rank 0's output."""
        from atom_b200.kvcache import BatchedKvCacheInt4
        x = torch.from_numpy((self.rng.standard_normal((b, self.ranks[0][0].q_proj.in_features)) * 0.5).astype(np.float16)).to(DEV)
        kvs = []
        for r in range(self.world):
            for c in self.seqs[r][:b]:
                c.acquire_one()
            kvs.append(BatchedKvCacheInt4(self.seqs[r][:b]))
        for t in self.rec.traces:
            t.clear()
        before = [(R.host(p.buf), R.host(p.param)) for p in self.pools]
        self.stream.wait_stream(torch.cuda.current_stream(DEV))
        outs = T.run_ranks(self.world, lambda r: T.chain_step(self.ranks[r], x, kvs[r]), self.rec, self.rdv, self.stream)
        torch.cuda.synchronize(DEV)
        after = [(R.host(p.buf), R.host(p.param)) for p in self.pools]
        if self.check:
            self.ref.check_step([list(t) for t in self.rec.traces], R.host(x), R.host(kvs[0]), [R.host(o) for o in outs], before, after)
        return R.host(outs[0]), after

    def pushes(self):
        return [int(s[0]) for s in self.states]


def _lens(n, P):
    return [P - 3 + (7 * i) % (3 * P) for i in range(n)]    # crossing page boundaries within the steps


@pytest.mark.timeout(900)
@pytest.mark.parametrize("world,kv_heads", [(1, None), (2, None), (4, None), (8, None), (4, 4), (8, 8)])
def test_toy_chain_decode_steps(monkeypatch, world, kv_heads):
    """hidden 2048, inter 5632 (768 / 640 at 8 ranks), 16 query heads, MHA or one KV head per rank; two chained layers over the
    batches 16, 64, 65, 3, 33: the fused push and the stand-alone all-reduce alternate and the written slot extent changes."""
    run = Ranks(monkeypatch, _config(2048, 5632, 16, kv_heads), world, _lens(65, 16), row_cap=1 << 24)
    for b in TOY_BATCHES:
        run.step(b)
    if world > 1:
        assert run.ranks[0][0].o_proj.can_push(64) and not run.ranks[0][0].o_proj.can_push(65)
        assert run.pushes() == [3 * (len(TOY_BATCHES) - 1)] * world       # o_proj twice and layer 0's down per pushed step


@pytest.mark.timeout(600)
def test_hidden_not_a_multiple_of_1024_takes_the_standalone_allreduce(monkeypatch):
    """hidden 1280 (10 heads) over 2 ranks: can_push is false at every batch, every all-reduce is the stand-alone one."""
    run = Ranks(monkeypatch, _config(1280, 3456, 10), 2, _lens(33, 16))
    assert not run.ranks[0][0].o_proj.can_push(16)
    for b in (16, 33, 5):
        run.step(b)
    assert run.pushes() == [0, 0]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kv_heads", [None, 8])
def test_bench_shape_one_step_at_8_ranks(monkeypatch, kv_heads):
    """The `tp` record's shape (hidden 8192, inter 22016 -> 2816 / 2688, 64 heads, page 32, batch 32) at 8 ranks, MHA and GQA 64/8 (one
    KV head per rank, G = 8), with KV lengths about 300; the oracle GEMMs run on row subsets."""
    run = Ranks(monkeypatch, _config(8192, 22016, 64, kv_heads), 8, [290 + 3 * i for i in range(32)], P=32)
    assert run.ranks[0][0].inter_sizes == [2816] * 4 + [2688] * 4
    run.step(32)
    assert run.pushes() == [3] * 8


@pytest.mark.timeout(900)
@pytest.mark.parametrize("world", [2, 8])
def test_fused_and_unfused_allreduce_agree(monkeypatch, world):
    """fuse = False (the stand-alone all-reduce at every batch) gives the fused run's outputs and pools bit for bit; the unfused run
    is checked against the reference too."""
    cfg = _config(2048, 5632, 16)
    fused = Ranks(monkeypatch, cfg, world, _lens(33, 16), check=False)
    steps = [fused.step(b) for b in (16, 33, 3)]
    monkeypatch.undo()                                  # the unfused run records with its own recorder
    unfused = Ranks(monkeypatch, cfg, world, _lens(33, 16), fuse=False, row_cap=1 << 24)
    for b, (out_f, pools_f) in zip((16, 33, 3), steps):
        out_u, pools_u = unfused.step(b)
        assert R.same(out_f, out_u), f"batch {b}: outputs differ"
        for r, ((bf, pf), (bu, pu)) in enumerate(zip(pools_f, pools_u)):
            assert R.same(bf, bu) and R.same(pf, pu), f"batch {b}: rank {r}'s pool differs"
    assert fused.pushes() == [9] * world and unfused.pushes() == [0] * world       # 3 steps x (o_proj twice, layer 0's down)


def _llama_twin(tp):
    """A LlamaDecoderLayer holding the parameters of the world-1 TP layer `tp`, fused after the copy (fuse_linear_rows copies the
    scales: operands fused before the copy would be stale)."""
    from atom_b200.llama import LlamaDecoderLayer
    from atom_b200.llama import LlamaConfig
    h = tp.q_proj.in_features
    cfg = LlamaConfig(hidden_size=h, intermediate_size=tp.gate_proj.out_features, num_attention_heads=tp.local_heads,
                      num_key_value_heads=tp.local_kv_heads, num_hidden_layers=1, rope_theta=tp.rope_theta)
    twin = LlamaDecoderLayer(cfg, tp.layer_idx).to(DEV).init_random(99)
    a, m = twin.self_attn, twin.mlp
    pairs = [(a.q_proj, tp.q_proj), (a.k_proj, tp.k_proj), (a.v_proj, tp.v_proj), (a.o_proj, tp.o_proj.local), (m.gate_proj, tp.gate_proj),
             (m.up_proj, tp.up_proj), (m.down_proj, tp.down_proj.local)]
    with torch.no_grad():
        for dst, src in pairs:
            for name in ("weight_int4", "weight_int8", "scale_int4", "scale_int8"):
                getattr(dst, name).copy_(getattr(src, name))
        for dst, src in ((twin.input_layernorm, tp.input_layernorm), (twin.post_attention_layernorm, tp.post_attention_layernorm)):
            dst.weight.copy_(src.weight)
            dst.reorder_index.copy_(src.reorder_index)
        a.reorder_index.copy_(tp.attn_reorder_index)
    return twin.fuse().eval()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("batch", [32, 65])
def test_world_1_equals_llama_decoder_layer(monkeypatch, batch):
    """At world 1 the TP layer is LlamaDecoderLayer: same K/V bytes and, at batch 32, the same output bit for bit.  At 65 the TP
    layer runs q_proj as its own GEMM (split-K under the automatic rule at M = 65) while LlamaAttention keeps the fused, un-split q/k/v
    launch, so only the K/V bytes are compared; both layers' steps are held to the reference."""
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4
    run = Ranks(monkeypatch, _config(2048, 5632, 16, 8), 1, _lens(batch, 16), layers=1, row_cap=1 << 24)
    pool = run.pools[0]
    buf, param = pool.buf.clone(), pool.param.clone()
    out_tp, _ = run.step(batch)
    tp_pool = (pool.buf.clone(), pool.param.clone())
    pool.buf.copy_(buf)
    pool.param.copy_(param)
    twin = _llama_twin(run.ranks[0][0])
    x = torch.from_numpy(R.host(run.rec.traces[0][0].args["hidden_states"])).to(DEV)
    monkeypatch.undo()
    rec = R.Recorder().install(monkeypatch)
    with torch.inference_mode():
        out, step, calls, before, after = R.run_step(rec, pool, twin, x, BatchLenInfo([], batch, DEV), None,
                                                     BatchedKvCacheInt4(run.seqs[0][:batch]), ids=False)
    ref = R.ModelRef([R.LayerParams(twin, 0)], 16, row_cap=1 << 24)
    T.seed_history(ref, step.dtab, before)
    ref.check_step(calls, step, before, after)
    assert torch.equal(tp_pool[0], pool.buf) and torch.equal(tp_pool[1].view(torch.int16), pool.param.view(torch.int16))
    if batch <= 64:
        assert R.same(out_tp, step.out)


@pytest.mark.timeout(300)
def test_world_1_chain_replays_from_a_cuda_graph():
    """A two-layer chained world-1 decode step replayed from a CUDA graph (what bench.py's `tp` record times on one GPU) equals the
    eager step: output and pool bit for bit."""
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    layers = T.make_ranks(_config(2048, 5632, 16), 1, 2, DEV, [None], seed=4)[0]
    pool = KvPoolInt4(2, 16, 128, 128, 16, DEV)
    pool.buf.random_(0, 256)
    pool.param.uniform_(0.01, 0.05)
    seqs = [KvCacheInt4(pool, n) for n in _lens(32, 16)]
    for c in seqs:
        c.acquire_one()
    kv = BatchedKvCacheInt4(seqs)
    x = torch.randn(32, 2048, device=DEV, dtype=torch.float16)
    buf, param = pool.buf.clone(), pool.param.clone()
    st = torch.cuda.Stream(DEV)
    st.wait_stream(torch.cuda.current_stream(DEV))
    with torch.inference_mode(), torch.cuda.stream(st):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            y = T.chain_step(layers, x, kv)
        g.replay()
        st.synchronize()
        graphed, graphed_pool = y.clone(), (pool.buf.clone(), pool.param.clone())
        pool.buf.copy_(buf)
        pool.param.copy_(param)
        eager = T.chain_step(layers, x, kv)
        st.synchronize()
    assert torch.equal(graphed, eager)
    assert torch.equal(graphed_pool[0], pool.buf) and torch.equal(graphed_pool[1].view(torch.int16), pool.param.view(torch.int16))
