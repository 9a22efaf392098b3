"""CPU self-test of tests/tp_ref64.py.  The real TPLlamaDecoderLayer code runs on the CPU with its ranks in threads, every kernel
replaced by its oracle (the operators of tests/test_layer_ref64_cpu.py) and the two halves of the push all-reduce emulated on the
oracle: the push GEMM keeps its rank's oracle partial, the reducing add+RMSNorm meets the other ranks at the rendezvous and sums
all of them.  The reference must (a) accept the traces of two chained layers at worlds 2 and 4, at batches on either side of 64,
and (b) reject each seeded fault with an error naming the rank, the layer and the stage."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import layer_ref64 as R
from tests import test_layer_ref64_cpu as C
from tests import tp_ref64 as T

P = 8
CPU = torch.device("cpu")


def _config(heads, kv_heads, hidden=1024, inter=1408):
    from atom_b200.llama import LlamaConfig
    return LlamaConfig(hidden_size=hidden, intermediate_size=inter, num_attention_heads=heads, num_key_value_heads=kv_heads,
                       num_hidden_layers=2, rope_theta=5e5)


class Harness:
    """World ranks of a two-layer TP chain on the oracle, each on its own pool; `fault` seeds one of FAULTS."""

    def __init__(self, monkeypatch, world, cfg, fault=None, batch=70):
        from atom_b200 import ops
        from atom_b200.kvcache import KvCacheInt4, KvPoolInt4
        self.world, self.fault = world, fault
        self.rdv = T.Rendezvous(world, timeout=60)
        impl = dict(C.ORACLE_OPS)
        impl.update(dense_layer_gemm_i4_fp16_push=self._push, reduce_add_rmsnorm_fp16_i4=self._reduce)
        self.rec = T.TPRecorder(world, impl)
        self.rec.install(monkeypatch)
        self._mine = [None] * world
        slot = 64 * cfg.hidden_size
        self.ars = [T.EmulatedAllReduce(r, self.rdv, self.rec, ops.ArHandle(0, None, slot, r, world), slot) for r in range(world)]
        self.ranks = T.make_ranks(cfg, world, 2, CPU, self.ars, seed=3)
        for chain in self.ranks:
            for layer in chain:
                layer.fuse()                      # init_random fuses on CUDA only
        if fault == "replicated_norm_differs":
            with torch.no_grad():
                self.ranks[1][1].post_attention_layernorm.weight[5] += 0.25
        hkv = self.ranks[0][0].local_kv_heads
        self.pools, self.seqs = [], []
        lens = [1 + (5 * i) % 13 for i in range(batch)]
        for r in range(world):
            pool = KvPoolInt4(2, hkv, 128, batch * 3 + 2, P, CPU)
            g = torch.Generator().manual_seed(40 + r)
            pool.buf.copy_(torch.randint(0, 256, pool.buf.shape, dtype=torch.uint8, generator=g))
            pool.param.copy_((torch.rand(pool.param.shape, generator=g) * 0.05).half())
            self.pools.append(pool)
            self.seqs.append([KvCacheInt4(pool, n) for n in lens])
        self.ref = T.TPRef(self.ranks, P, slot=slot)
        self.rng = np.random.default_rng(1)
        if fault in FAULTS:
            FAULTS[fault](self, monkeypatch)

    # ---- the push all-reduce's halves, on the oracle
    def _push(self, a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, ar, flags=0):
        self._mine[ar.rank] = C.dense_layer_gemm_i4_fp16(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale)
        from atom_b200 import ops
        return ops.PendingAllReduce(ar, (a.shape[0], b.shape[0]), a.device)

    def _reduce(self, pending, residual, weight, reorder_index, eps):
        parts = self.rdv.exchange(pending.ar.rank, self._mine[pending.ar.rank])
        if self.fault == "partial_missing":
            parts = parts[:1] + parts[2:]
        if self.fault == "fp16_accumulation":
            total = parts[0].clone()
            for p in parts[1:]:
                total = (total.double() + p.double()).half()
        else:
            total = T.torch_allreduce_sum(parts)
        return C.add_rmsnorm_fp16_i4(total, residual, weight, reorder_index, eps)

    def step(self, b):
        from atom_b200.kvcache import BatchedKvCacheInt4
        x = torch.from_numpy((self.rng.standard_normal((b, self.ranks[0][0].q_proj.in_features)) * 0.5).astype(np.float16))
        kvs = []
        for r in range(self.world):
            for c in self.seqs[r][:b]:
                c.acquire_one()
            kvs.append(BatchedKvCacheInt4(self.seqs[r][:b]))
        for t in self.rec.traces:
            t.clear()
        before = [(R.host(p.buf), R.host(p.param)) for p in self.pools]
        try:
            outs = T.run_ranks(self.world, lambda r: T.chain_step(self.ranks[r], x, kvs[r]), self.rec, self.rdv)
        except RuntimeError:              # a rank stopped on a shape error: its trace up to there names the stage that went wrong
            self.ref.check_step([list(t) for t in self.rec.traces], R.host(x), R.host(kvs[0]), [None] * self.world, before)
            raise
        after = [(R.host(p.buf), R.host(p.param)) for p in self.pools]
        self.ref.check_step([list(t) for t in self.rec.traces], R.host(x), R.host(kvs[0]), [R.host(o) for o in outs], before, after)
        return [list(t) for t in self.rec.traces]


# ---- seeded faults (each wraps an operator or a layer method; the reduce-side ones are in Harness._reduce)
def _kv_into_other_rank(h, monkeypatch):
    """Rank 1's append_kv kernel stores into rank 0's pool."""
    from atom_b200 import ops
    f = ops.append_kv_i4
    pool0 = h.pools[0]

    def append(kv, k, v, kp, vp, l):
        if h.rec._local.rank == 1:
            kv = type("KV", (), dict(data=pool0.buf, param=pool0.param, indptr=kv.indptr, indicies=kv.indicies,
                                     last_page_offset=kv.last_page_offset))()
        return f(kv, k, v, kp, vp, l)
    monkeypatch.setattr(ops, "append_kv_i4", append)


def _kv_into_other_layer(h, monkeypatch):
    """Rank 1 writes layer 0's K/V into layer 1's slots."""
    from atom_b200 import ops
    f = ops.append_kv_i4
    monkeypatch.setattr(ops, "append_kv_i4", lambda kv, k, v, kp, vp, l: f(kv, k, v, kp, vp, 1 if h.rec._local.rank == 1 else l))


def _other_rank_reorder(h, monkeypatch):
    """Rank 1 quantises its attention output with rank 0's attn_reorder_index."""
    from atom_b200 import ops
    f = ops.reorder_fp16_i4

    def reorder(x, idx):
        for mine, theirs in zip(h.ranks[1], h.ranks[0]):
            if idx is mine.attn_reorder_index:
                idx = theirs.attn_reorder_index
        return f(x, idx)
    monkeypatch.setattr(ops, "reorder_fp16_i4", reorder)


def _pending_reduced_twice(h, monkeypatch):
    """The next layer's input norm reduces the pending down projection into the residual, then does it once more."""
    from atom_b200.llama import LlamaRMSNormInt4
    from atom_b200 import ops
    f = LlamaRMSNormInt4.forward_add

    def forward_add(self, hidden_states, residual):
        if isinstance(hidden_states, ops.PendingAllReduce) and self is h.ranks[h.rec._local.rank][1].input_layernorm:
            residual, _ = f(self, hidden_states, residual)
        return f(self, hidden_states, residual)
    monkeypatch.setattr(LlamaRMSNormInt4, "forward_add", forward_add)


def _kv_rows_one_head_short(h, monkeypatch):
    """The fused q/k/v launch is told one KV head fewer than the rank holds."""
    from atom_b200 import ops
    f = ops.dense_layer_gemm_i4_qkv

    def qkv(*a, kv_rows=None, **k):
        return f(*a, kv_rows=kv_rows - 128, **k)
    monkeypatch.setattr(ops, "dense_layer_gemm_i4_qkv", qkv)


FAULTS = {"kv_into_other_rank": _kv_into_other_rank, "kv_into_other_layer": _kv_into_other_layer,
          "other_rank_reorder": _other_rank_reorder, "pending_reduced_twice": _pending_reduced_twice,
          "kv_rows_one_head_short": _kv_rows_one_head_short}


@pytest.mark.parametrize("world,heads,kv_heads", [(2, 8, 8), (4, 8, 4)])
def test_reference_accepts_the_oracle_trace(monkeypatch, world, heads, kv_heads):
    """Batches 5 (push all-reduce), 70 (stand-alone all-reduce, unfused q/k/v and gate/up) and 33: the first step of a sequence
    reads its history from the pool, later steps extend it."""
    h = Harness(monkeypatch, world, _config(heads, kv_heads))
    names = [[c.name for c in h.step(b)[0]] for b in (5, 70, 33)]
    for b, n in zip((5, 70, 33), names):       # the last layer's down_proj never pushes
        pushes = 0 if b > 64 else 3
        assert (n.count("dense_layer_gemm_i4_fp16_push"), n.count("reduce_add_rmsnorm_fp16_i4"), n.count(T.ALL_REDUCE)) == \
            (pushes, pushes, 4 - pushes), b
    assert n.count("dense_layer_gemm_i4_qkv") == 2 and names[1].count("dense_layer_gemm_i4_o4") == 4
    assert h.ranks[0][0].inter_sizes == ([768, 640] if world == 2 else [384, 384, 384, 256])
    rk = h.ref.ranks[world - 1]
    assert all(rk.ends[rk._end(c.indicies, c.seqlen)][0] == c.seqlen for c in h.seqs[world - 1][:70])


@pytest.mark.parametrize("fault,world,batch,stage", [
    ("partial_missing", 2, 5, r"rank 0 layer 0 post_attention_layernorm \(\+ all-reduce of o_proj\): residual \+ all-reduce"),
    ("fp16_accumulation", 4, 5, r"rank 0 layer \d post_attention_layernorm \(\+ all-reduce of o_proj\): residual \+ all-reduce"),
    ("kv_into_other_rank", 2, 5, r"rank [01] layer 0 (batch_decode: attention output outside|pool audit)"),
    ("kv_into_other_layer", 2, 5, r"rank 1 layer 0 append_kv: layer_idx 1, the layer is 0"),
    ("other_rank_reorder", 2, 70, r"rank 1 layer 0 o_proj reorder: `reorder_index`"),
    ("pending_reduced_twice", 2, 5, r"rank 0 layer 1 qkv_proj: expected a call to dense_layer_gemm_i4_qkv, got reduce_add_rmsnorm"),
    ("kv_rows_one_head_short", 4, 5, r"rank 0 layer 0 qkv_proj: kv_rows 128 != 256"),
    ("replicated_norm_differs", 2, 5, r"rank 1 layer 1 post_attention_layernorm: replicated `weight` differs from rank 0's"),
])
def test_reference_rejects_a_seeded_fault(monkeypatch, fault, world, batch, stage):
    with pytest.raises(R.WiringError, match=stage):
        h = Harness(monkeypatch, world, _config(8, 8), fault)
        h.step(batch)


def test_allreduce_sum_strips_the_sentinel_and_sums_in_rank_order():
    a = np.array([-0.0, 1.0, 2048.0, -0.0], np.float16)
    b = np.array([-0.0, -0.0, 1.0, 3.0], np.float16)
    c = np.array([-0.0, 0.0, 1.0, -0.0], np.float16)
    s = T.allreduce_sum([a, b, c])
    assert s.view(np.uint16).tolist()[0] == 0 and s.tolist()[1:] == [1.0, 2050.0, 3.0]     # FP16 accumulation: 2048
    assert O is not None and T.torch_allreduce_sum([torch.from_numpy(x) for x in (a, b, c)]).numpy().view(np.uint16).tolist() == \
        s.view(np.uint16).tolist()
