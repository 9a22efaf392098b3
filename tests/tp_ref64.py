"""Reference of one decode step of a chain of TPLlamaDecoderLayers (atom_b200/tp.py) over `world` ranks: every kernel call of every
rank, checked against an independent recomputation.

TEST INFRASTRUCTURE ONLY.  Built on tests/layer_ref64.py: each rank is a layer_ref64.ModelRef of its own shards (RankRef) that walks
that rank's own trace with ModelRef's stages -- input norm -> q/k/v (one fused launch for M <= 64, else q_proj, k_proj and v_proj) ->
append_kv + decode attention over the rank's OWN history of K/V bytes -> reorder -> o_proj -> post-attention norm -> gate/up -> down
-- and the same checks (quantisers, GEMMs bit exact against the oracle at the dispatcher's K split and within gemm_ref64's float64
bounds, attention within attn_ref64's bound, the pool audit).  What it adds is the tensor-parallel wiring:

  * the row-parallel projections (o_proj, down_proj).  With a push-capable all-reduce (world > 1, fused, M <= 64, hidden % 1024 == 0,
    M * hidden within a slot) the GEMM is dense_layer_gemm_i4_fp16_push and the all-reduce is formed by the reduce_add_rmsnorm_fp16_i4
    launch that follows it: o_proj's by the post-attention norm, down_proj's by the NEXT layer's input norm (the last layer of a chain
    never pushes).  Otherwise the GEMM is dense_layer_gemm_i4_fp16, followed at world > 1 by the stand-alone all-reduce (recorded
    under the name ALL_REDUCE), and the sum goes to add_rmsnorm_fp16_i4, or is added to the residual by torch after down_proj;
  * at every all-reduce point the tensor the next stage consumes must be exactly allreduce_sum(partial_0, ..., partial_{W-1}): the
    FP32 sum in rank order of every rank's partial, FP16 -0.0 sent as +0.0, rounded to FP16.  partial_r is the oracle's o16 of rank
    r's recorded operands at the K split gemm_ref64.dispatch gives (the push GEMM follows the EPI_O16 rule) -- this also pins the
    push GEMM's output, which no rank ever sees on its own -- or, for a stand-alone all-reduce, the rank's own (checked) GEMM output;
  * every rank's residual stream and layer output are the same bytes, and the replicated parameters (both norms' weight, reorder
    index and eps) are the same on every rank.

The layer is decode-only: TPRef.seed takes the running sequences' history from the pools as they were before the first step (those
bytes are the step's input); afterwards the history grows only from the K/V each step's checks accepted.

The ranks are walked in lock-step: RankRef.walk is a generator that stops at each all-reduce point with its partial, and TPRef hands
every rank the sum of all of them.  Errors name the rank, the layer and the stage.
"""
import threading

import numpy as np

from oracle import oracle as O
from tests import gemm_ref64 as G
from tests import layer_ref64 as R

ALL_REDUCE = "all_reduce"                   # the stand-alone all-reduce, as a test records it: args {"x": partial}, out: the sum
TP_OPS = R.RECORDED_OPS + ("dense_layer_gemm_i4_fp16_push", "reduce_add_rmsnorm_fp16_i4")


def allreduce_sum(parts):
    """fp16(sum_r fp32(partial_r)), summed in rank order from +0, FP16 -0.0 (the receive buffers' sentinel) sent as +0.0."""
    acc = np.zeros(np.shape(parts[0]), np.float32)
    for p in parts:
        p = np.asarray(p, np.float16)
        acc += np.where(p.view(np.uint16) == 0x8000, np.float16(0), p).astype(np.float32)
    return acc.astype(np.float16)


class TPLayerParams:
    """What the reference knows of one rank's TPLlamaDecoderLayer: its shards and replicated parameters, as stored (the attribute
    names of layer_ref64.LayerParams).  The fused q/k/v and gate/up operands are the reference's own row concatenation."""

    def __init__(self, layer):
        host = R.host
        self.index, self.hidden = layer.layer_idx, layer.q_proj.in_features
        self.hq, self.hkv, self.theta = layer.local_heads, layer.local_kv_heads, layer.rope_theta
        self.ln1, self.ln2 = R.norm_params(layer.input_layernorm), R.norm_params(layer.post_attention_layernorm)
        self.attn_index = host(layer.attn_reorder_index)
        self.q, self.k, self.v = R.Lin.of(layer.q_proj), R.Lin.of(layer.k_proj), R.Lin.of(layer.v_proj)
        self.qkv = R.Lin.cat([self.q, self.k, self.v])
        self.o, self.down = R.Lin.of(layer.o_proj.local), R.Lin.of(layer.down_proj.local)
        self.gate, self.up = R.Lin.of(layer.gate_proj), R.Lin.of(layer.up_proj)
        self.gu = R.Lin.cat([self.gate, self.up])
        self.inter = layer.gate_proj.out_features
        self.moe = None


class RankRef(R.ModelRef):
    """The reference of one rank: its layers' shards on its own KV pool."""

    def __init__(self, layers, P, rank, tp, row_cap):
        super().__init__([TPLayerParams(l) for l in layers], P, row_cap=row_cap)
        self.rank, self.tp = rank, tp

    def _where(self, st):
        return f"rank {self.rank} {st}"

    def _row_parallel(self, st, lin, act, m, push):
        """A row-parallel projection of the quantised `act`.  Generator: yields (stage, rows, partial) at the all-reduce point and
        returns ("pending", rows, partial) for a push GEMM (its sum is formed by the next reduce_add_rmsnorm launch), else
        ("sum", None, the FP16 all-reduced output)."""
        ksplit = G.dispatch(m, lin.n, lin.k, R.GEMM_AUTO)[1]
        if push:
            c = self._next(st, ["dense_layer_gemm_i4_fp16_push"])
            self._gemm_call(st, c, act, lin, R.GEMM_AUTO)
            ar = c.args["ar"]
            if (ar.rank, ar.world) != (self.rank, self.tp.world):
                self._fail(st, f"pushes as rank {ar.rank} of {ar.world}")
            rows = self._rows(m, lin.n, lin.k)
            t = (act[1], lin.b, act[3], lin.bs, act[0], lin.bk, act[2], lin.bks)
            return "pending", rows, O.gemm_i4_o16(*t, rows=rows, ksplit=ksplit)
        c = self._next(st, ["dense_layer_gemm_i4_fp16"])
        self._gemm_call(st, c, act, lin, R.GEMM_AUTO)
        self._o16(st, act, lin, c.out, ksplit)
        if self.tp.world == 1:
            return "sum", None, c.out
        sta = f"{st} all-reduce"
        a = self._next(sta, [ALL_REDUCE])
        self._eq(sta, "x", a.args["x"], c.out)
        _, total = yield sta, None, c.out
        if not R.same(a.out, total):
            bad = np.argwhere(np.asarray(a.out).view(np.uint16) != total.view(np.uint16))
            self._fail(sta, f"the all-reduced tensor is not fp16(sum_r fp32(partial_r)) in rank order ({len(bad)} values, first at "
                            f"{bad[:1].tolist()})")
        return "sum", None, a.out

    def _reduce_norm(self, st, ln, residual, pend, m):
        """reduce_add_rmsnorm_fp16_i4 consuming the push GEMMs' partials: the residual plus the all-reduce, and its quantised norm.
        Generator (yields at the all-reduce point); returns the kernel's (residual sum, quantised norm)."""
        c = self._next(st, ["reduce_add_rmsnorm_fp16_i4"])
        self._eq(st, "residual", c.args["residual"], residual)
        if tuple(c.args["pending"].shape) != tuple(np.shape(residual)) or c.args["pending"].ar.rank != self.rank:
            self._fail(st, f"reduces a pending all-reduce of shape {c.args['pending'].shape} as rank {c.args['pending'].ar.rank}")
        self._norm_args(st, c, ln)
        rows, total = yield st, pend[1], pend[2]
        s, x = c.out
        sr = s if rows is None else s[rows]
        if not R.same(sr, R.fp16_sum(residual if rows is None else residual[rows], total)):
            bad = np.argwhere(sr.view(np.uint16) != R.fp16_sum(residual if rows is None else residual[rows], total).view(np.uint16))
            self._fail(st, f"residual + all-reduce is not the exact FP16 sum of the residual and fp16(sum_r fp32(partial_r)) "
                           f"({len(bad)} values, first at {bad[:1].tolist()})")
        w, idx, eps = ln
        self._quant(st, x, O.rmsnorm_fp16_i4(sr, w, idx, eps), m, rows=rows, exact=False)
        return s, x

    def walk(self, calls, step):
        """Walk this rank's trace of one decode step (generator, see TPRef.check_step).  Returns (residual sums, layer output)."""
        self._calls, self._pos, self._doff = calls, 0, 0
        m = int(step.decode)
        _, drows = self._admit(step)
        residual, pend, sums = step.x, None, []
        push = self.tp.can_push(m)
        for l, p in enumerate(self.layers):
            L = f"layer {l}"
            last = l == len(self.layers) - 1
            # ---- input norm: the previous layer's pending down projection is reduced into the residual here
            st = f"{L} input_layernorm"
            if pend is not None:
                residual, x = yield from self._reduce_norm(f"{st} (+ all-reduce of layer {l - 1} down_proj)", p.ln1, residual, pend, m)
            else:
                c = self._next(st, ["rmsnorm_fp16_i4"])
                self._eq(st, "hidden_states", c.args["hidden_states"], residual)
                self._norm_args(st, c, p.ln1)
                x = c.out
                self._quant(st, x, O.rmsnorm_fp16_i4(residual, *p.ln1), m, exact=False)
            sums.append(residual)
            # ---- attention
            q, k4, ks, v4, vs = self._qkv(L, p, x, m, fused=m <= 64)
            attn = self._decode(L, l, p, q, k4, ks, v4, vs, 0, m, drows, step.dtab)
            xo = self._reorder(L, p, attn, m)
            kind, rows, o = yield from self._row_parallel(f"{L} o_proj", p.o, xo, m, push)
            # ---- post-attention norm (+ o_proj's all-reduce)
            st = f"{L} post_attention_layernorm"
            if kind == "pending":
                residual, x = yield from self._reduce_norm(f"{st} (+ all-reduce of o_proj)", p.ln2, residual, (kind, rows, o), m)
            else:
                c = self._next(st, ["add_rmsnorm_fp16_i4"])
                self._eq(st, "hidden_states", c.args["hidden_states"], o)
                self._eq(st, "residual", c.args["residual"], residual)
                self._norm_args(st, c, p.ln2)
                s, x = c.out
                if not R.same(s, R.fp16_sum(residual, o)):
                    self._fail(st, "residual + attention is not the exact FP16 sum")
                residual = s
                self._quant(st, x, O.rmsnorm_fp16_i4(s, *p.ln2), m, exact=False)
            sums.append(residual)
            # ---- MLP
            xa = self._gateup(L, p, x, m)
            kind, rows, d = yield from self._row_parallel(f"{L} down_proj", p.down, xa, m, push and not last)
            if kind == "pending":
                pend = (kind, rows, d)
            else:
                pend, residual = None, R.fp16_sum(residual, d)       # torch's `hidden_states + down_proj(act)`: the next layer's input
        if self._pos != len(calls):
            self._fail("end of step", f"{len(calls) - self._pos} kernel calls more than the step needs ({calls[self._pos].name} first)")
        if pend is not None:
            self._fail("end of step", "the last layer left its down projection pending")
        if step.out is not None and not R.same(step.out, residual):
            self._fail(f"layer {len(self.layers) - 1} output", "residual + down_proj is not the exact FP16 sum")
        return sums, residual

    def settle(self, before=None, after=None):
        """After the step: the pool audit (before / after: this rank's pool) and the sequences' new ends."""
        if after is not None:
            self._audit(before, after)
        self._settle()


def seed_history(ref, dtab, pool):
    """Give the ModelRef `ref` the sequences of the decode page table `dtab` that it does not know yet (each one position longer
    than before the step) and their history, in every layer, from `pool` = (data, param) as it was before that step.
    TPRef.check_step does this with its `before` pools: a sequence's history is read from the pool once, before its first step."""
    data, param = pool
    L = len(ref.layers)
    for pages, n in R.sequences(dtab, ref.P):
        n0 = n - 1
        ref._ensure(pages)
        if n0 == 0 or ref.ends.get(ref._end(pages, n0), [None])[0] == n0:
            continue
        pg, e = ref._slots(pages, np.arange(n0))
        ref.sd[pg, :, :, :, e], ref.sp[pg, :, :, :, e] = data[pg, :L, :, :, e], param[pg, :L, :, :, e]
        ref.known[pg, :, e] = True
        ref._register(pages, n0)


class TPRef:
    """The reference of a chain of TPLlamaDecoderLayers: ranks[r] is rank r's list of layers (layer_idx 0, 1, ... of its pool).
    fuse / slot: the all-reduce object's `fuse` flag and slot size, which decide where the layer pushes."""

    def __init__(self, ranks, P, fuse=True, slot=0, row_cap=1 << 27):
        self.world, self.fuse, self.slot = len(ranks), fuse, slot
        self.ranks = [RankRef(layers, P, r, self, row_cap) for r, layers in enumerate(ranks)]
        self.hidden = self.ranks[0].layers[0].hidden
        self._replicated()

    def can_push(self, m):
        """The fused push all-reduce runs (RowParallelLinearInt4.can_push, restated)."""
        return self.world > 1 and self.fuse and m <= 64 and self.hidden % 1024 == 0 and m * self.hidden <= self.slot

    def _replicated(self):
        r0 = self.ranks[0]
        for rk in self.ranks[1:]:
            for l, (p, p0) in enumerate(zip(rk.layers, r0.layers)):
                for name, ln, ln0 in (("input_layernorm", p.ln1, p0.ln1), ("post_attention_layernorm", p.ln2, p0.ln2)):
                    for what, a, b in zip(("weight", "reorder_index", "eps"), ln, ln0):
                        if not (R.same(a, b) if what != "eps" else a == b):
                            rk._fail(f"layer {l} {name}", f"replicated `{what}` differs from rank 0's")

    def seed(self, dtab, pools):
        """seed_history of every rank from its pool `pools[r]` = (data, param) as it was before the step of page table `dtab`."""
        for rk, pool in zip(self.ranks, pools):
            seed_history(rk, dtab, pool)

    def check_step(self, traces, x, dtab, outs, before=None, after=None):
        """Check one decode step: traces[r] is rank r's recorded calls, x the hidden states every rank was given, dtab the page
        table, outs[r] what rank r's chain returned, before / after[r] rank r's pool (data, param).  Raises layer_ref64.WiringError
        naming the rank, the layer and the stage of the first difference."""
        nd = len(dtab["indptr"]) - 1
        if before is not None:
            self.seed(dtab, before)
        gens = []
        for rk, calls, out in zip(self.ranks, traces, outs):
            gens.append(rk.walk(calls, R.Step([], nd, dtab=dtab, x=np.asarray(x), out=out)))
        results = [None] * self.world
        msgs = [self._advance(g, None, r, results) for r, g in enumerate(gens)]
        while any(msg is not None for msg in msgs):
            at = [msg[0] if msg else "end of step" for msg in msgs]
            for r in range(1, self.world):
                if at[r] != at[0]:
                    self.ranks[r]._fail(at[r], f"rank 0 is at `{at[0]}`: the ranks' traces diverge")
            rows = next((msg[1] for msg in msgs if msg[1] is not None), None)
            parts = []
            for r, (st, rr, part) in enumerate(msgs):
                if rr is not None and list(rr) != list(rows):
                    self.ranks[r]._fail(st, "rows of the partial differ from rank 0's")
                parts.append(part if rr is not None or rows is None else part[rows])
            total = allreduce_sum(parts)
            msgs = [self._advance(g, (rows, total), r, results) for r, g in enumerate(gens)]
        sums0, out0 = results[0]
        for r, (sums, out) in enumerate(results[1:], 1):
            for i, (s, s0) in enumerate(zip(sums, sums0)):
                if not R.same(s, s0):
                    stage = "input_layernorm" if i % 2 == 0 else "post_attention_layernorm"
                    self.ranks[r]._fail(f"layer {i // 2} {stage}", "the residual stream differs from rank 0's")
            if not R.same(out, out0):
                self.ranks[r]._fail(f"layer {len(self.ranks[r].layers) - 1} output", "the layer output differs from rank 0's")
        for r, rk in enumerate(self.ranks):
            rk.settle(None if before is None else before[r], None if after is None else after[r])

    @staticmethod
    def _advance(g, value, r, results):
        try:
            return g.send(value)
        except StopIteration as e:
            results[r] = e.value
            return None


# ------------------------------------------------------------------------------------------------------------------ emulated ranks
class TPRecorder(R.Recorder):
    """layer_ref64.Recorder of the TP ops whose calls go to the trace of the calling thread's rank (bind(rank) in each thread)."""

    def __init__(self, world, impl=None):
        super().__init__(impl, TP_OPS)
        self.traces = [[] for _ in range(world)]
        self._local = threading.local()

    def bind(self, rank):
        self._local.rank = rank

    def _log(self, call):
        self.traces[self._local.rank].append(call)

    def wrap(self, name, fn):
        """fn, recorded under `name`."""
        return self._wrap(name, fn)


class Rendezvous:
    """A host barrier of the ranks' threads (with a timeout; abort() releases everybody on an error) that can exchange one value
    per rank."""

    def __init__(self, world, timeout=120.0):
        self.barrier = threading.Barrier(world, timeout=timeout)
        self.slots = [None] * world

    def wait(self):
        self.barrier.wait()

    def exchange(self, rank, value):
        self.slots[rank] = value
        self.barrier.wait()
        got = list(self.slots)
        self.barrier.wait()              # nobody refills a slot before every rank has read them all
        return got

    def abort(self):
        self.barrier.abort()


def torch_allreduce_sum(parts):
    """allreduce_sum in torch, on the tensors' device: FP32 sum in rank order from +0, FP16 -0.0 sent as +0.0."""
    import torch
    acc = torch.zeros(parts[0].shape, dtype=torch.float32, device=parts[0].device)
    for p in parts:
        acc += p.masked_fill(p.view(torch.int16) == -32768, 0).float()
    return acc.half()


class EmulatedAllReduce:
    """The all-reduce object of one emulated rank, with the interface tp.py uses of comm.PushAllReduce: `handle` (an ops.ArHandle,
    or None), `fuse`, `slot`, `name`, and a stand-alone all-reduce: the ranks meet at the rendezvous and each forms the rank-order
    FP32 sum in torch.  The call is recorded under ALL_REDUCE."""
    name = "emulated ranks: rank-order FP32 sum in torch"

    def __init__(self, rank, rdv, rec, handle=None, slot=0, fuse=True):
        self.rank, self.rdv, self.handle, self.slot, self.fuse = rank, rdv, handle, slot, fuse
        self._call = rec.wrap(ALL_REDUCE, self.reduce)

    def __call__(self, x):
        return self._call(x)

    def reduce(self, x):
        return torch_allreduce_sum(self.rdv.exchange(self.rank, x))


def run_ranks(world, fn, rec, rdv, stream=None):
    """fn(rank) in one thread per rank (under inference_mode, on `stream` when given); returns the results in rank order.  An
    exception in any rank aborts the rendezvous and is raised here (the first one that is not the barrier's own)."""
    import torch
    out, errs = [None] * world, [None] * world

    def body(r):
        rec.bind(r)
        try:
            with torch.inference_mode():
                if stream is None:
                    out[r] = fn(r)
                else:
                    with torch.cuda.stream(stream):
                        out[r] = fn(r)
        except BaseException as e:  # noqa: BLE001
            errs[r] = e
            rdv.abort()

    threads = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    real = [e for e in errs if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    if real or any(errs):
        raise (real or [e for e in errs if e is not None])[0]
    return out


def make_ranks(cfg, world, layers, dev, allreduces, seed=0):
    """TPLlamaDecoderLayers (layer_idx 0..layers-1) of every rank.  Replicated parameters (norm weights and reorder indices) come
    from one generator and are the same on every rank; the shards (INT4 projections, attn_reorder_index) are the rank's own.  The
    fused q/k/v and gate/up operands are built last."""
    import torch
    from atom_b200.tp import TPLlamaDecoderLayer
    ranks = []
    for r in range(world):
        g = torch.Generator().manual_seed(seed)
        mine = torch.Generator().manual_seed(seed * 1000 + 17 * r + 1)
        chain = []
        for i in range(layers):
            layer = TPLlamaDecoderLayer(cfg, i, r, world, allreduce=allreduces[r]).to(dev).init_random(seed * 8 + i)
            with torch.no_grad():
                for n in (layer.input_layernorm, layer.post_attention_layernorm):
                    n.weight.copy_(torch.rand(n.weight.shape, generator=g).half() + 0.5)
                    n.reorder_index.copy_(torch.randperm(n.reorder_index.numel(), generator=g).to(torch.int16))
                layer.attn_reorder_index.copy_(torch.randperm(layer.attn_reorder_index.numel(), generator=mine).to(torch.int16))
            chain.append(layer.fuse().eval())
        ranks.append(chain)
    return ranks


def chain_step(layers, x, kv):
    """One decode step of a chain: forward_chain through every layer, `last` on the final one."""
    h, pend = x, None
    for i, layer in enumerate(layers):
        h, pend = layer.forward_chain(h, pend, kv, last=i == len(layers) - 1)
    return h
