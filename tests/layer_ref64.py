"""Reference of whole model steps: every tensor a Llama decoder-layer step stores, checked against an independent recomputation.

TEST INFRASTRUCTURE ONLY.  Plain numpy on the oracle (oracle/atom_oracle.c), gemm_ref64 and attn_ref64.

How a step is checked.  The layers call the kernels as `ops.<name>(...)`; a Recorder replaces those attributes with wrappers that
keep a host copy of every argument and output, in call order.  ModelRef.check_step then walks that trace with its own model of the
step:
  * the call at each point must be the one the step's shape implies: rmsnorm / add_rmsnorm -> qkv -> init_kv + prefill attention
    (prompts) -> append_kv + decode attention (running sequences) -> reorder -> o_proj -> add_rmsnorm -> gate/up (one fused launch
    for M <= 64, else two GEMMs + activate) -> down, per layer; for a MixtralDecoderLayer the MLP is route -> plan -> gather ->
    grouped gate/up -> grouped down -> combine;
  * its inputs must be, bit for bit, the tensors the reference says that stage consumes (the previous stage's output, the layer's
    parameters, the step's page tables, the layer's own index);
  * its output must match the reference's own result for those inputs: quantisers bit exact (rmsnorm: +-1 code, 2e-3 on the scale,
    the kernel's rsqrtf is approximate; activate: +-1 code, expf), residual sums exact, GEMMs bit exact against the oracle at the
    K split the dispatcher picks for the call's M (and FP16 GEMMs and the INT4 K/V quantiser within gemm_ref64's float64
    bounds), attention within the float64 bound of its kind (attn_ref64: prompts, decode; attn_ctx_ref64: prompts over a
    cached prefix; attn_verify_ref64: verify steps; attn_cascade_ref64: the shared-prefix cascade) on the reference's OWN
    shadow of the pool (it never reads the pool to compute attention).
Quantisation is discontinuous, so after checking a stage the reference continues from the kernel's value ("borrows" it): a rounding
flip upstream cannot spread, and a wiring fault shows at the stage where it happens, named in the error.
The shadow is what the reference says each physical slot holds: (page, layer, K|V, entry) -> the K/V codes and (scale, zero),
written by the stages it checked and by the fork hook (ModelRef.fork: a fork copies its partly filled page outside the recorded
operators).  Pages shared by forks carry one history.  Sequences are known by where their history ends: the (page, entry) of a
sequence's last cached token, its length and its pages.  A row of a step must continue a history the reference knows, at the
length it expects -- after a verify step that is the length the kept tokens leave (ModelRef.keep, or check_spec from the emitted
tokens) -- and may write only into pages no other holder has.
Before the step, every history slot the step reads must hold the shadow's bytes; after it, the pool is audited: the slots the
step wrote, in every layer, hold the shadow's bytes, and every other byte (slots past a sequence's length included) is what it
was before the step.
"""
import inspect
from collections import Counter
from dataclasses import dataclass, field

import numpy as np

from oracle import oracle as O
from tests import attn_ref64 as A
from tests import attn_verify_ref64 as VR
from tests import gemm_ref64 as G
from tests.attn_cascade_ref64 import cascade_bound
from tests.attn_ctx_ref64 import prefill_ctx_bound
from tests import moe_ref as ME

U16 = 2.0 ** -11
U32 = 2.0 ** -24
GEMM_AUTO = 0

GEMM_ARGS = {      # the operand names of each GEMM entry point: a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale
    "dense_layer_gemm_i4_fp16": ("a", "b", "a_scale", "b_scale", "a_keeper", "b_keeper", "a_keeper_scale", "b_keeper_scale"),
    "dense_layer_gemm_i4_o4": ("a", "b", "a_scale", "b_scale", "a_keeper", "b_keeper", "a_keeper_scale", "b_keeper_scale"),
    "dense_layer_gemm_i4_fp16_push": ("a", "b", "a_scale", "b_scale", "a_keeper", "b_keeper", "a_keeper_scale", "b_keeper_scale"),
    "dense_layer_gemm_i4_qkv": ("a", "b_qkv", "a_scale", "b_scale_qkv", "a_keeper", "b_keeper_qkv", "a_keeper_scale", "b_keeper_scale_qkv"),
    "dense_layer_gemm_i4_gateup_act": ("a", "b_gu", "a_scale", "b_scale_gu", "a_keeper", "b_keeper_gu", "a_keeper_scale",
                                       "b_keeper_scale_gu"),
}
RECORDED_OPS = ("rmsnorm_fp16_i4", "add_rmsnorm_fp16_i4", "dense_layer_gemm_i4_qkv", "init_kv_i4", "prefill_attention_i4",
                "append_kv_i4", "batch_decode_i4", "batch_verify_i4", "reorder_fp16_i4", "dense_layer_gemm_i4_fp16", "dense_layer_gemm_i4_o4",
                "dense_layer_gemm_i4_gateup_act", "activate_fp16_i4", "moe_route_f16", "moe_plan", "moe_gather_i4",
                "dense_layer_gemm_i4_gateup_act_grouped", "dense_layer_gemm_i4_fp16_grouped", "moe_combine_f16")


class WiringError(AssertionError):
    """A step's trace differs from the reference; the message names the layer and the stage."""


def host(x):
    """Host copy of an argument or result: tensors -> numpy, page tables -> dict of numpy, tuples element-wise."""
    if hasattr(x, "detach"):
        return x.detach().cpu().numpy().copy()
    if hasattr(x, "indptr") and hasattr(x, "last_page_offset"):
        tab = {"indptr": host(x.indptr), "indices": host(x.indicies), "last": host(x.last_page_offset)}
        if getattr(x, "shared_pages", None) is not None:          # prefix groups (forked rows) and their shared page counts
            tab.update(shared=host(x.shared_pages), groups=[(list(r), int(n)) for r, n in x.groups])
        return tab
    if isinstance(x, (tuple, list)) and any(hasattr(t, "detach") for t in x):
        return tuple(host(t) for t in x)
    return x


def same(a, b):
    """Same bytes (views of one buffer may differ in shape: [T, H*64] against [T, H, 64])."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.nbytes == b.nbytes and np.array_equal(a.reshape(-1).view(np.uint8), b.reshape(-1).view(np.uint8))


def fp16_sum(a, b):
    """FP16 a + b, rounded once (the float64 sum of two halves is exact)."""
    return (np.asarray(a, np.float64) + np.asarray(b, np.float64)).astype(np.float16)


@dataclass
class Call:
    name: str
    args: dict
    out: object


class Recorder:
    """Replaces the recorded `atom_b200.ops` functions (install(monkeypatch)) by wrappers that append a Call per invocation to
    `calls`.  `impl` maps a name to the function that does the work (default: the real operator); `names`: the recorded ops."""

    def __init__(self, impl=None, names=RECORDED_OPS):
        from atom_b200 import ops
        self.ops, self.calls = ops, []
        self.impl = {n: (impl or {}).get(n, getattr(ops, n)) for n in names}

    def install(self, monkeypatch):
        for name, fn in self.impl.items():
            monkeypatch.setattr(self.ops, name, self._wrap(name, fn))
        return self

    def _wrap(self, name, fn):
        sig = inspect.signature(fn)

        def rec(*args, **kwargs):
            b = sig.bind(*args, **kwargs)
            b.apply_defaults()
            out = fn(*args, **kwargs)
            self._log(Call(name, {k: host(v) for k, v in b.arguments.items()}, host(out)))
            return out
        return rec

    def _log(self, call):
        self.calls.append(call)


# ------------------------------------------------------------------------------------------------------------------ parameters
class Lin:
    """One INT4 projection: the tensors the layer passes (`raw`, in the order of the GEMM's b, b_scale, b_keeper, b_keeper_scale)
    and the oracle's operands (weight scales at pitch N)."""

    def __init__(self, w4, s4, w8, s8, n, k):
        self.raw = (w4, s4, w8, s8)
        g = k // 128 - 1
        self.n, self.k = n, k
        self.b, self.bk = w4, w8
        self.bs = np.ascontiguousarray(s4.reshape(-1)[:g * n].reshape(g, n))
        self.bks = np.ascontiguousarray(s8.reshape(-1)[:n])

    @classmethod
    def of(cls, lin):
        return cls(host(lin.weight_int4), host(lin.scale_int4), host(lin.weight_int8), host(lin.scale_int8), lin.out_features,
                   lin.in_features)

    @classmethod
    def cat(cls, lins):
        """The row concatenation of projections that share their input, as one launch takes it (weight scales at pitch sum N)."""
        return cls(np.concatenate([l.b for l in lins]), np.concatenate([l.bs for l in lins], 1), np.concatenate([l.bk for l in lins]),
                   np.concatenate([l.bks for l in lins]), sum(l.n for l in lins), lins[0].k)

    def rows(self, a, b):
        """The rows [a, b) of a row-concatenated projection (fused q/k/v, gate/up)."""
        return Lin(self.b[a:b], np.ascontiguousarray(self.bs[:, a:b]), self.bk[a:b], self.bks[a:b], b - a, self.k)


class MoeParams:
    """The sparse MoE block of a MixtralDecoderLayer: router [E, H] and the stacked expert operands, as stored."""

    def __init__(self, moe):
        self.e, self.k, self.inter = moe.num_experts, moe.top_k, moe.intermediate_size
        self.router = host(moe.router_weight)
        self.w13 = tuple(host(t) for t in (moe.w13_int4, moe.w13_scale, moe.w13_int8, moe.w13_keeper_scale))
        self.w2 = tuple(host(t) for t in (moe.w2_int4, moe.w2_scale, moe.w2_int8, moe.w2_keeper_scale))


def norm_params(norm):
    """(weight, reorder_index, eps) of a LlamaRMSNormInt4, as stored."""
    return host(norm.weight), host(norm.reorder_index), norm.variance_epsilon


class LayerParams:
    """What the reference knows of one LlamaDecoderLayer or MixtralDecoderLayer: its parameters, as stored.  The operands of the
    fused q/k/v and gate/up launches are the reference's own concatenation of q_proj / k_proj / v_proj and gate_proj / up_proj."""

    def __init__(self, layer, index):
        a = layer.self_attn
        self.index, self.hidden = index, a.hidden_size
        self.hq, self.hkv, self.theta = a.num_heads, a.num_kv_heads, a.rope_theta
        self.ln1, self.ln2 = norm_params(layer.input_layernorm), norm_params(layer.post_attention_layernorm)
        self.attn_index = host(a.reorder_index)
        self.qkv = Lin.cat([Lin.of(a.q_proj), Lin.of(a.k_proj), Lin.of(a.v_proj)])
        self.o = Lin.of(a.o_proj)
        self.moe = MoeParams(layer.block_sparse_moe) if hasattr(layer, "block_sparse_moe") else None
        if self.moe is None:
            mlp = layer.mlp
            self.gate, self.up, self.down = Lin.of(mlp.gate_proj), Lin.of(mlp.up_proj), Lin.of(mlp.down_proj)
            self.gu = Lin.cat([self.gate, self.up])
            self.inter = mlp.intermediate_size


# ------------------------------------------------------------------------------------------------------------------ helpers
def quant_rows(t, m):
    """Activation 4-tuple (o8, o4, s8, s4) of m rows -> (codes int [m, H] in the quantiser's order, keeper last; scales f16 [groups, m])."""
    o8, o4, s8, s4 = t
    codes = np.concatenate([O.unpack_int4(np.asarray(o4).view(np.uint8)), np.asarray(o8).view(np.int8)], 1).astype(np.int32)
    scales = np.concatenate([O.a_scale_from_layout(np.asarray(s4).view(np.float16), m),
                             O.a_scale_from_layout(np.asarray(s8).view(np.float16), m)[None]], 0)
    return codes, scales


def table_of(pages_per_seq, lens, P):
    indptr = np.concatenate([[0], np.cumsum([len(p) for p in pages_per_seq])]).astype(np.int32)
    indices = np.array([x for p in pages_per_seq for x in p], np.int32)
    return {"indptr": indptr, "indices": indices, "last": np.array([(n - 1) % P + 1 for n in lens], np.int32)}


def sequences(tab, P):
    """[(pages, length)] of a page table."""
    ip = tab["indptr"]
    return [(tab["indices"][ip[i]:ip[i + 1]].tolist(), (ip[i + 1] - ip[i] - 1) * P + int(tab["last"][i])) for i in range(len(ip) - 1)]


@dataclass
class Step:
    """One model step as the caller ran it.  x: the FP16 hidden states entering layer 0 (or None: embedding of ids); tables: the
    page tables the model was given (host(BatchedKvCacheInt4) or None); out: what the model returned (host copies)."""
    prefills: list
    decode: int
    ptab: dict = None
    dtab: dict = None
    ids: np.ndarray = None
    x: np.ndarray = None
    out: tuple = None
    rows: list = None                      # the rows whose logits the caller reads (serving loop), None = not checked
    decode_len: int = 1                    # S: rows of each running sequence (S > 1: a verify step)
    refs: list = None                      # holders of every pool page before the step (None: not known)
    info: dict = field(default_factory=dict)


class ModelRef:
    """The reference of a stack of LlamaDecoderLayers (or MixtralDecoderLayers) on one KV pool (page size P), optionally with the embedding, the final
    LlamaRMSNorm and lm_head of LlamaForCausalLM (numpy copies: embed [V, H], norm (w, eps), lm_head [V, H]).  sm_count: the SMs
    of the device the steps run on, for ops.decode_cascade's choice (None: the plain decode kernel is expected)."""

    def __init__(self, layers, P, embed=None, norm=None, lm_head=None, row_cap=1 << 27, prefill_rows=None, sm_count=None):
        self.layers, self.P = layers, P
        self.embed, self.norm, self.lm_head = embed, norm, lm_head
        self.row_cap = row_cap              # an oracle GEMM above this many multiply-adds is checked on a row subset
        self.prefill_rows = prefill_rows    # rows of each prompt where attn_ref64 evaluates the exact spread term (None: all)
        self.sm_count = sm_count
        self.sd = self.sp = self.known = None   # shadow: K/V codes [pages, L, 2, Hkv, P, 64], (s, z) [.., 2], written [pages, L, P]
        self.ends = {}                      # (page, entry) of a sequence's last cached token -> [length, its pages, holders]
        self.worst = {}                     # attention kind -> largest |kernel - float64| / bound seen
        self.calls = Counter()              # attention kind -> checked calls
        self._rows_step, self._S = [], 1

    # ---------------------------------------------------------------------------------------------------------- checks
    def _where(self, st):
        """The stage as errors name it."""
        return st

    def _fail(self, st, msg):
        raise WiringError(f"{self._where(st)}: {msg}")

    def _eq(self, st, what, got, want):
        if not same(got, want):
            self._fail(st, f"`{what}` is not the tensor this stage consumes")

    def _next(self, st, names):
        if self._pos >= len(self._calls):
            self._fail(st, f"expected a call to {' or '.join(names)}, the step made no more kernel calls")
        c = self._calls[self._pos]
        if c.name not in names:
            self._fail(st, f"expected a call to {' or '.join(names)}, got {c.name}")
        self._pos += 1
        return c

    def _rows(self, m, n, k):
        if m * n * k <= self.row_cap:
            return None
        r = {0, 1, 7, 8, 9, 15, 16, 17, m - 2, m - 1, self._doff - 1, self._doff, self._doff + 1}
        r |= set(np.random.default_rng(m).integers(0, m, 8).tolist())
        return sorted(x for x in r if 0 <= x < m)

    def _quant(self, st, got, ref, m, rows=None, exact=True):
        gc, gs = quant_rows(got, m)
        rc, rs = quant_rows(ref, len(rows) if rows is not None else m)
        if rows is not None:
            gc, gs = gc[rows], gs[:, rows]
        if exact:
            if not (np.array_equal(gc, rc) and np.array_equal(gs.view(np.uint16), rs.view(np.uint16))):
                bad = np.argwhere(gc != rc)
                self._fail(st, f"quantised tuple differs from the oracle ({len(bad)} codes, first at {bad[:1].tolist()})")
        else:
            dc = np.abs(gc - rc)
            if dc.max() > 1 or (dc != 0).mean() > 5e-3:
                self._fail(st, f"codes differ from the oracle by up to {dc.max()} ({(dc != 0).sum()} codes)")
            g64, r64 = gs.astype(np.float64), rs.astype(np.float64)
            if not (np.abs(g64 - r64) <= 2e-3 * np.abs(r64)).all():
                self._fail(st, "scales differ from the oracle by more than 2e-3")
        o8, o4, s8, s4 = got                                                 # all four replicas of each scale written
        idx = np.array([O.scale_index(r) for r in (range(m) if rows is None else rows)])
        for j in range(1, 4):
            if not (same(np.asarray(s8)[idx + 2 * j], np.asarray(s8)[idx]) and same(np.asarray(s4)[:, idx + 2 * j], np.asarray(s4)[:, idx])):
                self._fail(st, "scale replicas differ")
    def _gemm_call(self, st, c, act, lin, flags=None):
        want = (act[1], lin.raw[0], act[3], lin.raw[1], act[0], lin.raw[2], act[2], lin.raw[3])
        for name, w in zip(GEMM_ARGS[c.name], want):
            self._eq(st, name, c.args[name], w)
        if flags is not None and c.args.get("flags") != flags:
            self._fail(st, f"GEMM flags {c.args.get('flags')}, expected {flags}")

    def _o16(self, st, act, lin, out, ksplit):
        m = act[0].shape[0]
        rows = self._rows(m, lin.n, lin.k)
        t = (act[1], lin.b, act[3], lin.bs, act[0], lin.bk, act[2], lin.bks)
        ref = O.gemm_i4_o16(*t, rows=rows, ksplit=ksplit)
        got = out if rows is None else out[rows]
        if not same(got, ref):
            bad = np.argwhere(got.view(np.uint16) != ref.view(np.uint16))
            self._fail(st, f"FP16 GEMM differs from the oracle at K split {ksplit} ({len(bad)} values, first at {bad[:1].tolist()})")
        S, T = G.ref64(*t, rows=rows)
        try:
            G.check_o16(got, S, T, lin.k // 128 - 1, ksplit, what=self._where(st))
        except AssertionError as e:
            raise WiringError(str(e)) from None

    def _o4(self, st, act, lin, out, rows):
        t = (act[1], lin.b, act[3], lin.bs, act[0], lin.bk, act[2], lin.bks)
        d, ds = O.gemm_i4_o4(*t, rows=rows)
        gd, gds = (out[0], out[1]) if rows is None else (out[0][rows], out[1][rows])
        if not (same(gd, d) and same(gds, ds)):
            self._fail(st, "INT4 GEMM output (codes or (scale, zero)) differs from the oracle")
        S, T = G.ref64(*t, rows=rows)
        try:
            G.check_o4(gd, gds, S, T, lin.k // 128 - 1, what=self._where(st))
        except AssertionError as e:                                  # names the stage, (row, head) and element
            raise WiringError(str(e)) from None

    def _attn_bound(self, st, got, ref, bnd, kind="attention"):
        ratio = np.abs(np.asarray(got, np.float64).reshape(ref.shape) - ref) / bnd
        w = np.unravel_index(np.argmax(np.nan_to_num(ratio, nan=np.inf)), ratio.shape)
        self.worst[kind] = max(self.worst.get(kind, 0.0), float(ratio[w]))
        self.calls[kind] += 1
        if not (ratio <= 1).all():
            self._fail(st, f"attention output outside the float64 bound (x{ratio[w]:.3g} at {tuple(int(i) for i in w)})")

    def _table(self, st, got, want):
        for k in ("indptr", "indices", "last"):
            if not same(np.asarray(got[k], np.int32), np.asarray(want[k], np.int32)):
                self._fail(st, f"page table `{k}` {np.asarray(got[k]).tolist()} is not the step's {np.asarray(want[k]).tolist()}")

    # ---------------------------------------------------------------------------------------------------------- shadow
    def _ensure(self, pages):
        """Grow the shadow to hold `pages`."""
        n = max(pages, default=-1) + 1
        if self.sd is None:
            L, hkv = len(self.layers), self.layers[0].hkv
            self.sd = np.zeros((0, L, 2, hkv, self.P, 64), np.uint8)
            self.sp = np.zeros((0, L, 2, hkv, self.P, 2), np.float16)
            self.known = np.zeros((0, L, self.P), bool)
        if n > len(self.sd):
            more = n - len(self.sd) + 8
            self.sd = np.concatenate([self.sd, np.zeros((more,) + self.sd.shape[1:], np.uint8)])
            self.sp = np.concatenate([self.sp, np.zeros((more,) + self.sp.shape[1:], np.float16)])
            self.known = np.concatenate([self.known, np.zeros((more,) + self.known.shape[1:], bool)])

    def _slots(self, pages, pos):
        """(page, entry) index arrays of the positions `pos` of a sequence on `pages`."""
        pos = np.asarray(pos)
        return np.asarray(pages, np.int64)[pos // self.P], pos % self.P

    def _write(self, l, pages, pos, k4, ks, v4, vs, hkv):
        """The shadow takes what a checked cache write of layer l stores at positions `pos` (rows of k4 / ks / v4 / vs)."""
        pg, e = self._slots(pages, pos)
        self.sd[pg, l, 0, :, e], self.sp[pg, l, 0, :, e] = k4.reshape(-1, hkv, 64), ks.reshape(-1, hkv, 2)
        self.sd[pg, l, 1, :, e], self.sp[pg, l, 1, :, e] = v4.reshape(-1, hkv, 64), vs.reshape(-1, hkv, 2)
        self.known[pg, l, e] = True
        if l == 0:
            self._written.append((pg, e))

    def _end(self, pages, n):
        """The key of a sequence of n tokens on `pages`: the (page, entry) of its last token."""
        return int(pages[(n - 1) // self.P]), (n - 1) % self.P

    def _register(self, pages, n, holders=1):
        key = self._end(pages, n)
        e = self.ends.get(key)
        if e is not None and e[0] == n and e[1] == tuple(pages[:-(-n // self.P)]):
            e[2] += holders
        else:
            self.ends[key] = [n, tuple(int(x) for x in pages[:-(-n // self.P)]), holders]

    def fork(self, parent_pages, n, child_pages):
        """A fork (KvCacheInt4.fork) of the first n tokens of the sequence on `parent_pages` onto `child_pages`: the child shares
        the parent's full pages among them and holds a copy of the partly filled one, if any, in a page of its own."""
        P, full = self.P, n // self.P
        parent_pages, child_pages = [int(x) for x in parent_pages], [int(x) for x in child_pages]
        self._ensure(parent_pages + child_pages)
        if child_pages[:full] != parent_pages[:full] or len(child_pages) != -(-n // P):
            self._fail("fork", f"the child's pages {child_pages} are not the parent's full pages {parent_pages[:full]} + one copy")
        t = np.arange(n)
        pg, e = self._slots(parent_pages, t)
        if not self.known[pg, :, e].all():
            self._fail("fork", f"the parent's first {n} tokens are not all a history the reference saw written")
        if n % P:
            src, dst = parent_pages[full], child_pages[full]
            if dst in parent_pages:
                self._fail("fork", f"the partly filled page {src} is shared with the child (page {dst}), not copied")
            self.sd[dst], self.sp[dst] = self.sd[src], self.sp[src]
            self.known[dst] = False
            self.known[dst, :, :n % P] = self.known[src, :, :n % P]
        if n:
            self._register(child_pages, n)

    def keep(self, kept):
        """After a verify step: running sequence j keeps kept[j] of its S rows (KvCacheInt4.truncate to its length - S + kept[j]);
        the next step must continue it at that length."""
        for (pages, n, _, _), c in zip([r for r in self._rows_step if r[3]], kept):
            if not 1 <= int(c) <= self._S:
                raise ValueError(f"kept {c} outside [1, {self._S}]")
            key = self._end(pages, n)
            e = self.ends.get(key)
            if e is not None and e[0] == n:
                del self.ends[key]
            self._register(pages, n - self._S + int(c))

    # ---------------------------------------------------------------------------------------------------------- page tables
    def _admit(self, step):
        """Check the step's page tables against the sequences the reference knows: every row continues a history that ends
        where it says, at the length the reference expects (prompts: none, or the earlier chunks / the forked prefix of their
        sequence; running sequences: what their last step kept), and writes its new positions into pages it alone holds.
        Returns the rows of the prompts and of the running sequences, in batch order: (pages, length, new tokens, running)."""
        P, S = self.P, int(step.decode_len)
        self._written, self._S = [], S
        prows = [(p, n, k, False) for (p, n), k in zip(sequences(step.ptab, P), step.prefills)] if step.prefills else []
        if step.prefills and len(prows) != len(step.prefills):
            self._fail("page table", f"{len(prows)} prompt rows for {len(step.prefills)} prompts")
        drows = [(p, n, S, True) for p, n in sequences(step.dtab, P)] if step.decode else []
        if step.decode and len(drows) != step.decode:
            self._fail("page table", f"{len(drows)} decode rows for {step.decode} running sequences")
        rows = prows + drows
        self._ensure([x for r in rows for x in r[0]])
        held = Counter(x for r in rows for x in set(r[0]))
        for i, (pages, n, k, running) in enumerate(rows):
            what = f"decode row {i - len(prows)}" if running else f"prompt {i}"
            h = n - k
            if h < 0 or (running and h == 0):
                self._fail("page table", f"{what} holds {n} positions for {k} new tokens" + (" and no history" if h == 0 else ""))
            if h:
                key = self._end(pages, h)
                e = self.ends.get(key)
                if e is None or e[0] != h or e[1] != tuple(pages[:-(-h // P)]):
                    self._fail("page table", f"{what}: {n} positions on pages {pages} continue a history of {h} tokens that no "
                                             f"sequence the reference knows ends with" +
                                             (f" (the one ending there holds {e[0]} on {list(e[1])})" if e else ""))
                e[2] -= 1
                if not e[2]:
                    del self.ends[key]
            for pg in set(pages[h // P:]):
                refs = None if step.refs is None else step.refs[pg]
                if held[pg] > 1 or (refs is not None and refs != 1):
                    self._fail("page table", f"{what} writes into page {pg}, which {refs or held[pg]} sequences hold")
        self._rows_step = rows
        return prows, drows

    def _check_history(self, before, rows):
        """Every slot of history a step reads holds, in every layer, the bytes of the reference's shadow."""
        L = len(self.layers)
        for i, (pages, n, k, running) in enumerate(rows):
            if n == k:
                continue
            pg, e = self._slots(pages, np.arange(n - k))
            if not self.known[pg, :, e].all():
                self._fail("history", f"row {i} reads slots the reference never saw written")
            if not (same(before[0][pg, :L, :, :, e], self.sd[pg, :, :, :, e]) and
                    same(before[1][pg, :L, :, :, e], self.sp[pg, :, :, :, e])):
                self._fail("pool before the step", f"row {i}: its history in the pool is not what the reference saw written")

    def _settle(self):
        """After the step: every row's sequence ends at its whole length."""
        for pages, n, k, running in self._rows_step:
            self._register(pages, n)

    def check_step(self, calls, step, pool_before=None, pool_after=None):
        """Walk the trace `calls` of one step; raises WiringError naming the first stage that differs.  pool_before / pool_after:
        (data, param) host copies for the audit.  Returns step.info: the float64 logits and their bound when the model has a head."""
        self._calls, self._pos = calls, 0
        pf, nd, S = list(step.prefills), int(step.decode), int(step.decode_len)
        doff = sum(pf)
        self._doff = doff
        m = doff + nd * S
        prows, drows = self._admit(step)
        if pool_before is not None:
            self._check_history(pool_before, prows + drows)
        ctx = any(n > k for _, n, k, _ in prows)               # a prompt over a cached prefix (a chunk, a continuation)
        cum = np.concatenate([[0], np.cumsum(pf)]).astype(np.int32)
        if step.x is not None:
            residual = step.x
        else:
            residual = self.embed[np.asarray(step.ids)]
        delta = None
        for l, p in enumerate(self.layers):
            L = f"layer {l}"
            # ---- input norm (with the previous layer's closing residual add)
            w, idx, eps = p.ln1
            if delta is None:
                c = self._next(f"{L} input_layernorm", ["rmsnorm_fp16_i4"])
                self._eq(f"{L} input_layernorm", "hidden_states", c.args["hidden_states"], residual)
                x = c.out
                ref = O.rmsnorm_fp16_i4(residual, w, idx, eps)
            else:
                st = f"{L} input_layernorm (+ residual of layer {l - 1})"
                c = self._next(st, ["add_rmsnorm_fp16_i4"])
                self._eq(st, "hidden_states", c.args["hidden_states"], delta)
                self._eq(st, "residual", c.args["residual"], residual)
                s, x = c.out
                if not same(s, fp16_sum(residual, delta)):
                    self._fail(st, "residual + delta is not the exact FP16 sum")
                residual = s
                ref = O.rmsnorm_fp16_i4(s, w, idx, eps)
            st = f"{L} input_layernorm"
            self._norm_args(st, c, p.ln1)
            self._quant(st, x, ref, m, exact=False)
            q, k4, ks, v4, vs = self._qkv(L, p, x, m)
            stack = []
            # ---- prompts: cache write at the tail of each sequence, causal attention over its cached prefix and itself
            if pf:
                st = f"{L} init_kv"
                c = self._next(st, ["init_kv_i4"])
                for name, t in (("k", k4), ("v", v4), ("k_param", ks), ("v_param", vs)):
                    self._eq(st, name, c.args[name], t[:doff])
                self._table(st, c.args["kv"], step.ptab)
                self._eq(st, "seqlen_indptr", np.asarray(c.args["seqlen_indptr"], np.int32), cum)
                if c.args["layer_idx"] != l:
                    self._fail(st, f"layer_idx {c.args['layer_idx']}, the layer is {l}")
                for i, (pages, n, k, _) in enumerate(prows):
                    r = slice(cum[i], cum[i + 1])
                    self._write(l, pages, np.arange(n - k, n), k4[r], ks[r], v4[r], vs[r], p.hkv)
                st = f"{L} prefill_attention"
                c = self._next(st, ["prefill_attention_i4"])
                for name, t in (("q", q[:doff]), ("k", k4[:doff]), ("k_param", ks[:doff]), ("v", v4[:doff]), ("v_param", vs[:doff])):
                    self._eq(st, name, c.args[name], t)
                self._eq(st, "seqlen_indptr", np.asarray(c.args["seqlen_indptr"], np.int32), cum)
                if list(c.args["seqlens"]) != pf or c.args["rope_theta"] != p.theta:
                    self._fail(st, f"seqlens {c.args['seqlens']} / rope_theta {c.args['rope_theta']}, expected {pf} / {p.theta}")
                if ctx:
                    if c.args.get("kv") is None:
                        self._fail(st, "prompts over a cached prefix, called without `kv`")
                    self._table(st, c.args["kv"], step.ptab)
                    if c.args["layer_idx"] != l:
                        self._fail(st, f"layer_idx {c.args['layer_idx']}, the layer is {l}")
                    pt = step.ptab
                    ref, bnd = prefill_ctx_bound(q[:doff], k4[:doff], ks[:doff], v4[:doff], vs[:doff], pf, p.hq, p.theta, self.sd,
                                                 self.sp, pt["indptr"], pt["indices"], pt["last"], l, rows=self.prefill_rows)
                    self._attn_bound(st, c.out, ref, bnd, "prefill over a cached prefix")
                else:
                    if c.args.get("kv") is not None:
                        self._fail(st, "whole prompts, called with `kv`")
                    ref, bnd = A.prefill_bound(q[:doff], k4[:doff], ks[:doff], v4[:doff], vs[:doff], pf, p.hq, p.theta, rows=self.prefill_rows)
                    self._attn_bound(st, c.out, ref, bnd, "prefill")
                stack.append(c.out)
            # ---- running sequences: one appended position and decode attention, or S positions and verify attention
            if nd and S > 1:
                stack.append(self._verify(L, l, p, q, k4, ks, v4, vs, doff, drows, step.dtab, S))
            elif nd:
                stack.append(self._decode(L, l, p, q, k4, ks, v4, vs, doff, nd, drows, step.dtab))
            attn = np.concatenate(stack) if len(stack) > 1 else stack[0]
            # ---- o_proj
            xo = self._reorder(L, p, attn, m)
            st = f"{L} o_proj"
            c = self._next(st, ["dense_layer_gemm_i4_fp16"])
            self._gemm_call(st, c, xo, p.o, GEMM_AUTO)
            self._o16(st, xo, p.o, c.out, G.dispatch(m, p.hidden, p.hidden, GEMM_AUTO)[1])
            o = c.out
            # ---- post-attention norm
            st = f"{L} post_attention_layernorm"
            c = self._next(st, ["add_rmsnorm_fp16_i4"])
            self._eq(st, "hidden_states", c.args["hidden_states"], o)
            self._eq(st, "residual", c.args["residual"], residual)
            w, idx, eps = p.ln2
            self._norm_args(st, c, p.ln2)
            s, x = c.out
            if not same(s, fp16_sum(residual, o)):
                self._fail(st, "residual + attention is not the exact FP16 sum")
            residual = s
            self._quant(st, x, O.rmsnorm_fp16_i4(s, w, idx, eps), m, exact=False)
            delta = self._mlp(L, p, x, m) if p.moe is None else self._moe(L, p, residual, x, m)
        if self._pos != len(calls):
            self._fail("end of step", f"{len(calls) - self._pos} kernel calls more than the step needs ({calls[self._pos].name} first)")
        h = fp16_sum(residual, delta)
        if self.lm_head is None:
            if step.out is not None and not same(step.out, h):
                self._fail("layer output", "residual + delta is not the exact FP16 sum")
        else:
            self._head(step, h)
        if pool_before is not None:
            self._audit(pool_before, pool_after)
        self._settle()
        return step.info

    # ---------------------------------------------------------------------------------------------------------- stages
    def _norm_args(self, st, c, ln):
        w, idx, eps = ln
        self._eq(st, "weight", c.args["weight"], w)
        self._eq(st, "reorder_index", c.args["reorder_index"], idx)
        if c.args["eps"] != eps:
            self._fail(st, f"eps {c.args['eps']} != {eps}")

    def _qkv(self, L, p, x, m, fused=True):
        """The q/k/v projections of the quantised input x: one fused launch, or (fused=False) q_proj, k_proj and v_proj as three
        GEMMs on the projections' own operands (p.q, p.k, p.v).  Returns (q, k codes, k (scale, zero), v codes, v (scale, zero))."""
        st = f"{L} qkv_proj"
        nq, nkv = p.hq * 128, p.hkv * 128
        rows = self._rows(m, 2 * nkv, p.hidden)
        if fused:
            c = self._next(st, ["dense_layer_gemm_i4_qkv"])
            self._gemm_call(st, c, x, p.qkv)
            if c.args["kv_rows"] != nkv:
                self._fail(st, f"kv_rows {c.args['kv_rows']} != {nkv}")
            q, (k4, ks), (v4, vs) = c.out
            self._o16(st + " (q)", x, p.qkv.rows(0, nq), q, 1)
        else:
            c = self._next(f"{L} q_proj", ["dense_layer_gemm_i4_fp16"])
            self._gemm_call(f"{L} q_proj", c, x, p.q, GEMM_AUTO)
            q = c.out
            self._o16(f"{L} q_proj", x, p.q, q, G.dispatch(m, nq, p.hidden, GEMM_AUTO)[1])
            kv = []
            for name, lin in (("k_proj", p.k), ("v_proj", p.v)):
                c = self._next(f"{L} {name}", ["dense_layer_gemm_i4_o4"])
                self._gemm_call(f"{L} {name}", c, x, lin, GEMM_AUTO)
                kv.append(c.out)
            (k4, ks), (v4, vs) = kv
            st = f"{L} k_proj / v_proj"
        self._o4(st + " (k)", x, p.qkv.rows(nq, nq + nkv), (k4, ks), rows)
        self._o4(st + " (v)", x, p.qkv.rows(nq + nkv, nq + 2 * nkv), (v4, vs), rows)
        return q, k4, ks, v4, vs

    def _decode(self, L, l, p, q, k4, ks, v4, vs, doff, nd, drows, dtab):
        """append_kv of the rows [doff, doff + nd) and decode attention over each running sequence's history (the cascade's
        bound when the table has prefix groups and ops.decode_cascade picks it); returns the attention output [nd, heads * 128]."""
        st = f"{L} append_kv"
        c = self._next(st, ["append_kv_i4"])
        for name, t in (("k", k4), ("v", v4), ("k_param", ks), ("v_param", vs)):
            self._eq(st, name, c.args[name], t[doff:])
        self._table(st, c.args["kv"], dtab)
        if c.args["layer_idx"] != l:
            self._fail(st, f"layer_idx {c.args['layer_idx']}, the layer is {l}")
        for j, (pages, n, _, _) in enumerate(drows):
            r = slice(doff + j, doff + j + 1)
            self._write(l, pages, [n - 1], k4[r], ks[r], v4[r], vs[r], p.hkv)
        st = f"{L} batch_decode"
        c = self._next(st, ["batch_decode_i4"])
        self._eq(st, "q", c.args["q"], q[doff:])
        self._table(st, c.args["kv"], dtab)
        if c.args["layer_idx"] != l or c.args["rope_theta"] != p.theta:
            self._fail(st, f"layer_idx {c.args['layer_idx']} / rope_theta {c.args['rope_theta']}, expected {l} / {p.theta}")
        qd = q[doff:].reshape(nd, p.hq, 128)
        tab = (dtab["indptr"], dtab["indices"], dtab["last"])
        if c.args.get("kv_split", 0) == 0 and self._cascade(dtab, nd, p):
            ref, bnd = cascade_bound(qd, self.sd, self.sp, *tab, l, p.hq, p.theta, dtab["shared"])
            self._attn_bound(st + " (cascade)", c.out, ref, bnd, "cascade decode")
        else:
            ref, bnd = A.decode_bound(qd, self.sd, self.sp, *tab, l, p.hq, p.theta)
            self._attn_bound(st, c.out, ref, bnd, "decode")
        return c.out.reshape(nd, p.hq * 128)

    def _cascade(self, dtab, nd, p):
        """Whether batch_decode_i4 runs the shared-prefix cascade on this table (ops.decode_cascade, on sm_count SMs)."""
        if not dtab.get("groups") or self.sm_count is None:
            return False
        from atom_b200 import ops
        return ops.decode_cascade(dtab["groups"], nd, self.P, p.hkv, p.hq // p.hkv, self.sm_count)

    def _verify(self, L, l, p, q, k4, ks, v4, vs, doff, drows, dtab, S):
        """A verify step: init_kv of each running sequence's S rows at stride S to its last S positions, and verify attention
        of those rows over the sequence's history and, causally, each other; returns the attention output [nd * S, heads * 128].
        The verify kernel does not use prefix groups: its output is held to verify_bound whatever groups the table has."""
        nd = len(drows)
        n = nd * S
        st = f"{L} init_kv (verify)"
        c = self._next(st, ["init_kv_i4"])
        for name, t in (("k", k4), ("v", v4), ("k_param", ks), ("v_param", vs)):
            self._eq(st, name, c.args[name], t[doff:])
        self._table(st, c.args["kv"], dtab)
        self._eq(st, "seqlen_indptr", np.asarray(c.args["seqlen_indptr"], np.int32), np.arange(0, n + 1, S, dtype=np.int32))
        if c.args["layer_idx"] != l:
            self._fail(st, f"layer_idx {c.args['layer_idx']}, the layer is {l}")
        for j, (pages, ln, _, _) in enumerate(drows):
            r = slice(doff + j * S, doff + (j + 1) * S)
            self._write(l, pages, np.arange(ln - S, ln), k4[r], ks[r], v4[r], vs[r], p.hkv)
        st = f"{L} batch_verify"
        c = self._next(st, ["batch_verify_i4"])
        self._eq(st, "q", c.args["q"], q[doff:])
        self._table(st, c.args["kv"], dtab)
        a = c.args
        if a["tokens_per_seq"] != S or a["layer_idx"] != l or a["rope_theta"] != p.theta:
            self._fail(st, f"tokens_per_seq {a['tokens_per_seq']} / layer_idx {a['layer_idx']} / rope_theta {a['rope_theta']}, expected "
                           f"{S} / {l} / {p.theta}")
        longest = max(ln for _, ln, _, _ in drows)
        if a["max_len"] is not None and a["max_len"] < longest:
            self._fail(st, f"max_len {a['max_len']} below the longest sequence's {longest} tokens")
        ref, bnd = VR.verify_bound(q[doff:].reshape(n, p.hq, 128), self.sd, self.sp, dtab["indptr"], dtab["indices"], dtab["last"], l,
                                   p.hq, p.theta, S)
        self._attn_bound(st, c.out, ref, bnd, "verify")
        return c.out.reshape(n, p.hq * 128)

    def _reorder(self, L, p, attn, m):
        st = f"{L} o_proj reorder"
        c = self._next(st, ["reorder_fp16_i4"])
        self._eq(st, "hidden_states ([prefill attention; decode attention])", c.args["hidden_states"], attn)
        self._eq(st, "reorder_index", c.args["reorder_index"], p.attn_index)
        self._quant(st, c.out, O.reorder_fp16_i4(attn.reshape(m, p.hq * 128), p.attn_index), m)
        return c.out

    def _mlp(self, L, p, x, m):
        """gate/up and activate, then down; returns the FP16 delta."""
        xa = self._gateup(L, p, x, m)
        st = f"{L} down_proj"
        c = self._next(st, ["dense_layer_gemm_i4_fp16"])
        self._gemm_call(st, c, xa, p.down, GEMM_AUTO)
        self._o16(st, xa, p.down, c.out, G.dispatch(m, p.hidden, p.inter, GEMM_AUTO)[1])
        return c.out

    def _gateup(self, L, p, x, m):
        """gate/up (one fused launch for M <= 64, else two GEMMs and activate); returns the quantised activation."""
        if m <= 64:
            st = f"{L} gate/up (fused)"
            c = self._next(st, ["dense_layer_gemm_i4_gateup_act"])
            self._gemm_call(st, c, x, p.gu)
            rows = self._rows(m, 2 * p.inter, p.hidden)
            gate = O.gemm_i4_o16(x[1], p.gate.b, x[3], p.gate.bs, x[0], p.gate.bk, x[2], p.gate.bks, rows=rows)
            up = O.gemm_i4_o16(x[1], p.up.b, x[3], p.up.bs, x[0], p.up.bk, x[2], p.up.bks, rows=rows)
            self._quant(st, c.out, O.activate_fp16_i4(gate, up), m, rows=rows, exact=False)
        else:
            outs = []
            for name, lin in (("gate_proj", p.gate), ("up_proj", p.up)):
                st = f"{L} {name}"
                c = self._next(st, ["dense_layer_gemm_i4_fp16"])
                self._gemm_call(st, c, x, lin, GEMM_AUTO)
                self._o16(st, x, lin, c.out, G.dispatch(m, p.inter, p.hidden, GEMM_AUTO)[1])
                outs.append(c.out)
            st = f"{L} activate"
            c = self._next(st, ["activate_fp16_i4"])
            self._eq(st, "a (gate)", c.args["a"], outs[0])
            self._eq(st, "b (up)", c.args["b"], outs[1])
            self._quant(st, c.out, O.activate_fp16_i4(outs[0], outs[1]), m, exact=False)
        return c.out

    def _moe(self, L, p, s, x, m):
        """The sparse MoE block on the residual sum s and its quantised post-attention norm x; returns the FP16 delta."""
        mo = p.moe
        w, idx, eps = p.ln2
        st = f"{L} moe route"
        c = self._next(st, ["moe_route_f16"])
        for name, t in (("hidden_sum", s), ("norm_weight", w), ("reorder_index", idx), ("router_weight", mo.router)):
            self._eq(st, name, c.args[name], t)
        if c.args["eps"] != eps or c.args["top_k"] != mo.k:
            self._fail(st, f"eps {c.args['eps']} / top_k {c.args['top_k']}, expected {eps} / {mo.k}")
        ids, tw = c.out
        # float64 logits of the exact normalised row (reordered order).  The kernel's row is that row rounded to FP16 (u relative,
        # 2^-25 absolute below the normal range) after an FP32 rsqrtf (2^-20 with slack), and its FP32 dot products carry
        # moe_ref.logit_error_bound: delta bounds |kernel logit - float64 logit|.
        s64 = s.astype(np.float64)
        y = (s64 * w.astype(np.float64) / np.sqrt((s64 * s64).mean(1, keepdims=True) + eps))[:, idx]
        wr = mo.router.astype(np.float64)
        lg = y @ wr.T
        ay = np.abs(y) @ np.abs(wr).T
        n = p.hidden // 32 + 5                                                    # moe_ref.logit_error_bound, every row at once
        delta = n * U32 / (1 - n * U32) * ((np.abs(y) * (1 + U16) + 2.0 ** -25) @ np.abs(wr).T) + (U16 + 2.0 ** -20) * ay \
            + 2.0 ** -25 * np.abs(wr).sum(1)
        if ids.shape != (m, mo.k) or (ids < 0).any() or (ids >= mo.e).any() or \
                any(len(set(r)) != mo.k for r in ids.tolist()):
            self._fail(st, "topk_ids are not k distinct experts per token")
        srt = -np.sort(-lg, axis=1)
        for t in range(m):
            d = delta[t].max()
            if mo.k == mo.e or srt[t, mo.k - 1] - srt[t, mo.k] > 2 * d:
                want = sorted(ME.topk_f64(lg[t], mo.k)[0].tolist())
                if sorted(ids[t].tolist()) != want:
                    self._fail(st, f"token {t}: experts {sorted(ids[t].tolist())}, the float64 top-{mo.k} is {want}")
            pe = np.exp(lg[t, ids[t]] - lg[t, ids[t]].max())
            w64 = pe / pe.sum()
            ulp = 2.0 ** (np.floor(np.log2(np.maximum(w64, 2.0 ** -14))) - 10)
            if not (np.abs(tw[t].astype(np.float64) - w64) <= w64 * np.expm1(2 * d) + ulp).all():
                self._fail(st, f"token {t}: routing weights {tw[t].tolist()}, float64 {w64.tolist()}")
        bn = ME.token_tile(m, mo.e, mo.k)
        tmax = ME.tiles_max(m, mo.e, mo.k, bn)
        rows_cap = tmax * bn
        st = f"{L} moe plan"
        c = self._next(st, ["moe_plan"])
        self._eq(st, "topk_ids", c.args["topk_ids"], ids)
        if (c.args["num_experts"], c.args["token_tile"], c.args["tiles_max"]) != (mo.e, bn, tmax):
            self._fail(st, f"(experts, token tile, tiles) {(c.args['num_experts'], c.args['token_tile'], c.args['tiles_max'])}, "
                           f"expected {(mo.e, bn, tmax)}")
        dest, tiles = c.out
        rd, rt = ME.plan(ids, mo.e, bn, tmax)
        if not (np.array_equal(dest, rd) and np.array_equal(tiles, rt)):
            self._fail(st, "dest_row / tile table differ from the routing's plan")
        st = f"{L} moe gather"
        c = self._next(st, ["moe_gather_i4"])
        if not all(same(u, v) for u, v in zip(c.args["x"], x)):
            self._fail(st, "`x` is not the tensor this stage consumes")
        self._eq(st, "dest_row", c.args["dest_row"], dest)
        if c.args["rows_cap"] != rows_cap:
            self._fail(st, f"rows_cap {c.args['rows_cap']}, expected {rows_cap}")
        xp = c.out
        tok, live = np.repeat(np.arange(m), mo.k), dest.reshape(-1)
        gc, gs = quant_rows(xp, rows_cap)
        rc, rs = quant_rows(x, m)
        if not (np.array_equal(gc[live], rc[tok]) and same(gs[:, live], rs[:, tok])):
            self._fail(st, "a permuted row is not its token's quantised row")
        experts = [(e, dest[ids == e]) for e in range(mo.e) if (ids == e).any()]
        st = f"{L} moe gate/up (grouped)"
        c = self._next(st, ["dense_layer_gemm_i4_gateup_act_grouped"])
        self._grouped_args(st, c, xp, ("w13_int4", "w13_scale", "w13_int8", "w13_keeper_scale"), mo.w13, tiles, bn)
        act = c.out
        w4, s4, w8, s8 = mo.w13
        for e, r in experts:
            g = O.gemm_i4_o16(xp[1], w4[e], xp[3], s4[e], xp[0], w8[e], xp[2], s8[e], rows=r)
            self._quant(f"{st}, expert {e}", act, O.activate_fp16_i4(g[:, :mo.inter], g[:, mo.inter:]), rows_cap, rows=r, exact=False)
        st = f"{L} moe down (grouped)"
        c = self._next(st, ["dense_layer_gemm_i4_fp16_grouped"])
        self._grouped_args(st, c, act, ("w2_int4", "w2_scale", "w2_int8", "w2_keeper_scale"), mo.w2, tiles, bn)
        y = c.out
        w4, s4, w8, s8 = mo.w2
        for e, r in experts:
            t = (act[1], w4[e], act[3], s4[e], act[0], w8[e], act[2], s8[e])
            ref = O.gemm_i4_o16(*t, rows=r)
            if not same(y[r], ref):
                self._fail(f"{st}, expert {e}", "FP16 GEMM differs from the oracle")
            S, T = G.ref64(*t, rows=r)
            G.check_o16(y[r], S, T, mo.inter // 128 - 1, 1, what=f"{st}, expert {e}")
        st = f"{L} moe combine"
        c = self._next(st, ["moe_combine_f16"])
        for name, t in (("y", y), ("topk_ids", ids), ("topk_weights", tw), ("dest_row", dest)):
            self._eq(st, name, c.args[name], t)
        ref = np.zeros((m, p.hidden), np.float16)                      # ascending experts, FP16 products and adds from +0
        for e in range(mo.e):
            t, k = np.nonzero(ids == e)
            prod = (y[dest[t, k]].astype(np.float64) * tw[t, k, None].astype(np.float64)).astype(np.float16)
            ref[t] = fp16_sum(ref[t], prod)
        if not same(c.out, ref):
            self._fail(st, "the combine is not the ascending-expert FP16 index_add_ loop")
        return c.out

    def _grouped_args(self, st, c, xin, names, w, tiles, bn):
        if not all(same(u, v) for u, v in zip(c.args["x"], xin)):
            self._fail(st, "`x` is not the tensor this stage consumes")
        for name, t in zip(names, w):
            self._eq(st, name, c.args[name], t)
        self._eq(st, "tiles", c.args["tiles"], tiles)
        if c.args["token_tile"] != bn:
            self._fail(st, f"token_tile {c.args['token_tile']}, expected {bn}")

    def _head(self, step, h):
        """LlamaRMSNorm (torch, FP32 statistics, two FP16 roundings) and lm_head (FP16 GEMM, FP32 accumulation) in float64."""
        logits, hn = step.out
        w, eps = self.norm
        x = h.astype(np.float64)
        n64 = x / np.sqrt((x * x).mean(1, keepdims=True) + eps) * w.astype(np.float64)
        bnd = (2 * U16 + 2.0 ** -20) * np.abs(n64) + 2.0 ** -24
        if not (np.abs(hn.astype(np.float64) - n64) <= bnd).all():
            self._fail("final norm", "LlamaRMSNorm output outside its bound")
        W = self.lm_head.astype(np.float64)
        n = hn.astype(np.float64)                                       # borrowed
        S, T = n @ W.T, np.abs(n) @ np.abs(W).T
        K = W.shape[1]
        err = K * U32 / (1 - K * U32) * T
        hi = np.abs(S) + err
        b = err + np.maximum(2.0 ** (np.floor(np.log2(np.maximum(hi, 2.0 ** -14))) - 11), 2.0 ** -25)
        if not (np.abs(logits.astype(np.float64) - S) <= b).all():
            self._fail("lm_head", "logits outside gamma_K sum|x w| + half an ulp of the float64 product")
        step.info.update(logits64=S, bound=b)
        if step.rows is not None:
            dec = list(range(sum(step.prefills), sum(step.prefills) + step.decode * step.decode_len))
            rows, last = [int(r) for r in step.rows], cum_last(step.prefills)
            first = rows[:len(rows) - len(dec)]
            if rows[len(first):] != dec or any(r not in last for r in first) or first != sorted(set(first)):
                self._fail("last_token_rows", f"logits read at rows {rows}: the last token of prompts it completes (of {last}) and every "
                                              f"decode row ({dec}) are expected")

    def _audit(self, before, after):
        """The slots the step wrote hold the shadow's bytes in every layer; every other byte is as it was before the step."""
        data, param = before[0].copy(), before[1].copy()
        L = len(self.layers)
        for pg, e in self._written:
            data[pg, :L, :, :, e], param[pg, :L, :, :, e] = self.sd[pg, :, :, :, e], self.sp[pg, :, :, :, e]
        bad_d = np.argwhere(data != after[0])
        bad_p = np.argwhere(param.view(np.uint16) != after[1].view(np.uint16))
        if len(bad_d) or len(bad_p):
            where = (bad_d if len(bad_d) else bad_p)[0].tolist()
            self._fail(f"layer {where[1]} pool audit", f"{len(bad_d)} data bytes and {len(bad_p)} parameters differ from the reference's shadow "
                                     f"(slots the step wrote) or from the pool before the step (all others); first at "
                                     f"[page, layer, k|v, head, entry] = {where[:5]}")

    def _argmax(self, step, st, r, token):
        """token is the float64 argmax of logits row r wherever the top-2 gap exceeds twice the logits' bound."""
        S, b = step.info["logits64"], step.info["bound"]
        top = np.argsort(S[r])[::-1][:2]
        if S[r, top[0]] - S[r, top[1]] > 2 * (b[r, top[0]] + b[r, top[1]]) and int(token) != int(top[0]):
            self._fail(st, f"row {r}: token {int(token)}, the float64 argmax is {int(top[0])}")

    def check_tokens(self, step, tokens):
        """Greedy tokens of a step (one per row of step.rows, or of the last row of each prompt and every decode row): the argmax
        of the float64 logits wherever the top-2 gap exceeds twice the logits' bound."""
        rows = step.rows if step.rows is not None else \
            cum_last(step.prefills) + list(range(sum(step.prefills), sum(step.prefills) + step.decode * step.decode_len))
        for r, t in zip(rows, tokens):
            self._argmax(step, "greedy token", int(r), t)

    def check_spec(self, step, drafts, emitted, room=None, stop_ids=()):
        """Greedy speculative tokens of a step (its rows: step.rows, as the scheduler reads them).  emitted: the tokens each
        sequence emitted -- one for each prompt the step completes, then every running sequence's; drafts: each running
        sequence's drafts (the inputs of its rows 1, 2, ..).  Row by row, emitted token j is the float64 argmax of row j, and draft
        j + 1 is accepted exactly when it equals that token: a sequence emits its accepted prefix + 1 tokens.  room: tokens each
        running sequence may still emit (its output length), stop_ids: ids that end a request.  The tokens a sequence keeps --
        emitted, cut at the room and at the first stop id -- set the length the next step must continue it at (keep).  Returns
        the kept counts."""
        st = "speculative commit"
        S, nd, doff = int(step.decode_len), int(step.decode), sum(step.prefills)
        rows = [int(r) for r in step.rows]
        first = len(rows) - nd * S
        if len(emitted) != first + nd or len(drafts) != nd:
            self._fail(st, f"{len(emitted)} sequences emitted and {len(drafts)} drafted, the step has {first} prompts it completes and "
                           f"{nd} running sequences")
        for i in range(first):
            if len(emitted[i]) != 1:
                self._fail(st, f"prompt {i}: {len(emitted[i])} tokens emitted for its first")
            self._argmax(step, st, rows[i], emitted[i][0])
        kept = []
        for i in range(nd):
            em, dr = [int(t) for t in emitted[first + i]], [int(t) for t in drafts[i]]
            j = 0
            while True:
                if j >= len(em):
                    self._fail(st, f"sequence {i}: {len(em)} tokens emitted, its accepted drafts call for {j + 1}")
                self._argmax(step, st, doff + i * S + j, em[j])
                if j + 1 < S and j < len(dr) and dr[j] == em[j]:
                    j += 1
                    continue
                break
            if len(em) != j + 1:
                self._fail(st, f"sequence {i}: {len(em)} tokens emitted ({em}); its drafts {dr} against the emitted tokens accept {j}")
            c = j + 1 if room is None else min(j + 1, int(room[i]))
            c = next((t + 1 for t in range(c) if em[t] in stop_ids), c)
            kept.append(c)
        self.keep(kept)
        return kept


def cum_last(prefills):
    return (np.cumsum(prefills) - 1).tolist() if len(prefills) else []


# ------------------------------------------------------------------------------------------------------------------ driving
def model_ref(model, P, **kw):
    """ModelRef of a LlamaForCausalLM (layers fused)."""
    m = model.model
    return ModelRef([LayerParams(l, i) for i, l in enumerate(m.layers)], P, embed=host(m.embed_tokens.weight),
                    norm=(host(m.norm.weight), m.norm.variance_epsilon), lm_head=host(model.lm_head.weight), **kw)


def run_step(rec, pool, fn, inp, blen, prefill_kv, decode_kv, ids=True):
    """fn(inp, blen, prefill_kv, decode_kv) with the kernels recorded.  inp: token ids (ids=True) or the FP16 hidden states.
    Returns (out, Step, calls, pool before, pool after) for ModelRef.check_step (set Step.rows first where tokens are read)."""
    step = Step(list(blen.prefills), blen.decode, host(prefill_kv) if prefill_kv is not None else None,
                host(decode_kv) if decode_kv is not None else None, decode_len=getattr(blen, "decode_len", 1),
                refs=list(pool._refs) if hasattr(pool, "_refs") else None)
    if ids:
        step.ids = host(inp)
    else:
        step.x = host(inp)
    before = (host(pool.buf), host(pool.param))
    rec.calls.clear()
    out = fn(inp, blen, prefill_kv, decode_kv)
    step.out = host(out)
    return out, step, list(rec.calls), before, (host(pool.buf), host(pool.param))
