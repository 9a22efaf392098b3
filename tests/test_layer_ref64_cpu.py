"""CPU self-test of tests/layer_ref64.py.  The real LlamaForCausalLM code runs on the CPU with every kernel replaced by its oracle
(oracle/atom_oracle.c; attn_ref64, attn_ctx_ref64 and attn_verify_ref64 for attention), which gives a recorded trace of a
two-layer prefill step and a mixed prefill + decode step, and of a serving sequence with chunked prompts, forks, continuations and
verify steps truncated to several kept counts.  The reference must (a) accept those traces and (b) reject each seeded wiring
fault, naming the stage."""
import types

import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import attn_ref64 as A
from tests import attn_verify_ref64 as VR
from tests import gemm_ref64 as G
from tests.attn_ctx_ref64 import prefill_ctx_ref
from tests import layer_ref64 as R

P = 8


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def _quant(t4):
    o8, o4, s8, s4 = t4
    return (torch.from_numpy(o8), torch.from_numpy(o4.view(np.int8)), torch.from_numpy(s8), torch.from_numpy(s4))


def _o16(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, ksplit):
    return O.gemm_i4_o16(*[_np(t) for t in (a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale)], ksplit=ksplit)


def _cols(s, a, b):
    s = _np(s)
    return np.ascontiguousarray(s.reshape(s.shape[0], -1)[:, a:b]) if s.ndim == 2 else np.ascontiguousarray(s[a:b])


# ---- the operators, on the oracle (same names and signatures as atom_b200.ops)
def rmsnorm_fp16_i4(hidden_states, weight, reorder_index, eps):
    return _quant(O.rmsnorm_fp16_i4(_np(hidden_states), _np(weight).astype(np.float16), _np(reorder_index), eps))


def add_rmsnorm_fp16_i4(hidden_states, residual, weight, reorder_index, eps):
    s = R.fp16_sum(_np(residual), _np(hidden_states))
    return torch.from_numpy(s), rmsnorm_fp16_i4(torch.from_numpy(s), weight, reorder_index, eps)


def reorder_fp16_i4(hidden_states, reorder_index):
    return _quant(O.reorder_fp16_i4(_np(hidden_states), _np(reorder_index)))


def activate_fp16_i4(a, b):
    return _quant(O.activate_fp16_i4(_np(a), _np(b)))


def dense_layer_gemm_i4_fp16(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, flags=0):
    ksplit = G.dispatch(a.shape[0], b.shape[0], a.shape[1] * 2 + 128, flags)[1]
    return torch.from_numpy(_o16(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, ksplit))


def dense_layer_gemm_i4_o4(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, flags=0):
    d, ds = O.gemm_i4_o4(*[_np(t) for t in (a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale)])
    return torch.from_numpy(d), torch.from_numpy(ds)


def dense_layer_gemm_i4_qkv(a, b_qkv, a_scale, b_scale_qkv, a_keeper, b_keeper_qkv, a_keeper_scale, b_keeper_scale_qkv, flags=0,
                            kv_rows=None):
    n3 = b_qkv.shape[0]
    nq = n3 - 2 * kv_rows
    part = lambda lo, hi: (a, b_qkv[lo:hi], a_scale, _cols(b_scale_qkv, lo, hi), a_keeper, b_keeper_qkv[lo:hi], a_keeper_scale,  # noqa: E731
                           _cols(b_keeper_scale_qkv, lo, hi))
    q = torch.from_numpy(_o16(*part(0, nq), 1))
    return q, dense_layer_gemm_i4_o4(*part(nq, nq + kv_rows)), dense_layer_gemm_i4_o4(*part(nq + kv_rows, n3))


def dense_layer_gemm_i4_gateup_act(a, b_gu, a_scale, b_scale_gu, a_keeper, b_keeper_gu, a_keeper_scale, b_keeper_scale_gu, flags=0):
    i = b_gu.shape[0] // 2
    part = lambda lo, hi: (a, b_gu[lo:hi], a_scale, _cols(b_scale_gu, lo, hi), a_keeper, b_keeper_gu[lo:hi], a_keeper_scale,  # noqa: E731
                           _cols(b_keeper_scale_gu, lo, hi))
    return _quant(O.activate_fp16_i4(_o16(*part(0, i), 1), _o16(*part(i, 2 * i), 1)))


def _table(kv):
    return _np(kv.indptr), _np(kv.indicies), _np(kv.last_page_offset)


def init_kv_i4(kv, k, v, k_param, v_param, seqlen_indptr, layer_idx):
    O.init_kv_i4(_np(kv.data), _np(kv.param), *_table(kv), _np(k), _np(v), _np(k_param), _np(v_param), _np(seqlen_indptr), layer_idx)


def append_kv_i4(kv, k, v, k_param, v_param, layer_idx):
    O.append_kv_i4(_np(kv.data), _np(kv.param), *_table(kv), _np(k), _np(v), _np(k_param), _np(v_param), layer_idx)


def prefill_attention_i4(q, k, k_param, v, v_param, seqlen_indptr, seqlens=None, rope_theta=10000.0, *, kv=None, layer_idx=None):
    if kv is None:
        o = A.prefill_ref(_np(q), _np(k), _np(k_param), _np(v), _np(v_param), seqlens, q.shape[1] // 128, rope_theta)
    else:
        o = prefill_ctx_ref(_np(q), _np(k), _np(k_param), _np(v), _np(v_param), seqlens, q.shape[1] // 128, rope_theta, _np(kv.data),
                            _np(kv.param), *_table(kv), layer_idx)
    return torch.from_numpy(o.astype(np.float16))


def batch_decode_i4(q, kv, layer_idx, rope_theta=10000.0):
    """decode_ref on the pool: over forked rows too (shared pages hold the same bytes for every holder)."""
    o = A.decode_ref(_np(q), _np(kv.data), _np(kv.param), *_table(kv), layer_idx, q.shape[1], rope_theta)
    return torch.from_numpy(o.astype(np.float16))


def batch_verify_i4(q, kv, layer_idx, tokens_per_seq, rope_theta=10000.0, max_len=None, nchunks=0, **defect):
    o = VR.verify_variant(_np(q), _np(kv.data), _np(kv.param), *_table(kv), layer_idx, q.shape[1], rope_theta, tokens_per_seq, **defect)
    return torch.from_numpy(o.astype(np.float16))


ORACLE_OPS = {n: globals()[n] for n in R.RECORDED_OPS if n in globals()}      # the Llama layers' kernels


# ---- seeded kernel faults: the layer passes the right arguments, the kernel stores to the wrong place.  Only the reference's
#      own history (decode attention bound, pool audit) can see them.
def _append_late_in_kernel(kv, k, v, k_param, v_param, layer_idx):
    late = types.SimpleNamespace(data=kv.data, param=kv.param, indptr=kv.indptr, indicies=kv.indicies,
                                 last_page_offset=kv.last_page_offset + 1)
    append_kv_i4(late, k, v, k_param, v_param, layer_idx)


def _init_kv_into_layer0_in_kernel(kv, k, v, k_param, v_param, seqlen_indptr, layer_idx):
    init_kv_i4(kv, k, v, k_param, v_param, seqlen_indptr, 0)


def _ctx_positions_from_zero_in_kernel(q, k, k_param, v, v_param, seqlen_indptr, seqlens=None, rope_theta=10000.0, *, kv=None,
                                       layer_idx=None):
    """The chunk's queries rotated at positions 0 .. n - 1 instead of ctx .. ctx + n - 1 (its keys where they are): q turned
    back by ctx positions in float64 before the exact reference."""
    if kv is None:
        return prefill_attention_i4(q, k, k_param, v, v_param, seqlen_indptr, seqlens, rope_theta)
    qq = _np(q).astype(np.float64).reshape(len(_np(q)), -1, 2, 64)
    f = A.freqs(rope_theta)
    off = 0
    for n, total in zip(seqlens, kv.seqlens):
        z = (qq[off:off + n, :, 0] + 1j * qq[off:off + n, :, 1]) * np.exp(-1j * (total - n) * f)
        qq[off:off + n, :, 0], qq[off:off + n, :, 1] = z.real, z.imag
        off += n
    o = prefill_ctx_ref(qq.reshape(len(qq), -1), _np(k), _np(k_param), _np(v), _np(v_param), seqlens, q.shape[1] // 128, rope_theta,
                        _np(kv.data), _np(kv.param), *_table(kv), layer_idx)
    return torch.from_numpy(o.astype(np.float16))


def _verify_defect(**defect):
    return lambda q, kv, layer_idx, tokens_per_seq, rope_theta=10000.0, max_len=None, nchunks=0: \
        batch_verify_i4(q, kv, layer_idx, tokens_per_seq, rope_theta, max_len, nchunks, **defect)


KERNEL_FAULTS = {"append_late_in_kernel": ("append_kv_i4", _append_late_in_kernel),
                 "init_kv_into_layer0_in_kernel": ("init_kv_i4", _init_kv_into_layer0_in_kernel),
                 "ctx_positions_from_zero_in_kernel": ("prefill_attention_i4", _ctx_positions_from_zero_in_kernel),
                 "verify_limit_off_by_one_in_kernel": ("batch_verify_i4", _verify_defect(limit_shift=1)),
                 "verify_rotated_at_last_in_kernel": ("batch_verify_i4", _verify_defect(rotate_at_last=True)),
                 "verify_kv_head_mod_in_kernel": ("batch_verify_i4", _verify_defect(head_mod=True))}


# ---- the seeded faults: each wraps an operator (a wiring mistake between the layer and the kernel) or a model method
def _fault(monkeypatch, name, state):
    from atom_b200 import ops
    from atom_b200 import textgen
    from atom_b200.llama import LlamaDecoderLayer
    if name == "kv_rows_swapped":              # the K/V of the first two running sequences exchanged
        f = ops.append_kv_i4
        monkeypatch.setattr(ops, "append_kv_i4", lambda kv, k, v, kp, vp, l: f(kv, k[[1, 0]], v[[1, 0]], kp[[1, 0]], vp[[1, 0]], l))
    elif name == "append_late":                # the new token written one position past the end
        f = ops.append_kv_i4
        late = lambda kv: types.SimpleNamespace(data=kv.data, param=kv.param, indptr=kv.indptr, indicies=kv.indicies,  # noqa: E731
                                                last_page_offset=kv.last_page_offset + 1)
        monkeypatch.setattr(ops, "append_kv_i4", lambda kv, k, v, kp, vp, l: f(late(kv), k, v, kp, vp, l))
    elif name == "layer1_into_layer0":         # every layer writes its K/V into layer 0's slots
        fa, fi = ops.append_kv_i4, ops.init_kv_i4
        monkeypatch.setattr(ops, "append_kv_i4", lambda kv, k, v, kp, vp, l: fa(kv, k, v, kp, vp, 0))
        monkeypatch.setattr(ops, "init_kv_i4", lambda kv, k, v, kp, vp, ip, l: fi(kv, k, v, kp, vp, ip, 0))
    elif name == "cat_order":                  # [decode attention; prefill attention]
        f = ops.reorder_fp16_i4

        def swapped(h, idx):
            d = state["doff"]
            return f(torch.cat([h[d:], h[:d]]) if 0 < d < h.shape[0] else h, idx)
        monkeypatch.setattr(ops, "reorder_fp16_i4", swapped)
    elif name == "delta_dropped":              # forward_residual loses the previous layer's MLP delta
        f = LlamaDecoderLayer.forward_residual
        monkeypatch.setattr(LlamaDecoderLayer, "forward_residual", lambda self, res, delta, *a: f(self, res, None, *a))
    elif name == "last_token_rows_off_by_one":
        f = textgen.TextGenScheduler.last_token_rows
        monkeypatch.setattr(textgen.TextGenScheduler, "last_token_rows", lambda self: [r - 1 for r in f(self)])
    else:
        raise ValueError(name)


def _model(hidden=256, heads=2, kv_heads=1):
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(3)
    torch.set_default_dtype(torch.float16)
    try:
        model = LlamaForCausalLM(LlamaConfig(hidden_size=hidden, intermediate_size=384, num_attention_heads=heads, num_key_value_heads=kv_heads,
                                             num_hidden_layers=2, vocab_size=64, rope_theta=5e5)).eval()
    finally:
        torch.set_default_dtype(torch.float32)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    for layer in model.model.layers:
        layer.fuse()
        for n in (layer.input_layernorm, layer.post_attention_layernorm):
            n.weight.data.uniform_(0.5, 1.5)
    model.model.norm.weight.data.uniform_(0.5, 1.5)
    return model


def _run(monkeypatch, fault=None):
    """Step 1 prefills prompts [5, 11]; step 2 is mixed: prompt [7], then one token of each of the two."""
    from atom_b200 import textgen
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    monkeypatch.setattr(torch.cuda.nvtx, "range_push", lambda *a: None)
    monkeypatch.setattr(torch.cuda.nvtx, "range_pop", lambda *a: None)
    model = _model()
    cpu = torch.device("cpu")
    impl = dict(ORACLE_OPS)
    if fault in KERNEL_FAULTS:
        impl.update([KERNEL_FAULTS[fault]])
    rec = R.Recorder(impl).install(monkeypatch)
    state = {"doff": 0}
    if fault and fault not in KERNEL_FAULTS:
        _fault(monkeypatch, fault, state)
    ref = R.model_ref(model, P)
    pool = KvPoolInt4(2, 1, 128, 12, P, cpu)
    pool.buf.random_(0, 256)
    pool.param.view(torch.int16).random_(-32768, 32767)         # any bits, NaN included: the audit compares bytes
    rng = np.random.default_rng(0)
    seqs, last = [], []
    for prompts, running in (([5, 11], []), ([7], [0, 1])):
        for i in running:
            seqs[i].acquire_one()
        new = [KvCacheInt4(pool, n) for n in prompts]
        ids = torch.tensor(sum((rng.integers(0, 64, n).tolist() for n in prompts), []) + [last[i] for i in running])
        blen = BatchLenInfo(prompts, len(running), cpu)
        state["doff"] = blen.doff
        with torch.inference_mode():
            out, step, calls, before, after = R.run_step(rec, pool, model, ids, blen, BatchedKvCacheInt4(new),
                                                         BatchedKvCacheInt4([seqs[i] for i in running]) if running else None)
        step.rows = textgen.TextGenScheduler.last_token_rows(types.SimpleNamespace(_blen=blen))
        tokens = torch.argmax(out[0][step.rows], -1).tolist()
        ref.check_step(calls, step, before, after)
        ref.check_tokens(step, tokens)
        if not running:
            seqs, last = new, tokens
    return ref


def test_reference_accepts_the_oracle_trace(monkeypatch):
    ref = _run(monkeypatch)
    assert sorted(e[0] for e in ref.ends.values()) == [6, 7, 12]


@pytest.mark.parametrize("fault,stage", [
    ("kv_rows_swapped", r"layer 0 append_kv: `k`"),
    ("append_late", r"layer 0 append_kv: page table `last`"),
    ("layer1_into_layer0", r"layer 1 init_kv: layer_idx 0"),
    ("cat_order", r"layer 0 o_proj reorder: `hidden_states \(\[prefill attention; decode attention\]\)`"),
    ("delta_dropped", r"layer 1 input_layernorm \(\+ residual of layer 0\): expected a call to add_rmsnorm_fp16_i4, got rmsnorm"),
    ("last_token_rows_off_by_one", r"last_token_rows"),
])
def test_reference_rejects_a_seeded_wiring_fault(monkeypatch, fault, stage):
    with pytest.raises(R.WiringError, match=stage):
        _run(monkeypatch, fault)


@pytest.mark.parametrize("fault,stage", [
    ("append_late_in_kernel", r"layer 0 batch_decode: attention output outside the float64 bound"),
    ("init_kv_into_layer0_in_kernel", r"pool audit"),
])
def test_reference_rejects_a_kernel_that_stores_to_the_wrong_slot(monkeypatch, fault, stage):
    with pytest.raises(R.WiringError, match=stage):
        _run(monkeypatch, fault)


# ---- serving sequences: chunked prompts, forks, continuations and verify steps
class Driver:
    """Steps of a model (token ids in, logits out) or of a layer stack (ids=False: hidden states in) as the serving scheduler
    forms them, every one checked by `ref`.  Sequences are named; a prompt chunk of a sequence is the tail of its cached tokens;
    `fork` starts a sequence on another's first n tokens (the reference is told through a wrapper of KvCacheInt4.fork).  A step's
    running sequences carry S rows each -- their last token and drafts -- and, for S > 1, keep either the counts the test gives
    (ModelRef.keep) or what greedy acceptance of the drafts emits (ModelRef.check_spec, models only)."""

    def __init__(self, monkeypatch, fn, pool, ref, impl=None, fault=None, ids=True, vocab=64, setup=None):
        from atom_b200 import textgen
        from atom_b200.kvcache import KvCacheInt4
        self.rec = R.Recorder(impl).install(monkeypatch)
        if setup is not None:               # (seeded faults: around the recorded operators, under the fork hook)
            setup()
        self.fn, self.pool, self.ref, self.fault, self.ids, self.vocab = fn, pool, ref, fault, ids, vocab
        real = KvCacheInt4.fork

        def fork(kv, n=None):
            child = real(kv, n)
            ref.fork(list(kv.indicies), child.seqlen, list(child.indicies))
            return child
        monkeypatch.setattr(KvCacheInt4, "fork", fork)
        self.rows_of = textgen.TextGenScheduler.last_token_rows
        self.kv, self.total, self.done, self.last = {}, {}, {}, {}
        self.rng = np.random.default_rng(1)
        self.kept = []

    def fork(self, name, parent, n=None, total=0):
        self.kv[name] = self.kv[parent].fork(n)
        self.total[name], self.done[name] = total, 0

    def step(self, chunks=(), running=(), S=1, kept=None):
        """chunks: [(name, tokens, prompt length)] (a new name starts a sequence; prompt length None = the root of forks, which
        draws no token); running: names of running sequences."""
        from atom_b200.cat_tensor import BatchLenInfo
        from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4
        dev = self.pool.device
        new = []
        for name, n, total in chunks:
            if name not in self.kv:
                self.kv[name], self.total[name], self.done[name] = KvCacheInt4(self.pool, 0), total, 0
            elif total is not None:
                self.total[name] = total
            self.kv[name].acquire(n)
            new.append((types.SimpleNamespace(prompt=[0] * (self.total[name] or 0), req_idx=-1 if self.total[name] is None else 0),
                        self.done[name], n))
            self.done[name] += n
        drafts = {r: self.rng.integers(0, self.vocab, S - 1).tolist() for r in running}
        for r in running:
            self.kv[r].acquire(S - 1)
        m = sum(n for _, n, _ in chunks) + S * len(running)
        if self.ids:
            inp = torch.tensor(sum((self.rng.integers(0, self.vocab, n).tolist() for _, n, _ in chunks), []) +
                               sum(([self.last[r]] + drafts[r] for r in running), []), device=dev)
        else:
            inp = torch.from_numpy((self.rng.standard_normal((m, self.ref.layers[0].hidden)) * 0.5).astype(np.float16)).to(dev)
        blen = BatchLenInfo([n for _, n, _ in chunks], len(running), dev, decode_len=S)
        with torch.inference_mode():
            out, step, calls, before, after = R.run_step(
                self.rec, self.pool, self.fn, inp, blen, BatchedKvCacheInt4([self.kv[c] for c, _, _ in chunks]) if chunks else None,
                BatchedKvCacheInt4([self.kv[r] for r in running]) if running else None, ids=self.ids)
        firsts = [c for (c, _, _), (p, s, k) in zip(chunks, new) if self.total[c] is not None and s + k == self.total[c]]
        if self.ref.lm_head is not None:
            step.rows = self.rows_of(types.SimpleNamespace(_blen=blen, _new=new))
        self.ref.check_step(calls, step, before, after)
        emitted = self._emit(step, out, blen, firsts, running, drafts, S, kept)
        self.kept.append([len(e) for e in emitted[len(firsts):]])
        for name, em in zip(firsts + list(running), emitted):
            if name in running:
                self.kv[name].truncate(self.kv[name].seqlen - S + len(em))
            self.last[name] = em[-1]
            self.kv[name].acquire_one()
        return step

    def _emit(self, step, out, blen, firsts, running, drafts, S, kept):
        """The tokens each sequence emits, checked: one per completed prompt, then the running sequences' (kept[i] of them, or
        greedy acceptance of the drafts)."""
        if self.ref.lm_head is None:
            assert S == 1 or kept is not None
            if S > 1:
                self.ref.keep(kept)
            return [[0]] * len(firsts) + [[0] * (1 if kept is None else kept[i]) for i in range(len(running))]
        logits = out[0].float()
        arg = lambda r: int(torch.argmax(logits[r]))                                                   # noqa: E731
        emitted = [[arg(r)] for r in step.rows[:len(firsts)]]
        for i, r in enumerate(running):
            base = blen.doff + i * S
            if kept is not None:
                emitted.append([arg(base + j) for j in range(kept[i])])
                continue
            em, j = [], 0                           # greedy acceptance, row by row
            while True:
                t = arg(base + j)
                if self.fault == "commit_accepts_non_argmax" and j < S - 1 and drafts[r][j] != t:
                    t = drafts[r][j]
                em.append(t)
                if j + 1 < S and drafts[r][j] == t:
                    j += 1
                    continue
                break
            emitted.append(em)
        if S > 1 and kept is not None:
            self.ref.check_tokens(step, [e[0] for e in emitted[:len(firsts)]])
            self.ref.keep(kept)
        else:
            self.ref.check_spec(step, [drafts[r] for r in running], emitted)
        return emitted


def _serving_fault(monkeypatch, name, P):
    from atom_b200 import ops
    from atom_b200 import textgen
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import KvCacheInt4
    if name == "continuation_without_kv":             # the layer drops the cache from a prompt over a cached prefix
        f = ops.prefill_attention_i4
        monkeypatch.setattr(ops, "prefill_attention_i4", lambda *a, kv=None, layer_idx=None, **k: f(*a, **k))
    elif name == "verify_kv_at_stride_1":             # a verify step's K/V rows written one per sequence
        monkeypatch.setattr(BatchLenInfo, "decode_indptr", property(
            lambda self: None if self.decode_len == 1 else torch.arange(0, self.decode + 1, dtype=torch.int32)))
    elif name in ("truncate_keeps_one_more", "truncate_keeps_one_less"):
        f, d = KvCacheInt4.truncate, 1 if name.endswith("more") else -1
        monkeypatch.setattr(KvCacheInt4, "truncate", lambda self, n: f(self, min(n + d, self.seqlen)))
    elif name == "fork_shares_partial_page":          # the partly filled page shared instead of copied
        def fork(self, n=None):
            n = self.seqlen if n is None else n
            child = KvCacheInt4(self.pool, 0)
            for page in self.indicies[:-(-n // P)]:
                self.pool.share_block(page)
                child._pages.append(page)
            child._seqlen = n
            return child
        monkeypatch.setattr(KvCacheInt4, "fork", fork)
    elif name == "verify_rows_one_per_sequence":     # the logits of a verify step read at each sequence's first row only
        f = textgen.TextGenScheduler.last_token_rows

        def rows(self):
            b = self._blen
            r = f(self)
            return r[:len(r) - b.decode * b.decode_len] + [b.doff + i * b.decode_len for i in range(b.decode)]
        monkeypatch.setattr(textgen.TextGenScheduler, "last_token_rows", rows)
    elif name != "commit_accepts_non_argmax":        # (the driver's own acceptance)
        raise ValueError(name)


def _serve(monkeypatch, fault=None):
    """A root R of 13 tokens and the first chunk of X (30 tokens); X's second chunk (from position 11, off a 16-row boundary) with
    forks of R at 8 (aligned, pages shared) and 13 (its partly filled page copied) and their continuation prompts; a verify step
    (S = 4) with a new prompt Y, kept 4 / 1 (back across a page boundary) / 2 (inside a page); a verify step with greedy
    acceptance; a decode step; a verify step (S = 2) and a last decode step."""
    from atom_b200.kvcache import KvPoolInt4
    monkeypatch.setattr(torch.cuda.nvtx, "range_push", lambda *a: None)
    monkeypatch.setattr(torch.cuda.nvtx, "range_pop", lambda *a: None)
    model = _model(hidden=512, heads=4, kv_heads=2)
    impl = dict(ORACLE_OPS)
    if fault in KERNEL_FAULTS:
        impl.update([KERNEL_FAULTS[fault]])
    pool = KvPoolInt4(2, 2, 128, 40, P, torch.device("cpu"))
    pool.buf.random_(0, 256)
    pool.param.view(torch.int16).random_(-32768, 32767)
    d = Driver(monkeypatch, model, pool, R.model_ref(model, P), impl, fault,
               setup=lambda: fault and fault not in KERNEL_FAULTS and _serving_fault(monkeypatch, fault, P))
    d.step([("R", 13, None), ("X", 11, 30)])
    d.fork("F1", "R", 8, total=5)
    d.fork("F2", "R", total=6)
    d.step([("X", 19, None), ("F1", 5, None), ("F2", 6, None)])
    d.lens = [[d.kv[n].seqlen for n in ("X", "F1", "F2")]]
    d.step([("Y", 7, 7)], ["X", "F1", "F2"], S=4, kept=[4, 1, 2])
    d.lens.append([d.kv[n].seqlen for n in ("X", "F1", "F2", "Y")])
    d.step([], ["X", "F1", "F2", "Y"], S=3)
    d.step([("Z", 9, 9)], ["X", "F1", "F2", "Y"])
    d.step([], ["X", "F1", "F2", "Y", "Z"], S=2, kept=[2, 1, 2, 1, 2])
    d.step([], ["X", "F1", "F2", "Y", "Z"])
    return d


def test_reference_accepts_chunks_forks_and_verify_steps(monkeypatch):
    d = _serve(monkeypatch)
    ref = d.ref
    assert d.lens == [[31, 14, 20], [35, 15, 22, 8]]           # (+ the next token's slot)
    assert dict(ref.calls) == {"prefill": 3 * 2, "prefill over a cached prefix": 2, "verify": 3 * 2, "decode": 2 * 2}
    assert all(ref.ends[ref._end(kv.indicies, kv.seqlen - 1)][0] == kv.seqlen - 1 for n, kv in d.kv.items() if n != "R")


@pytest.mark.parametrize("fault,stage", [
    ("continuation_without_kv", r"layer 0 prefill_attention: prompts over a cached prefix, called without `kv`"),
    ("ctx_positions_from_zero_in_kernel", r"layer 0 prefill_attention: attention output outside the float64 bound"),
    ("verify_limit_off_by_one_in_kernel", r"layer 0 batch_verify: attention output outside the float64 bound"),
    ("verify_rotated_at_last_in_kernel", r"layer 0 batch_verify: attention output outside the float64 bound"),
    ("verify_kv_head_mod_in_kernel", r"layer 0 batch_verify: attention output outside the float64 bound"),
    ("verify_kv_at_stride_1", r"layer 0 init_kv \(verify\): `seqlen_indptr`"),
    ("truncate_keeps_one_more", r"page table: decode row 1: 18 positions .* continue a history of 15 tokens"),
    ("truncate_keeps_one_less", r"page table: decode row 0: 36 positions .* continue a history of 33 tokens"),
    ("fork_shares_partial_page", r"fork: the partly filled page \d+ is shared"),
    ("commit_accepts_non_argmax", r"speculative commit: row \d+: token \d+, the float64 argmax is"),
    ("verify_rows_one_per_sequence", r"last_token_rows"),
])
def test_reference_rejects_a_seeded_serving_fault(monkeypatch, fault, stage):
    with pytest.raises(R.WiringError, match=stage):
        _serve(monkeypatch, fault)


def test_check_spec_follows_the_greedy_acceptance_rule():
    """check_spec on synthetic float64 logits: two running sequences of S = 4 rows whose argmaxes are known; drafts accepted while
    they equal the argmax, the emitted count, the cut at the output length and at a stop id, and the lengths it keeps."""
    ref = R.ModelRef([types.SimpleNamespace(hkv=1)], 8)
    V, S = 16, 4
    want = [3, 5, 7, 9, 2, 4, 6, 8]                              # the argmax of rows 0 .. 7
    logits = np.zeros((8, V))
    logits[np.arange(8), want] = 10.0
    step = R.Step([], 2, decode_len=S, rows=list(range(8)), info={"logits64": logits, "bound": np.full((8, V), 1e-3)})
    ref._rows_step, ref._S = [([0, 1], 12, S, True), ([2], 6, S, True)], S
    kept = ref.check_spec(step, [[3, 5, 1], [4]], [[3, 5, 7], [2]])
    assert kept == [3, 1] and ref.ends[(1, 2)][0] == 11 and ref.ends[(2, 2)][0] == 3
    ref._rows_step = [([0, 1], 12, S, True), ([2], 6, S, True)]
    assert ref.check_spec(step, [[3, 5, 7], [2, 4]], [[3, 5, 7, 9], [2, 4, 6]], room=[2, 5], stop_ids={4}) == [2, 2]
    for drafts, emitted, msg in (([[3, 5, 1], [4]], [[3, 5], [2]], r"sequence 0: 2 tokens emitted, its accepted drafts call for 3"),
                                 ([[3, 5, 1], [4]], [[3, 5, 7, 9], [2]], r"sequence 0: 4 tokens emitted"),
                                 ([[3, 1, 1], [4]], [[3, 1, 1, 9], [2]], r"row 1: token 1, the float64 argmax is 5")):
        ref._rows_step = [([0, 1], 12, S, True), ([2], 6, S, True)]
        with pytest.raises(R.WiringError, match=msg):
            ref.check_spec(step, drafts, emitted)
