"""GPU suite (-m gpu): decoder-layer and model steps checked tensor by tensor against tests/layer_ref64.py -- prefill, mixed
prefill + decode and decode steps on multi-layer pools, both MLP paths on either side of the M = 64 switch, the Llama-7B shapes,
chunked prompts and continuations on forks, verify steps truncated and continued, and the serving loop's tokens with chunked
prefill, a shared prefix and speculative decoding.  Every kernel call of a step is recorded; the reference checks which call comes, what it was given and
what it returned, then audits the whole KV pool."""
import numpy as np
import pytest
import torch

from tests import layer_ref64 as R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True)
def fp32_lm_head_reduction():
    """lm_head is a torch FP16 GEMM: keep its split-K reductions in FP32, the arithmetic the logits bound counts."""
    old = torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
    yield
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = old


def _model(layers, hidden, inter, heads, kv_heads, theta, vocab=128, seed=11):
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(seed)
    torch.set_default_dtype(torch.float16)
    try:
        with DEV:
            model = LlamaForCausalLM(LlamaConfig(hidden_size=hidden, intermediate_size=inter, num_attention_heads=heads,
                                                 num_key_value_heads=kv_heads, num_hidden_layers=layers, vocab_size=vocab,
                                                 rope_theta=theta))
    finally:
        torch.set_default_dtype(torch.float32)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    for layer in model.model.layers:
        layer.fuse()
        for n in (layer.input_layernorm, layer.post_attention_layernorm):
            n.weight.data.uniform_(0.5, 1.5)
    return model.eval()


class Run:
    """Steps of `fn` (a model on token ids, or a layer on hidden states) over sequences of one pool, each checked by `ref`."""

    def __init__(self, monkeypatch, fn, ref, pool, ids=True):
        self.rec = R.Recorder().install(monkeypatch)
        self.fn, self.ref, self.pool, self.ids = fn, ref, pool, ids
        self.seqs, self.last = [], []
        self.rng = np.random.default_rng(0)

    def step(self, prompts, decode=True):
        """Prefill `prompts` and (decode=True) one token of every running sequence, in that batch order."""
        from atom_b200.cat_tensor import BatchLenInfo
        from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4
        running = self.seqs if decode else []
        for c in running:
            c.acquire_one()
        new = [KvCacheInt4(self.pool, n) for n in prompts]
        blen = BatchLenInfo(prompts, len(running), DEV)
        m = sum(prompts) + len(running)
        if self.ids:
            toks = sum((self.rng.integers(0, 128, n).tolist() for n in prompts), []) + list(self.last[:len(running)])
            inp = torch.tensor(toks, dtype=torch.long, device=DEV)
        else:
            inp = torch.from_numpy((self.rng.standard_normal((m, self.ref.layers[0].hidden)) * 0.5).astype(np.float16)).to(DEV)
        with torch.inference_mode():
            out, step, calls, before, after = R.run_step(self.rec, self.pool, self.fn, inp, blen,
                                                         BatchedKvCacheInt4(new) if new else None,
                                                         BatchedKvCacheInt4(running) if running else None, ids=self.ids)
        tokens = []
        if self.ref.lm_head is not None:
            step.rows = (np.cumsum(prompts) - 1).tolist() + list(range(sum(prompts), m))
            tokens = torch.argmax(out[0][step.rows], -1).tolist()
        self.ref.check_step(calls, step, before, after)
        if tokens:
            self.ref.check_tokens(step, tokens)
            self.last = tokens[len(prompts):] + tokens[:len(prompts)]
        self.seqs = running + new
        return step


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kv_heads,theta,P", [(4, 1e4, 16), (2, 5e5, 32), (1, 5e5, 16), (4, 5e5, 32), (2, 1e4, 16), (1, 1e4, 32)])
def test_two_layer_llama_prefill_mixed_and_decode_steps(monkeypatch, kv_heads, theta, P):
    """Prompts [5, 37, 16], then a mixed step (prompt [21] + the three), then 20 decode steps: lengths cross page boundaries."""
    from atom_b200.kvcache import KvPoolInt4
    model = _model(2, 512, 1024, 4, kv_heads, theta)
    pool = KvPoolInt4(2, kv_heads, 128, 24, P, DEV)
    pool.buf.random_(0, 256)
    pool.param.view(torch.int16).random_(-32768, 32767)
    run = Run(monkeypatch, model, R.model_ref(model, P), pool)
    run.step([5, 37, 16])
    run.step([21])
    for _ in range(20):
        run.step([])
    assert [c.seqlen for c in run.seqs] == [26, 58, 37, 41]


def _layer(hidden, inter, heads, kv_heads, theta=1e4, seed=5):
    from atom_b200.llama import LlamaConfig, LlamaDecoderLayer
    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=hidden, intermediate_size=inter, num_attention_heads=heads, num_key_value_heads=kv_heads,
                      num_hidden_layers=1, rope_theta=theta)
    layer = LlamaDecoderLayer(cfg, 0).to(DEV).init_random(seed)
    for n in (layer.input_layernorm, layer.post_attention_layernorm):
        n.weight.data.uniform_(0.5, 1.5)
    return layer.eval()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("batch", [64, 65])
def test_decode_batch_on_either_side_of_the_fused_mlp_switch(monkeypatch, batch):
    """A decode batch of 64 runs the fused gate/up launch and split-K GEMMs, 65 the separate gate and up GEMMs + activate."""
    from atom_b200.kvcache import KvPoolInt4
    layer = _layer(512, 1024, 4, 2)
    P = 16
    pool = KvPoolInt4(1, 2, 128, batch * 2 + 4, P, DEV)
    pool.buf.random_(0, 256)
    run = Run(monkeypatch, layer, R.ModelRef([R.LayerParams(layer, 0)], P), pool, ids=False)
    lens = [1 + (7 * i) % 23 for i in range(batch)]
    run.step(lens[:40])
    run.step(lens[40:])                     # mixed: 40 decode rows, M = 40 + sum(...) > 64
    run.step([])
    run.step([])


@pytest.mark.timeout(600)
def test_mixed_step_over_64_rows_with_a_small_decode_part(monkeypatch):
    """M = 70 (unfused MLP, un-split GEMMs) while the decode part is 30 rows; a prefill + decode boundary at a row that is not a
    multiple of 16 (the pair-shared weight-scale column depends on the row mod 16)."""
    from atom_b200.kvcache import KvPoolInt4
    layer = _layer(512, 1024, 4, 1, theta=5e5)
    P = 16
    pool = KvPoolInt4(1, 1, 128, 48, P, DEV)
    pool.buf.random_(0, 256)
    run = Run(monkeypatch, layer, R.ModelRef([R.LayerParams(layer, 0)], P), pool, ids=False)
    run.step([3] * 30)
    step = run.step([40])
    assert step.prefills == [40] and step.decode == 30


@pytest.mark.timeout(900)
def test_llama_7b_layer_prefill_then_decode(monkeypatch):
    """The real dispatch shapes (4096 / 11008 / 32 heads): split-K o_proj and down at decode, fused gate/up at 11008.  Prompts
    [300, 17], then two decode steps; the oracle GEMMs run on row subsets."""
    from atom_b200.kvcache import KvPoolInt4
    layer = _layer(4096, 11008, 32, 32)
    P = 16
    pool = KvPoolInt4(1, 32, 128, 26, P, DEV)
    pool.buf.random_(0, 256)
    ref = R.ModelRef([R.LayerParams(layer, 0)], P, prefill_rows={0: [0, 1, 15, 16, 150, 299], 1: [0, 8, 16]})
    run = Run(monkeypatch, layer, ref, pool, ids=False)
    run.step([300, 17])
    run.step([])
    run.step([])


def _mixtral_layer(cfg, seed=7):
    from atom_b200.mixtral import MixtralDecoderLayer
    torch.manual_seed(seed)
    layer = MixtralDecoderLayer(cfg, 0).to(DEV).init_random(seed)
    for n in (layer.input_layernorm, layer.post_attention_layernorm):
        n.weight.data.uniform_(0.5, 1.5)
    return layer.eval()


@pytest.mark.timeout(600)
def test_mixtral_layer_prefill_mixed_and_decode_steps(monkeypatch):
    """Toy Mixtral layer (512 / 1024, 4 experts, top-2, 4 query and 2 KV heads, base 1e6): routing against the float64 top-k,
    plan, gather, grouped gate/up and down per (token, expert), and the combine, through prefill, mixed and decode steps."""
    from atom_b200.kvcache import KvPoolInt4
    from atom_b200.mixtral import MixtralConfig
    cfg = MixtralConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=1,
                        num_local_experts=4, num_experts_per_tok=2, rope_theta=1e6)
    layer = _mixtral_layer(cfg)
    P = 16
    pool = KvPoolInt4(1, 2, 128, 24, P, DEV)
    pool.buf.random_(0, 256)
    run = Run(monkeypatch, layer, R.ModelRef([R.LayerParams(layer, 0)], P), pool, ids=False)
    run.step([5, 37, 16])
    run.step([21])
    for _ in range(4):
        run.step([])


@pytest.mark.timeout(900)
def test_mixtral_8x7b_layer_decode_step(monkeypatch):
    """One decode step at the real MixtralConfig() shape (4096 / 14336, 8 experts, top-2, 32 / 8 heads), after a short prefill."""
    from atom_b200.kvcache import KvPoolInt4
    from atom_b200.mixtral import MixtralConfig
    layer = _mixtral_layer(MixtralConfig(num_hidden_layers=1))
    P = 16
    pool = KvPoolInt4(1, 8, 128, 8, P, DEV)
    pool.buf.random_(0, 256)
    run = Run(monkeypatch, layer, R.ModelRef([R.LayerParams(layer, 0)], P), pool, ids=False)
    run.step([5, 3, 9])
    step = run.step([])
    assert step.decode == 3


@pytest.mark.timeout(900)
def test_serving_loop_tokens_follow_the_float64_logits(monkeypatch):
    """run_textgen on the model of test_z_textgen_gpu.py: every step of the loop is checked (prefill, mixed and decode batches as
    the scheduler forms them), the logits are read at the scheduler's last_token_rows, and every emitted token is the argmax of
    the float64 logits wherever the top-2 gap exceeds twice the bound."""
    from atom_b200 import textgen as tg
    _, steps, _ = _serving_run(monkeypatch, tg.TextGenConfig(3))
    assert any(p and d for p, d, _ in steps), "the loop made no mixed step"


@pytest.mark.timeout(300)
def test_graphed_decode_step_equals_its_eager_replay():
    """One decode step replayed from DecodeGraphRunner's CUDA graph gives the logits and the pool of the same step run eagerly on a
    copy of the pool, bit for bit."""
    from atom_b200 import textgen as tg
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    model = _model(2, 512, 1024, 4, 2, 5e5)
    pool = KvPoolInt4(2, 2, 128, 16, 16, DEV)
    pool.buf.random_(0, 256)
    pool.param.uniform_(0.01, 0.05)
    seqs = [KvCacheInt4(pool, n) for n in (16, 9, 40)]
    for c in seqs:
        c.acquire_one()
    logits = {}

    def keep(ids, blen, prefill_kv, decode_kv):
        logits["graph"], h = model(ids, blen, prefill_kv, decode_kv)
        return logits["graph"], h

    buf, param = pool.buf.clone(), pool.param.clone()
    toks = [3, 77, 101]
    with torch.inference_mode():
        runner = tg.DecodeGraphRunner(keep, pool, DEV, max_pages_per_seq=4)
        runner.run(toks, seqs)
        graphed = logits["graph"].clone()
        graphed_pool = (pool.buf.clone(), pool.param.clone())
        pool.buf.copy_(buf)
        pool.param.copy_(param)
        eager, _ = model(torch.tensor(toks, device=DEV), BatchLenInfo([], 3, DEV), None, BatchedKvCacheInt4(seqs))
    assert torch.equal(graphed, eager)
    assert torch.equal(graphed_pool[0], pool.buf) and torch.equal(graphed_pool[1].view(torch.int16), pool.param.view(torch.int16))


# ------------------------------------------------------------------------------------------------ chunks, forks, verify steps
def _driver(monkeypatch, fn, pool, ref, ids=True):
    from tests.test_layer_ref64_cpu import Driver
    return Driver(monkeypatch, fn, pool, ref, ids=ids, vocab=128)


def _pool(layers, kv_heads, pages, P):
    from atom_b200.kvcache import KvPoolInt4
    pool = KvPoolInt4(layers, kv_heads, 128, pages, P, DEV)
    pool.buf.random_(0, 256)
    pool.param.view(torch.int16).random_(-32768, 32767)
    return pool


def _worst(ref):
    """The largest error-to-bound ratio of each attention kind the reference checked (printed for the record, -s)."""
    print({k: round(v, 4) for k, v in sorted(ref.worst.items())}, dict(ref.calls))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kv_heads,P", [(1, 16), (2, 32), (4, 16), (4, 32)])
def test_chunked_prefill_and_continuations_on_forks(monkeypatch, kv_heads, P):
    """Two-layer model: a root prefilled in two chunks (the second from position 21), a prompt chunked beside decode rows, forks of
    the root at an aligned and an unaligned length with continuation prompts, then decode steps over the forks' shared pages."""
    model = _model(2, 512, 1024, 4, kv_heads, 5e5 if P == 32 else 1e4)
    pool = _pool(2, kv_heads, 40, P)
    d = _driver(monkeypatch, model, pool, R.model_ref(model, P))
    d.step([("R", 21, None), ("A", 16, 16)])
    d.step([("R", 29, None), ("B", 19, 60)], ["A"])          # R from 21, B's first chunk: mixed with a decode row
    d.fork("F1", "R", P, total=9)                             # aligned: shares the first page
    d.fork("F2", "R", total=P + 3)                            # at 50: its partly filled page copied
    d.step([("B", 41, None), ("F1", 9, 9), ("F2", P + 3, P + 3)], ["A"])
    for _ in range(P // 2 + 2):
        d.step([], ["A", "B", "F1", "F2"])
    assert d.ref.calls["prefill over a cached prefix"] == 2 * 2 and d.ref.calls["decode"] == 2 * (P // 2 + 4)
    _worst(d.ref)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kv_heads", [2, 4])
def test_verify_steps_with_prompt_chunks_truncated_and_continued(monkeypatch, kv_heads):
    """Two-layer model, GQA (2 KV heads) or MHA (4): verify steps of S = 4, 8 and 2 rows per sequence beside prompt chunks,
    truncated to kept counts from 1 to S (back across page boundaries and inside pages), a verify step with greedy acceptance
    of the drafts, and decode steps between them."""
    model = _model(2, 512, 1024, 4, kv_heads, 5e5)
    P = 16
    pool = _pool(2, kv_heads, 48, P)
    d = _driver(monkeypatch, model, pool, R.model_ref(model, P))
    d.step([("A", 13, 13), ("B", 30, 30), ("C", 17, 40)])
    d.step([("C", 23, None)], ["A", "B"], S=4, kept=[4, 1])
    d.step([("D", 5, 5)], ["A", "B", "C"], S=8, kept=[3, 8, 1])
    d.step([], ["A", "B", "C", "D"], S=2, kept=[2, 1, 2, 1])
    d.step([], ["A", "B", "C", "D"])
    d.step([], ["A", "B", "C", "D"], S=4)
    d.step([("E", 9, 9)], ["A", "B", "C", "D"], S=8, kept=[8, 5, 2, 7])
    d.step([], ["A", "B", "C", "D", "E"])
    assert d.ref.calls["verify"] == 2 * 5
    _worst(d.ref)


@pytest.mark.timeout(900)
def test_mixtral_layer_verify_steps(monkeypatch):
    """Toy Mixtral layer (512 / 1024, 4 experts, top-2, 4 query and 2 KV heads): the MoE block on batches of S-row verify steps
    beside prompt chunks, truncated and continued."""
    from atom_b200.mixtral import MixtralConfig
    cfg = MixtralConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=1,
                        num_local_experts=4, num_experts_per_tok=2, rope_theta=1e6)
    layer = _mixtral_layer(cfg)
    P = 16
    pool = _pool(1, 2, 24, P)
    d = _driver(monkeypatch, layer, pool, R.ModelRef([R.LayerParams(layer, 0)], P), ids=False)
    d.step([("A", 5, 5), ("B", 20, 37)])
    d.step([("B", 17, None)], ["A"], S=4, kept=[2])
    d.step([("C", 9, 9)], ["A", "B"], S=8, kept=[8, 3])
    d.step([], ["A", "B", "C"], S=2, kept=[1, 2, 2])
    d.step([], ["A", "B", "C"])
    assert d.ref.calls["verify"] == 3
    _worst(d.ref)


def _serving_run(monkeypatch, cfg, maxlen=72):
    """run_textgen, eager, on the model of test_z_textgen_gpu.py with every step checked and every emitted token held to the
    float64 logits (check_tokens, or check_spec under speculation, which also sets the lengths the truncations must leave)."""
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvCacheInt4, KvPoolInt4
    model = _model(2, 512, 1024, 4, None, 1e4)
    P = 16
    K = 0 if cfg.speculate is None else cfg.speculate.num_draft
    pool = KvPoolInt4(2, 4, 128, tg.pool_capacity(3, maxlen + cfg.shared_prefix, P, K) + 8, P, DEV)
    ref = R.model_ref(model, P, sm_count=torch.cuda.get_device_properties(DEV).multi_processor_count)
    rec = R.Recorder().install(monkeypatch)
    pending, steps = {}, []
    fork = KvCacheInt4.fork

    def forked(kv, n=None):
        child = fork(kv, n)
        ref.fork(list(kv.indicies), child.seqlen, list(child.indicies))
        return child
    monkeypatch.setattr(KvCacheInt4, "fork", forked)

    class Wrapped:
        lm_head = model.lm_head             # the scheduler draws prompt ids below lm_head.out_features

        def __call__(self, ids, blen, prefill_kv, decode_kv):
            out, pending["step"], pending["calls"], pending["before"], pending["after"] = R.run_step(rec, pool, model, ids, blen,
                                                                                                    prefill_kv, decode_kv)
            return out

    rows_of, commit, commit_spec = tg.TextGenScheduler.last_token_rows, tg.TextGenScheduler.commit, tg.TextGenScheduler.commit_spec

    def last_token_rows(self):
        pending["step"].rows = rows_of(self)
        return pending["step"].rows

    def checked(self):
        s = pending.pop("step")
        ref.check_step(pending["calls"], s, pending["before"], pending["after"])
        steps.append((s.prefills, s.decode, s.decode_len))
        return s

    def checked_commit(self, next_tokens, t1, t2, *a, **k):
        if k.get("_speculative"):
            return commit(self, next_tokens, t1, t2, *a, **k)
        ref.check_tokens(checked(self), next_tokens)
        return commit(self, next_tokens, t1, t2, *a, **k)

    def checked_commit_spec(self, out, t1, t2, logprobs=None):
        s = checked(self)
        out = np.asarray(out)
        room = [int(self.rs.output_lens[r.req_idx]) - len(r.output) for r in self.workset]
        ref.check_spec(s, [list(r.drafts) for r in self.workset], [o[2:2 + int(o[0])].tolist() for o in out], room, self.stop_token_ids)
        return commit_spec(self, out, t1, t2, logprobs)

    monkeypatch.setattr(tg.TextGenScheduler, "last_token_rows", last_token_rows)
    monkeypatch.setattr(tg.TextGenScheduler, "commit", checked_commit)
    monkeypatch.setattr(tg.TextGenScheduler, "commit_spec", checked_commit_spec)
    rs = tg.generate_request_set(7, maxlen)
    res = tg.run_textgen(Wrapped(), rs, cfg, pool, DEV, sync=torch.cuda.synchronize, keep_tokens=True)
    assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
    assert pool.num_free_blocks == pool.capacity                # every page given back, truncations included
    _worst(ref)
    return res, steps, ref


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("kind", ["chunked", "shared_prefix", "speculative", "all"])
def test_serving_loop_variants_follow_the_float64_logits(monkeypatch, kind):
    """The serving loop with chunked prefill (16 tokens a step), a 70-token shared prefix forked for every request (24-token
    chunks), speculative decoding (4 drafts of 1- to 3-grams), and all three together: every step checked, every emitted token
    the float64 argmax wherever the top-2 gap is clear, and under speculation the drafts accepted exactly when they are it."""
    from atom_b200 import textgen as tg
    spec = tg.SpeculativeParams(4, 3, 1) if kind in ("speculative", "all") else None
    chunk = {"chunked": 16, "shared_prefix": 24, "all": 16}.get(kind)
    shared = 70 if kind in ("shared_prefix", "all") else 0
    res, steps, ref = _serving_run(monkeypatch, tg.TextGenConfig(3, prefill_chunk=chunk, shared_prefix=shared, speculate=spec))
    if chunk:
        assert ref.calls["prefill over a cached prefix"] > 0
    if spec is not None:
        st = res.speculative
        assert any(S > 1 for _, _, S in steps) and ref.calls["verify"] > 0
        assert 0 < st["accepted_tokens"] < st["drafted_tokens"], st          # drafts both accepted and rejected
