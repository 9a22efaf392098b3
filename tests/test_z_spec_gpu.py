"""GPU suite (-m gpu): speculative decoding's kernels and serving path -- the draft sampler (ops.sample_tokens(drafts=)) against
tests/spec_ref.py outside the ambiguity regions and bit for bit against the plain sampler on rows without a candidate; the
commit and proposal kernel (ops.spec_commit_propose) bit for bit against the numpy reference; CUDA-graph replays with new
drafts; and the serving harness with a stand-in model and with small random INT4 Llamas (GQA 32:8 and MHA)."""
import numpy as np
import pytest
import torch

from tests import sample_penalty_ref64 as RP
from tests import sample_ref64 as R
from tests import spec_ref as SR

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _logits(b, v, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((b, v), generator=g) * 2.5
    x[:, :3] += 6                                   # a few strong tokens: drafts are accepted often enough to matter
    return x.half()


def _params(b, seed):
    rng = np.random.default_rng(seed)
    T = rng.choice([0.0, 0.6, 1.0, 1.3], b).astype(np.float32)
    K = rng.choice([0, 1, 40, 1000], b).astype(np.int32)
    P = rng.choice([1.0, 0.9, 0.6], b).astype(np.float32)
    M = rng.choice([0.0, 0.0, 0.02], b).astype(np.float32)
    keys = [(int(rng.integers(0, 2 ** 63)), int(i)) for i in range(b)]
    ctrs = [int(rng.integers(0, 2 ** 40)) for _ in range(b)]
    return T, K, P, M, keys, ctrs


def _drafts(l16, b, v, seed):
    """Per row: none, the argmax, the runner-up, a random token."""
    rng = np.random.default_rng(seed + 1)
    order = np.argsort(-l16.astype(np.float32), axis=1, kind="stable")
    kind = rng.integers(0, 4, b)
    d = np.where(kind == 0, -1, np.where(kind == 1, order[:, 0], np.where(kind == 2, order[:, 1], rng.integers(0, v, b))))
    return d.astype(np.int32)


@pytest.mark.parametrize("V", [32000, 128256])
def test_draft_sampler_matches_the_reference_outside_ambiguity(V):
    from atom_b200 import ops
    B, amb, checked, accepted = 48, 0, 0, 0
    for seed in range(4):
        x = _logits(B, V, seed)
        T, K, P, M, keys, ctrs = _params(B, seed)
        l16 = x.numpy()
        d = _drafts(l16, B, V, seed)
        tok, lp, ids, lps = [t.cpu().numpy() for t in ops.sample_tokens(x.to(DEV), T, K, P, keys, ctrs, min_p=M, logprobs=4,
                                                                          drafts=d.tolist())]
        ref = SR.sample_draft_np(l16, T, K, P, keys, ctrs, d, min_p=M)
        plain = [t.cpu().numpy() for t in ops.sample_tokens(x.to(DEV), T, K, P, keys, ctrs, min_p=M, logprobs=4)]
        for i in range(B):
            if SR.draft_ambiguous(l16[i], float(T[i]), int(K[i]), np.float32(P[i]), keys[i], ctrs[i], int(d[i]), float(M[i])):
                amb += 1
                continue
            checked += 1
            assert tok[i] == ref[i], (i, T[i], K[i], P[i], M[i], d[i], tok[i], ref[i])
            accepted += int(d[i] >= 0 and tok[i] == d[i])
            # the top-n list does not depend on the draw; the logprob is the emitted token's
            assert np.array_equal(ids[i], plain[2][i]) and np.array_equal(lps[i].view(np.int32), plain[3][i].view(np.int32))
            want = RP._logprobs_row(l16[i], int(tok[i]), 4, ())[0]
            assert abs(float(lp[i]) - float(want)) <= 1e-5 + 1e-6 * abs(float(want)), (i, lp[i], want)
    assert checked >= 0.9 * (checked + amb) and accepted > 10


def test_rows_without_a_candidate_are_the_plain_sampler_bit_for_bit():
    from atom_b200 import ops
    B, V = 64, 50257
    x = _logits(B, V, 9).to(DEV)
    T, K, P, M, keys, ctrs = _params(B, 9)
    for opts in ({}, {"min_p": M}, {"logprobs": 6}, {"min_p": M, "logprobs": 0}):
        a = ops.sample_tokens(x, T, K, P, keys, ctrs, drafts=[-1] * B, **opts)
        b = ops.sample_tokens(x, T, K, P, keys, ctrs, **opts)
        a, b = (a, b) if isinstance(a, tuple) else ((a,), (b,))
        for u, w in zip(a, b):
            assert torch.equal(u.view(torch.int32) if u.dtype == torch.float32 else u,
                               w.view(torch.int32) if w.dtype == torch.float32 else w)


def test_out_of_range_drafts_give_minus_one_and_greedy_ignores_the_draft():
    from atom_b200 import ops
    B, V = 8, 32000
    x = _logits(B, V, 3).to(DEV)
    d = torch.tensor([-2, V, V + 5, -100, 0, 1, 2, -1], dtype=torch.int32, device=DEV)
    tok = ops.sample_tokens(x, 0.7, 0, 1.0, [(1, i) for i in range(B)], list(range(B)), drafts=d).cpu().numpy()
    assert (tok[:4] == -1).all() and (tok[4:] >= 0).all()
    with pytest.raises(RuntimeError):
        ops.sample_tokens(x, 0.7, 0, 1.0, [(1, i) for i in range(B)], list(range(B)), drafts=[V] * B)
    am = torch.argmax(x, dim=-1).cpu().numpy()
    for dd in ([-1] * B, am.tolist(), ((am + 1) % V).tolist()):
        g = ops.sample_tokens(x, 0.0, 0, 1.0, [(1, i) for i in range(B)], list(range(B)), drafts=dd).cpu().numpy()
        assert np.array_equal(g, am)


def test_a_captured_draft_sampler_replays_with_new_drafts():
    from atom_b200 import ops
    B, V = 16, 32000
    x = _logits(B, V, 5).to(DEV)
    T = torch.full((B,), 0.9, device=DEV)
    K = torch.zeros(B, dtype=torch.int32, device=DEV)
    P = torch.full((B,), 0.95, device=DEV)
    keys = torch.tensor([[7, i] for i in range(B)], dtype=torch.int64, device=DEV)
    ctr = torch.zeros(B, dtype=torch.int64, device=DEV)
    d = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.sample_tokens(x, T, K, P, keys, ctr, drafts=d)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = ops.sample_tokens(x, T, K, P, keys, ctr, drafts=d)
    torch.cuda.current_stream().wait_stream(s)
    rng = np.random.default_rng(0)
    for step in range(6):
        d.copy_(torch.from_numpy(rng.integers(-1, 4, B).astype(np.int32)))
        ctr.fill_(step)
        g.replay()
        want = ops.sample_tokens(x, T, K, P, keys, ctr, drafts=d)
        assert torch.equal(out, want)


@pytest.mark.parametrize("nmin,nmax", [(1, 1), (1, 3), (2, 4), (3, 16)])
def test_commit_propose_matches_the_reference(nmin, nmax):
    from atom_b200 import ops
    rng = np.random.default_rng(nmin * 31 + nmax)
    for k in range(1, 8):
        nslots, cap, B = 12, 300, 9
        hist = np.zeros((nslots, cap), np.int32)
        lens = rng.integers(0, cap, nslots).astype(np.int32)
        lens[:2] = cap                              # full slots: nothing more is written
        lens[2] = cap - 2
        lens[3] = 0
        for s_ in range(nslots):
            hist[s_, :lens[s_]] = rng.integers(0, 5, lens[s_])     # a small alphabet: many matches, ties to the latest
        slots = rng.permutation(nslots)[:B].astype(np.int32)
        S = int(rng.integers(1, k + 2))
        rows = np.concatenate([[0], np.cumsum(rng.choice([1, S], B))]).astype(np.int32)
        R_ = int(rows[-1])
        cands = rng.integers(-1, 5, R_).astype(np.int32)
        for i in range(B):                         # the last row of a sequence has no candidate
            cands[rows[i + 1] - 1] = -1
        tokens = np.where(rng.random(R_) < 0.7, cands, rng.integers(0, 5, R_)).astype(np.int32)
        out = torch.zeros((B, 2 * k + 3), dtype=torch.int32, device=DEV)
        h_d, l_d = torch.from_numpy(hist.copy()).to(DEV), torch.from_numpy(lens.copy()).to(DEV)
        t = lambda a: torch.from_numpy(a).to(DEV)     # noqa: E731
        ops.spec_commit_propose(t(tokens), t(cands), t(rows), t(slots), h_d, l_d, out, k, nmin, nmax)
        ref_out = np.zeros((B, 2 * k + 3), np.int32)
        SR.commit_propose_np(tokens, cands, rows, slots, hist, lens, ref_out, k, nmin, nmax)
        assert np.array_equal(out.cpu().numpy(), ref_out), k
        assert np.array_equal(h_d.cpu().numpy(), hist) and np.array_equal(l_d.cpu().numpy(), lens)


def test_commit_propose_rejects_bad_arguments_on_the_host():
    from atom_b200 import ops
    h, lens = ops.spec_history(4, 16, DEV)
    i32 = lambda a: torch.tensor(a, dtype=torch.int32, device=DEV)     # noqa: E731
    out = torch.zeros((1, 2 * 4 + 3), dtype=torch.int32, device=DEV)
    args = (i32([1]), i32([-1]), i32([0, 1]))
    for bad in (dict(slots=[4]), dict(slots=[-1]), dict(k=8), dict(k=0), dict(nmin=0), dict(nmin=3, nmax=2), dict(nmax=17)):
        a = dict(slots=[0], k=4, nmin=1, nmax=3)
        a.update(bad)
        o = out if a["k"] == 4 else torch.zeros((1, 2 * a["k"] + 3), dtype=torch.int32, device=DEV)
        with pytest.raises(RuntimeError):
            ops.spec_commit_propose(*args, a["slots"], h, lens, o, a["k"], a["nmin"], a["nmax"])
    with pytest.raises(RuntimeError):
        ops.spec_commit_propose(*args, [0], h[:, :3].contiguous(), lens, out, 4, 1, 3)     # cap < k + 1


class _CycleLM:
    """The CPU suite's stand-in model on the device: FP16 logits whose argmax continues t with (t % 5) + 1."""
    config = type("Config", (), {"vocab_size": 97})

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        nxt = ids.long() % 5 + 1
        x = torch.sin(ids.float()[:, None] * 0.3 + torch.arange(97, device=ids.device, dtype=torch.float32)[None])
        return (x + 4 * torch.nn.functional.one_hot(nxt, 97).float()).half(), None


def test_harness_with_a_stand_in_model_gives_the_greedy_tokens_graphed_and_eager():
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvPoolInt4
    rs = tg.generate_request_set(10, 80)
    toks = {}
    for spec in (None, tg.SpeculativeParams(num_draft=4)):
        for graphs in (False, True):
            for shared in (0, 24):
                pool = KvPoolInt4(1, 2, 128, tg.pool_capacity(4, 80 + shared, 16) + 8, 16, DEV)
                cfg = tg.TextGenConfig(4, prefill_chunk=11, shared_prefix=shared, speculate=spec)
                runner = tg.DecodeGraphRunner(_CycleLM(), pool, DEV, max_pages_per_seq=(80 + shared) // 16 + 2,
                                              speculate=spec) if graphs else None
                res = tg.run_textgen(_CycleLM(), rs, cfg, pool, DEV, keep_tokens=True, decode_runner=runner)
                assert pool.num_free_blocks == pool.capacity
                if spec is not None:
                    assert res.speculative["verify_steps"] > 0 and res.speculative["accepted_tokens"] > 0
                toks[(spec is None, graphs, shared)] = res.tokens
    for graphs in (False, True):
        for shared in (0, 24):
            assert toks[(False, graphs, shared)] == toks[(True, False, shared)]


class _Recorder(torch.nn.Module):
    """Wraps the model: keeps every eager step's logits so each emitted token can be traced to its row."""

    def __init__(self, model):
        super().__init__()
        self.model, self.steps = model, []
        self.lm_head = model.lm_head

    def forward(self, ids, blen, prefill_kv, decode_kv):
        logits, h = self.model(ids, blen, prefill_kv, decode_kv)
        if not torch.cuda.is_current_stream_capturing():
            self.steps.append(logits.float().cpu())
        return logits, h


def _llama(heads, kv_heads):
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(21)
    torch.set_default_dtype(torch.float16)
    try:
        with DEV:
            model = LlamaForCausalLM(LlamaConfig(hidden_size=128 * heads, intermediate_size=2048, num_attention_heads=heads,
                                                 num_key_value_heads=kv_heads, num_hidden_layers=2, vocab_size=256))
    finally:
        torch.set_default_dtype(torch.float32)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    return model.eval()


def _harness(model, kv_heads, graphs, sampling, chunk, shared, spec, propose_op=None):
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvPoolInt4
    rs = tg.generate_request_set(8, 96)
    pool = KvPoolInt4(2, kv_heads, 128, tg.pool_capacity(4, 96 + shared, 16) + 8, 16, DEV)
    cfg = tg.TextGenConfig(4, prefill_chunk=chunk, shared_prefix=shared, sampling=sampling, speculate=spec)
    runner = tg.DecodeGraphRunner(model, pool, DEV, max_pages_per_seq=(96 + shared) // 16 + 2, sampling=sampling,
                                  speculate=spec) if graphs else None
    res = tg.run_textgen(model, rs, cfg, pool, DEV, sync=torch.cuda.synchronize, keep_tokens=True, decode_runner=runner,
                         propose_op=propose_op)
    assert pool.num_free_blocks == pool.capacity
    assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
    return res


@pytest.mark.timeout(900)
@pytest.mark.parametrize("heads,kv_heads", [(32, 8), (8, 8)])
def test_small_llama_speculative_serving(heads, kv_heads, monkeypatch):
    from atom_b200 import ops
    from atom_b200 import textgen as tg
    model = _llama(heads, kv_heads)
    spec = tg.SpeculativeParams(num_draft=4, ngram_max=3, ngram_min=1)
    # every emitted token is the argmax of the logits row that produced it: eager steps, each step's logits recorded, and the
    # commit's output traced to the step's rows through the scheduler's last_token_rows() and sequence_rows()
    scheds = []

    class _Sched(tg.TextGenScheduler):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            scheds.append(self)

    monkeypatch.setattr(tg, "TextGenScheduler", _Sched)
    rec = _Recorder(model)
    checked = {"tokens": 0, "drafts": 0}

    def propose(tokens, cands, row_indptr, slots, history, lengths, out, k, nmin, nmax):
        ops.spec_commit_propose(tokens, cands, row_indptr, slots, history, lengths, out, k, nmin, nmax)
        sched, logits = scheds[-1], rec.steps[-1]
        rows, seq, o = sched.last_token_rows(), sched.sequence_rows(), out.cpu().numpy()
        assert seq == row_indptr.cpu().tolist()
        for i in range(len(seq) - 1):
            for j in range(int(o[i, 0])):
                assert int(o[i, 2 + j]) == int(torch.argmax(logits[rows[seq[i] + j]])), (i, j)
                checked["tokens"] += 1
                checked["drafts"] += j > 0
        return out

    res = _harness(rec, kv_heads, False, None, 13, 24, spec, propose_op=propose)
    assert res.speculative["verify_steps"] > 0 and checked["drafts"] > 0
    assert checked["tokens"] >= int(res.output_lens.sum())
    # graphed and eager agree bit for bit, greedy and sampled, with chunked prefill and shared prefixes mixing verify rows in
    for sampling in (None, tg.SamplingParams(0.8, top_p=0.95, seed=4)):
        for chunk, shared in ((None, 0), (13, 24)):
            a = _harness(model, kv_heads, False, sampling, chunk, shared, spec)
            b = _harness(model, kv_heads, True, sampling, chunk, shared, spec)
            assert a.tokens == b.tokens and a.speculative == b.speculative
            assert b.graphed_steps > 0 and a.speculative["verify_steps"] > 0
