"""GPU suite (-m gpu): beam search in the serving harness on 2-layer random INT4 Llamas (GQA 32:8 and MHA, pages of 16 and 32
tokens) -- width 1 gives the greedy tokens eagerly and from CUDA graphs, graphed and eager beam runs agree bit for bit, and every
eager step's beam decisions equal tests/beam_ref.py's on the logits rows that step produced, merged with the sampler's own
log-probabilities."""
import numpy as np
import pytest
import torch

from tests import beam_ref as BR

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


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


def _run(model, kv_heads, P, beam, graphs, chunk=None, shared=0, stops=(), beam_select_op=None):
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvPoolInt4
    rs = tg.generate_request_set(8, 64)
    bs = 8
    pool = KvPoolInt4(2, kv_heads, 128, tg.pool_capacity(bs, 64 + shared, P), P, DEV)
    cfg = tg.TextGenConfig(bs, prefill_chunk=chunk, shared_prefix=shared, stop_token_ids=stops, beam=beam)
    runner = tg.DecodeGraphRunner(model, pool, DEV, max_pages_per_seq=(64 + shared) // P + 2, beam=beam,
                                  stop_token_ids=stops) if graphs else None
    res = tg.run_textgen(model, rs, cfg, pool, DEV, sync=torch.cuda.synchronize, keep_tokens=True, decode_runner=runner,
                         beam_select_op=beam_select_op)
    assert pool.num_free_blocks == pool.capacity
    if graphs:
        assert res.graphed_steps > 0
    return res, tg.report(rs, cfg, res)


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("heads,kv_heads,P", [(32, 8, 16), (8, 8, 32)])
def test_width_one_is_greedy_and_graphs_match_eager(heads, kv_heads, P):
    from atom_b200 import textgen as tg
    model = _llama(heads, kv_heads)
    greedy, _ = _run(model, kv_heads, P, None, False)
    for graphs in (False, True):
        one, _ = _run(model, kv_heads, P, tg.BeamSearchParams(1), graphs)
        assert one.tokens == greedy.tokens
    beam = tg.BeamSearchParams(4, 0.8)
    a, ra = _run(model, kv_heads, P, beam, False)
    b, rb = _run(model, kv_heads, P, beam, True)
    assert a.tokens == b.tokens and np.array_equal(a.beam_scores, b.beam_scores)
    assert ra["beam"]["page_copies"] == rb["beam"]["page_copies"] > 0
    print(f"H={heads} KV={kv_heads} P={P}: W=4 {ra['beam']['page_copies']} page copies, {rb['graphed_decode_steps']} graphed steps")


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("width", [2, 4])
def test_every_step_matches_the_reference(width):
    from atom_b200 import ops
    from atom_b200 import textgen as tg
    model = _llama(32, 8)
    steps = {"n": 0}

    def checked(logits, row_indptr, sums, w, stop_ids=(), out=None, workspace=None):
        res = ops.beam_select(logits, row_indptr, sums, w, stop_ids, out=out, workspace=workspace)
        R = logits.shape[0]
        _, _, ids, lps = ops.sample_tokens(logits.contiguous(), [0.0] * R, [0] * R, [1.0] * R, [(0, r) for r in range(R)], [0] * R,
                                           logprobs=ops.SAMPLE_TOP_N_MAX)
        ids, lps = ids.cpu().numpy(), lps.cpu().numpy()
        lp_rows = [{int(t): lps[r, j] for j, t in enumerate(ids[r]) if t >= 0} for r in range(R)]
        want = BR.beam_select_np(logits.cpu().numpy(), row_indptr.cpu().numpy(), sums.cpu().numpy(), w, stop_ids, lp_rows=lp_rows)
        for got, exp in zip(res, want):
            assert np.array_equal(got.cpu().numpy().view(np.int32), exp.view(np.int32))
        steps["n"] += 1
        return res

    res, rep = _run(model, 8, 16, tg.BeamSearchParams(width, 1.0), False, chunk=24, shared=20, stops=(5, 77),
                    beam_select_op=checked)
    assert steps["n"] > 0 and rep["beam"]["page_copies"] > 0
    print(f"W={width}: {steps['n']} steps checked, {rep['beam']['page_copies']} page copies, "
          f"{rep['beam']['stop_finished_requests']} requests ended on a stop id")


@pytest.fixture
def fp32_lm_head_reduction():
    """lm_head is a torch FP16 GEMM: keep its split-K reductions in FP32, the arithmetic the logits bound counts."""
    old = torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
    yield
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = old


def _ref_model(kv_heads):
    """The two-layer model of tests/test_z_layer_ref64_gpu.py (fused layers, perturbed norms), 4 query heads."""
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(11)
    torch.set_default_dtype(torch.float16)
    try:
        with DEV:
            model = LlamaForCausalLM(LlamaConfig(hidden_size=512, intermediate_size=1024, num_attention_heads=4,
                                                 num_key_value_heads=kv_heads, num_hidden_layers=2, vocab_size=128))
    finally:
        torch.set_default_dtype(torch.float32)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    for layer in model.model.layers:
        layer.fuse()
        for n in (layer.input_layernorm, layer.post_attention_layernorm):
            n.weight.data.uniform_(0.5, 1.5)
    return model.eval()


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("width,kv_heads,P,shared,rows,maxlen,chunk", [(2, None, 16, 40, 4, 48, 16), (4, 2, 16, 40, 8, 48, 16),
                                                                     (4, None, 32, 40, 8, 48, 16), (4, 2, 32, 1200, 16, 24, 512)])
def test_every_beam_step_passes_the_float64_step_reference(monkeypatch, fp32_lm_head_reduction, width, kv_heads, P, shared, rows,
                                                          maxlen, chunk):
    """The eager serving loop with beams, chunked prefill, a shared prefix and two stop ids: every
    step is checked tensor by tensor by layer_ref64.ModelRef (the cascade decode, which 16 beams of 4 requests on a 1200-token
    prefix take, held to its bound), each deferred fork is fed
    to ModelRef.fork after the page-copy launch that carries it, so the next step's history audit covers the copied slots, and
    every beam step's decisions equal beam_ref's on the logits the step produced."""
    from atom_b200 import ops
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import KvCacheInt4, KvPoolInt4
    from tests import layer_ref64 as R
    model = _ref_model(kv_heads)
    bs, stops = rows, (5, 77)
    pool = KvPoolInt4(2, kv_heads or 4, 128, tg.pool_capacity(bs, maxlen + shared, P), P, DEV)
    ref = R.model_ref(model, P, sm_count=torch.cuda.get_device_properties(DEV).multi_processor_count)
    rec = R.Recorder().install(monkeypatch)
    pending, deferred, seen = {}, [], {"steps": 0, "beam_steps": 0, "forks": 0, "copies": 0, "near_ties": 0}
    fork = KvCacheInt4.fork

    def forked(kv, n=None, copies=None):
        child = fork(kv, n, copies)
        entry = (list(kv.indicies), child.seqlen, list(child.indicies))
        if copies is None:
            ref.fork(*entry)                        # the eager copy is done
        else:
            deferred.append(entry)                  # fed to the reference once its copy has run
        return child
    monkeypatch.setattr(KvCacheInt4, "fork", forked)

    def flush():
        for entry in deferred:
            ref.fork(*entry)
            seen["forks"] += 1
        deferred.clear()

    def copy(pool_, src, dst, slots):
        ops.copy_kv_pages(pool_, src, dst, slots)
        seen["copies"] += len(src)
        flush()

    class Wrapped:
        lm_head = model.lm_head

        def __call__(self, ids, blen, prefill_kv, decode_kv):
            flush()                                 # forks without a copy (a full last page) join before the step too
            out, pending["step"], pending["calls"], pending["before"], pending["after"] = R.run_step(rec, pool, model, ids, blen,
                                                                                                    prefill_kv, decode_kv)
            return out

    def select(logits, row_indptr, sums, w, stop_ids=(), out=None, workspace=None):
        res = ops.beam_select(logits, row_indptr, sums, w, stop_ids, out=out, workspace=workspace)
        Rn = logits.shape[0]
        _, _, ids, lps = ops.sample_tokens(logits.contiguous(), [0.0] * Rn, [0] * Rn, [1.0] * Rn, [(0, r) for r in range(Rn)],
                                           [0] * Rn, logprobs=ops.SAMPLE_TOP_N_MAX)
        ids, lps = ids.cpu().numpy(), lps.cpu().numpy()
        lp_rows = [{int(t): lps[r, j] for j, t in enumerate(ids[r]) if t >= 0} for r in range(Rn)]
        lg, ip, sm = logits.cpu().numpy(), row_indptr.cpu().numpy(), sums.cpu().numpy()
        got = [x.cpu().numpy() for x in res]
        for g, e in zip(got, BR.beam_select_np(lg, ip, sm, w, stop_ids, lp_rows=lp_rows)):
            assert np.array_equal(g.view(np.int32), e.view(np.int32))
        f64 = BR.beam_select_np(lg, ip, sm, w, stop_ids)
        for i in range(len(ip) - 1):
            for a, b in zip(map(tuple, np.concatenate([got[0][i], got[2][i]])), map(tuple, np.concatenate([f64[0][i], f64[2][i]]))):
                if a != b:
                    assert a[0] >= 0 and b[0] >= 0 and BR.near_tie(lg, sm, a, b), (i, a, b)
                    seen["near_ties"] += 1
        seen["beam_steps"] += 1
        return res

    rows_of, commit_beam = tg.TextGenScheduler.last_token_rows, tg.TextGenScheduler.commit_beam

    def last_token_rows(self):
        pending["step"].rows = rows_of(self)
        return pending["step"].rows

    def checked_commit_beam(self, *a, **k):
        ref.check_step(pending["calls"], pending.pop("step"), pending["before"], pending["after"])
        seen["steps"] += 1
        return commit_beam(self, *a, **k)

    monkeypatch.setattr(tg.TextGenScheduler, "last_token_rows", last_token_rows)
    monkeypatch.setattr(tg.TextGenScheduler, "commit_beam", checked_commit_beam)
    rs = tg.generate_request_set(6, maxlen)
    cfg = tg.TextGenConfig(bs, prefill_chunk=chunk, shared_prefix=shared, stop_token_ids=stops,
                           beam=tg.BeamSearchParams(width, 0.7))
    res = tg.run_textgen(Wrapped(), rs, cfg, pool, DEV, sync=torch.cuda.synchronize, keep_tokens=True, beam_select_op=select,
                         copy_op=copy)
    assert pool.num_free_blocks == pool.capacity
    assert not deferred
    assert seen["copies"] == res.beam["page_copies"] > 0 and seen["forks"] >= seen["copies"]
    assert ref.calls["prefill over a cached prefix"] > 0
    if shared >= 1024:                              # 16 beams on a long shared prefix: ops.decode_cascade picks the cascade
        assert ref.calls["cascade decode"] > 0
    print(f"W={width} kv_heads={kv_heads} P={P}: {seen}, worst error/bound {dict((k, round(v, 4)) for k, v in ref.worst.items())}, "
          f"{dict(ref.calls)}")
