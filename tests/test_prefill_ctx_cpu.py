"""CPU suite: prefill over a cached prefix (chunked prefill, prompt continuation) -- the float64 reference against the
whole-prompt one, the chunked scheduler of atom_b200/textgen.py with a stand-in model, and the host helpers (KvCacheInt4.acquire,
BatchedKvCacheInt4.seqlens, the argument checks of ops.prefill_attention_i4)."""
import numpy as np
import pytest
import torch

from atom_b200 import ops
from atom_b200 import textgen as tg
from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
from tests import attn_ctx_ref64 as C
from tests import attn_ref64 as R


# ------------------------------------------------------------------------------------------------ float64 reference
@pytest.mark.parametrize("regime", ["moderate", "sink"])
def test_reference_at_empty_context_is_the_prefill_reference(regime):
    rng = np.random.default_rng(1)
    lens, hq, hkv, theta = [1, 17, 64, 129], 8, 2, 5e5
    (q, k4, kp, v4, vp), pool = C.make_ctx_case(rng, [0] * 4, lens, hq, hkv, 16, regime)
    ref, bnd = C.prefill_ctx_bound(q, k4, kp, v4, vp, lens, hq, theta, *pool)
    ref0, bnd0 = R.prefill_bound(q, k4, kp, v4, vp, lens, hq, theta)
    assert np.array_equal(ref, ref0) and np.array_equal(bnd, bnd0)
    assert np.array_equal(C.prefill_ctx_ref(q, k4, kp, v4, vp, lens, hq, theta, *pool), R.prefill_ref(q, k4, kp, v4, vp, lens, hq, theta))


def _truncate(pool, n, P):
    """The page table of a one-sequence pool cut to its first n tokens."""
    data, param, indptr, indices, last = pool
    pages = (n + P - 1) // P
    return data, param, np.array([0, pages], np.int32), indices[:pages], np.array([(n - 1) % P + 1], np.int32)


@pytest.mark.parametrize("P", [8, 32])
def test_chunks_reproduce_the_one_shot_reference(P):
    rng = np.random.default_rng(2)
    n, hq, hkv, theta = 300, 4, 2, 1e4
    (q, k4, kp, v4, vp), pool = C.make_ctx_case(rng, [0], [n], hq, hkv, P, "sink")
    whole = R.prefill_ref(q, k4, kp, v4, vp, [n], hq, theta)
    a = 0
    for c in (64, 100, 1, 135):
        b = a + c
        part = C.prefill_ctx_ref(q[a:b], k4[a:b], kp[a:b], v4[a:b], vp[a:b], [c], hq, theta, *_truncate(pool, b, P))
        assert np.abs(part - whole[a:b]).max() <= 1e-12
        a = b
    assert a == n


def test_bound_grows_with_the_context():
    """The context lengthens the angle and accumulation terms: the same chunk over a longer prefix gets a larger bound."""
    rng = np.random.default_rng(3)
    (q, k4, kp, v4, vp), pool = C.make_ctx_case(rng, [1000], [17], 2, 2, 16)
    _, bnd = C.prefill_ctx_bound(q, k4, kp, v4, vp, [17], 2, 1e4, *pool)
    assert np.isfinite(bnd).all() and (bnd > 0).all()
    assert bnd.min() > R.E


# ------------------------------------------------------------------------------------------------ scheduler
class _FakeLM:
    """argmax(row) = (input id * 7 + 3) % vocab; checks every step's page table against its chunks and records them."""

    def __init__(self, vocab, batch_size, block_len):
        self.vocab, self.batch_size, self.block_len = vocab, batch_size, block_len
        self.calls = []

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        assert ids.numel() == blen.doff + blen.decode
        assert len(blen.prefills) + blen.decode <= self.batch_size
        assert (prefill_kv is None) == (len(blen.prefills) == 0) and (decode_kv is None) == (blen.decode == 0)
        seqlens = firsts = None
        if prefill_kv is not None:
            firsts = prefill_kv.indicies[prefill_kv.indptr[:-1].long()].tolist()   # first page: names a live request
            n_pages = (prefill_kv.indptr[1:] - prefill_kv.indptr[:-1]).tolist()
            seqlens = list(prefill_kv.seqlens)
            for chunk, s, pages, last in zip(blen.prefills, seqlens, n_pages, prefill_kv.last_page_offset.tolist()):
                assert s >= chunk and pages == -(-s // self.block_len) and last == (s - 1) % self.block_len + 1
        self.calls.append((list(blen.prefills), blen.decode, seqlens, ids.tolist(), firsts))
        nxt = (ids.long() * 7 + 3) % self.vocab
        return torch.nn.functional.one_hot(nxt, self.vocab).float(), None


def _run(rs, bs, block, chunk, capacity=None):
    pool = KvPoolInt4(1, 1, 128, capacity or tg.pool_capacity(bs, int((rs.prompt_lens + rs.output_lens).max()), block), block,
                      torch.device("cpu"))
    lm = _FakeLM(97, bs, block)
    cap = pool.num_free_blocks
    res = tg.run_textgen(lm, rs, tg.TextGenConfig(bs, prefill_chunk=chunk), pool, torch.device("cpu"), keep_tokens=True)
    assert pool.num_free_blocks == cap                                   # the pool ends full
    return res, lm


@pytest.mark.parametrize("bs,maxlen", [(4, 96), (7, 64)])
def test_no_chunk_and_large_chunks_give_todays_schedule(bs, maxlen):
    """A budget no step reaches (N >= every step's prompt tokens, e.g. N >= all prompts together) is today's schedule."""
    rs = tg.generate_request_set(3 * bs + 2, maxlen)
    base, lm0 = _run(rs, bs, 16, None)
    assert all(c[2] is None or c[2] == c[0] for c in lm0.calls)          # without chunking every prompt is its whole sequence
    for chunk in (max(sum(c[0]) for c in lm0.calls), int(rs.prompt_lens.sum()), 10 ** 6):
        res, lm = _run(rs, bs, 16, chunk)
        assert res.tokens == base.tokens and res.steps == base.steps
        assert [c[:4] for c in lm.calls] == [c[:4] for c in lm0.calls]


def test_large_chunk_equals_no_chunk_when_steps_fit():
    rs = tg.RequestSet(np.array([5, 9, 3, 7, 2], np.int32), np.array([4, 3, 6, 2, 5], np.int32))
    base, lm0 = _run(rs, 3, 8, None)
    res, lm = _run(rs, 3, 8, 10 ** 6)
    assert res.tokens == base.tokens and [c[:3] for c in lm.calls] == [c[:3] for c in lm0.calls]


@pytest.mark.parametrize("chunk", [1, 7, 64])
@pytest.mark.parametrize("bs,maxlen", [(4, 96), (3, 200)])
def test_chunked_schedule_processes_every_prompt_token_once(chunk, bs, maxlen):
    rs = tg.generate_request_set(3 * bs + 2, maxlen)
    res, lm = _run(rs, bs, 16, chunk)
    assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
    for toks in res.tokens:
        assert all(toks[i + 1] == (toks[i] * 7 + 3) % 97 for i in range(len(toks) - 1))
    # every step carries at most N prompt tokens; each chunk is the tail of its sequence, so replaying the chunks request by
    # request (in admission order) rebuilds every prompt exactly once
    assert all(sum(c[0]) <= chunk for c in lm.calls)
    fed, live, order = {}, {}, []
    for prefills, _, seqlens, ids, firsts in lm.calls:
        off = 0
        for n, s, page in zip(prefills, seqlens or [], firsts or []):
            if s == n:                                                    # a first chunk: a new request
                live[page] = len(order); order.append(len(order)); fed[live[page]] = []
            key = live[page]
            assert len(fed[key]) == s - n                                 # the chunk continues where the last one ended
            fed[key] += ids[off:off + n]
            off += n
    assert [len(fed[k]) for k in order] == rs.prompt_lens.tolist()       # FCFS, every prompt token once
    rows = sum(sum(c[0]) + c[1] for c in lm.calls)
    assert rows == int(rs.prompt_lens.sum() + rs.output_lens.sum()) - len(rs)
    # partly prefilled requests continue first: a step's continuing chunks precede its first chunks
    for prefills, _, seqlens, _, _ in lm.calls:
        firsts = [s == n for n, s in zip(prefills, seqlens or [])]
        assert firsts == sorted(firsts)


def test_rows_tokens_and_latencies_line_up():
    rs = tg.RequestSet(np.array([20, 3, 11], np.int32), np.array([3, 2, 4], np.int32))
    pool = KvPoolInt4(1, 1, 128, 32, 8, torch.device("cpu"))
    sched = tg.TextGenScheduler(rs, 3, pool, torch.device("cpu"), vocab_size=50, prefill_chunk=8)
    clock, seen = 0.0, []
    while not sched.finished:
        sched.admit()
        batch = sched.next_batch()
        rows = sched.last_token_rows()
        done_in_step = [s + n == len(p.prompt) for p, s, n in sched._new]
        assert len(rows) == sum(done_in_step) + batch.blen.decode
        assert sched.prompt_tokens == sum(batch.blen.prefills) <= 8
        seen.append((list(batch.blen.prefills), rows))
        sched.commit([1] * len(rows), clock, clock + 1.0)
        clock += 2.0
    res = sched.result(clock, len(seen))
    # request 0 (20 tokens) takes three 8-token steps: its encode latency spans them (first step start -> third step end)
    assert seen[0][0] == [8] and seen[1][0] == [8] and seen[2][0][0] == 4
    assert res.encode_latency[0] == pytest.approx(5.0)
    assert (res.decode_latency >= res.encode_latency).all()
    assert pool.num_free_blocks == 32


def test_admission_reserves_the_rest_of_partly_prefilled_prompts():
    """Pages: a 40-token prompt in 16-token chunks holds 1, 2, 3 pages of its 3 + 1 spare; a second request must not take the
    pages the first has yet to fill, and the pool never over-commits."""
    rs = tg.RequestSet(np.array([40, 40], np.int32), np.array([3, 3], np.int32))
    block = 16                                                          # 4 + 4 pages would be needed for both at once
    res, lm = _run(rs, 2, block, 16, capacity=7)                        # an over-commit would raise "out of pages"
    assert [len(t) for t in res.tokens] == [3, 3]
    starts = [i for i, c in enumerate(lm.calls) for n, s in zip(c[0], c[2] or []) if s == n]
    assert len(starts) == 2 and starts[0] == 0
    assert lm.calls[starts[1]][1] == 0 and lm.calls[starts[1] - 1][1] == 1   # request 1 waited until request 0 had finished
    with pytest.raises(RuntimeError, match="KV pool too small"):
        _run(tg.RequestSet(np.array([40], np.int32), np.array([2], np.int32)), 1, block, 16, capacity=3)


def test_prefill_chunk_must_be_positive():
    pool = KvPoolInt4(1, 1, 128, 4, 16, torch.device("cpu"))
    with pytest.raises(ValueError, match="prefill_chunk"):
        tg.TextGenScheduler(tg.RequestSet(np.array([3], np.int32), np.array([2], np.int32)), 1, pool, "cpu", prefill_chunk=0)


# ------------------------------------------------------------------------------------------------ host helpers
def test_acquire_grows_by_n_tokens_and_batch_records_lengths():
    pool = KvPoolInt4(1, 1, 128, 8, 16, torch.device("cpu"))
    a = KvCacheInt4(pool, 10)
    a.acquire(6)
    assert a.seqlen == 16 and len(a.indicies) == 1 and a.last_page_offset == 16
    a.acquire(1)
    assert a.seqlen == 17 and len(a.indicies) == 2
    a.acquire(0)
    assert a.seqlen == 17 and len(a.indicies) == 2
    b = KvCacheInt4(pool, 0)
    b.acquire(33)
    assert len(b.indicies) == 3 and b.last_page_offset == 1
    with pytest.raises(ValueError):
        b.acquire(-1)
    batch = BatchedKvCacheInt4([a, b])
    assert batch.seqlens == [17, 33]
    a.acquire_one()
    assert batch.seqlens == [17, 33]                                    # captured at construction
    a.release(); b.release()
    assert pool.num_free_blocks == 8


def test_prefill_context_checks():
    class Kv:
        seqlens = [10, 5]
    assert ops._prefill_contexts(None, None, [3, 4]) == [0, 0]
    assert ops._prefill_contexts(Kv(), 0, [3, 5]) == [7, 0]
    with pytest.raises(RuntimeError, match="fewer than its prompt"):
        ops._prefill_contexts(Kv(), 0, [3, 6])
    with pytest.raises(RuntimeError, match="2 sequences for 3 prompts"):
        ops._prefill_contexts(Kv(), 0, [1, 1, 1])
    with pytest.raises(RuntimeError, match="no host sequence lengths"):
        ops._prefill_contexts(object(), 0, [1, 1])
    with pytest.raises(RuntimeError, match="layer_idx"):
        ops._prefill_contexts(Kv(), None, [3, 5])
