"""CPU suite: the serving harness with a shared system prompt (TextGenConfig.shared_prefix).  A stand-in model records every
step; the pool lives on the CPU and no kernel is launched."""
import numpy as np
import pytest
import torch

from atom_b200 import textgen as tg
from atom_b200.kvcache import KvPoolInt4


class _RecordingLM:
    """Greedy chain (next = 7 * id + 3 mod vocab) that records, per step, the prompt chunks, the decode rows, the decode batch's
    prefix groups, and the pages in use checked against their closed form."""

    def __init__(self, vocab, pool, shared):
        self.vocab, self.pool, self.shared = vocab, pool, shared
        self.calls = []
        self.sched = None

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        groups = None if decode_kv is None else decode_kv.groups
        self.calls.append((list(blen.prefills), blen.decode, groups))
        s, P = self.sched, self.pool.block_len
        if s is not None:
            # pages in use: the system prompt's once, then per live request the pages from shared // P on
            live = [r.kvcache for r in s.workset] + [p.kvcache for p in s._prefilling if p.req_idx >= 0]
            root = s._root.kvcache if s._root is not None else None
            want = (len(root.indicies) if root is not None else 0) + sum(
                -(-c.seqlen // P) - (self.shared // P if root is not None else 0) for c in live)
            assert self.pool.capacity - self.pool.num_free_blocks == want
        nxt = (ids.long() * 7 + 3) % self.vocab
        return torch.nn.functional.one_hot(nxt, self.vocab).float(), None


def _run(monkeypatch, rs, batch, shared, chunk=None, block=16, capacity=None):
    cap = capacity or tg.pool_capacity(batch, 200, block) + 8 + batch
    pool = KvPoolInt4(1, 2, 128, cap, block, torch.device("cpu"))
    lm = _RecordingLM(97, pool, shared)
    orig = tg.TextGenScheduler.__init__

    def init(self, *a, **k):                       # hand the scheduler to the stand-in model for its page check
        orig(self, *a, **k)
        lm.sched = self
    with monkeypatch.context() as m:
        m.setattr(tg.TextGenScheduler, "__init__", init)
        res = tg.run_textgen(lm, rs, tg.TextGenConfig(batch, prefill_chunk=chunk, shared_prefix=shared), pool,
                             torch.device("cpu"), keep_tokens=True)
    return res, lm, pool


@pytest.mark.parametrize("shared,chunk", [(40, None), (64, None), (7, None), (100, 32), (33, 8)])
def test_system_prompt_is_prefilled_once_then_forked(monkeypatch, shared, chunk):
    rs = tg.generate_request_set(11, 64)
    res, lm, pool = _run(monkeypatch, rs, 4, shared, chunk)
    assert pool.num_free_blocks == pool.capacity                            # the root was released after the last request
    assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
    # every prompt token, the system prompt's included, is processed exactly once; decode rows as without a prefix
    rows = sum(sum(p) + d for p, d, _ in lm.calls)
    assert rows == shared + int(rs.prompt_lens.sum() + rs.output_lens.sum()) - len(rs)
    # the root first: the steps before the first request carry only system-prompt chunks, which add up to it
    cum = np.cumsum([sum(p) for p, _, _ in lm.calls])
    first_req = int(np.argmax(cum > shared))
    assert sum(sum(p) for p, _, _ in lm.calls[:first_req]) == shared
    assert all(d == 0 for _, d, _ in lm.calls[:first_req])
    if chunk is not None:
        assert all(sum(p) <= chunk for p, _, _ in lm.calls)
    # decode batches of two or more forked rows form one group over the shared full pages
    for p, d, groups in lm.calls:
        if d >= 2 and shared >= 16:
            assert len(groups) == 1 and groups[0][1] == shared // 16 and len(groups[0][0]) == d
        elif d:
            assert groups == []


def test_admission_counts_only_the_pages_a_fork_takes(monkeypatch):
    block, shared = 16, 40                       # 2 full pages shared, 8 tokens copied into each fork's own page
    rs = tg.RequestSet(np.array([20, 20, 20], np.int32), np.array([3, 3, 3], np.int32))
    # root 3 pages; a fork of a 20-token prompt: ceil(60 / 16) - 2 = 2 pages + 1 spare = 3: room for two requests in 9 pages
    sched = tg.TextGenScheduler(rs, 3, KvPoolInt4(1, 1, 128, 9, block, torch.device("cpu")), torch.device("cpu"), 97,
                                shared_prefix=shared)
    assert sched._pages_needed(20) == 3 and sched._pages_needed(8) == 2 and sched._pages_needed(24) == 3
    res, lm, pool = _run(monkeypatch, rs, 3, shared, capacity=9)
    assert lm.calls[0][0] == [40] and lm.calls[1][0] == [20, 20]            # the third request waits for pages
    assert [len(t) for t in res.tokens] == [3, 3, 3] and pool.num_free_blocks == 9
    # unshared, the same requests need 5 + 5 + 5 pages at once: sharing is what lets two run in 9 pages
    assert tg.TextGenScheduler(rs, 3, KvPoolInt4(1, 1, 128, 9, block, torch.device("cpu")), torch.device("cpu"), 97,
                               shared_prefix=0)._pages_needed(60) == 5


@pytest.mark.parametrize("chunk", [None, 24])
def test_shared_prefix_zero_is_todays_schedule(monkeypatch, chunk):
    rs = tg.generate_request_set(9, 64)
    a, la, _ = _run(monkeypatch, rs, 3, 0, chunk)
    pool = KvPoolInt4(1, 2, 128, tg.pool_capacity(3, 200, 16) + 8 + 3, 16, torch.device("cpu"))
    lm = _RecordingLM(97, pool, 0)
    b = tg.run_textgen(lm, rs, tg.TextGenConfig(3, prefill_chunk=chunk), pool, torch.device("cpu"), keep_tokens=True)
    assert la.calls == lm.calls and a.tokens == b.tokens
    # the request set and the per-request prompts do not depend on the system prompt
    s0 = tg.TextGenScheduler(rs, 3, pool, torch.device("cpu"), 97)
    s1 = tg.TextGenScheduler(rs, 3, KvPoolInt4(1, 2, 128, 64, 16, torch.device("cpu")), torch.device("cpu"), 97, shared_prefix=50)
    assert s0._rng.integers(0, 97, 20).tolist() == s1._rng.integers(0, 97, 20).tolist()
    with pytest.raises(ValueError):
        tg.TextGenScheduler(rs, 3, pool, torch.device("cpu"), 97, shared_prefix=-1)


class _TableLM:
    """Records, per call, the decode page table and prefix-group tables the model was handed (host copies)."""

    def __init__(self, vocab):
        self.vocab, self.tables = vocab, []

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        if decode_kv is not None and prefill_kv is None:
            b = blen.decode
            ip = decode_kv.indptr.tolist()
            t = {"indptr": ip, "last": decode_kv.last_page_offset.tolist(), "indices": decode_kv.indicies[:ip[-1]].tolist(),
                 "groups": getattr(decode_kv, "groups", [])}
            if t["groups"]:
                gi = decode_kv.group_indptr.tolist()
                t.update(gindptr=gi, members=decode_kv.group_members[:gi[-1]].tolist(), shared=decode_kv.shared_pages[:b].tolist(),
                         bounds=getattr(decode_kv, "group_bounds", None))
            self.tables.append(t)
        nxt = (ids.long() * 7 + 3) % self.vocab
        return torch.nn.functional.one_hot(nxt, self.vocab).float(), None


@pytest.mark.parametrize("shared", [0, 40])
def test_decode_graph_runner_carries_the_prefix_groups_in_its_static_buffer(shared):
    """DecodeGraphRunner with capture=False: the group tables it hands the model from its static buffer equal those of the eager
    BatchedKvCacheInt4, step by step, and state the bounds the graph is sized from (B members, max_pages shared pages)."""
    rs = tg.generate_request_set(11, 64)
    block, bs, maxp = 16, 4, 64 // 16 + 1 + 3
    runs = []
    for use_runner in (False, True):
        pool = KvPoolInt4(1, 2, 128, tg.pool_capacity(bs, 64, block) + 3 + bs, block, torch.device("cpu"))
        lm = _TableLM(97)
        runner = tg.DecodeGraphRunner(lm, pool, "cpu", max_pages_per_seq=maxp, capture=False) if use_runner else None
        res = tg.run_textgen(lm, rs, tg.TextGenConfig(bs, shared_prefix=shared), pool, torch.device("cpu"), keep_tokens=True,
                             decode_runner=runner)
        assert pool.num_free_blocks == pool.capacity
        runs.append((res.tokens, lm.tables))
    (tok_e, tab_e), (tok_g, tab_g) = runs
    assert tok_e == tok_g and len(tab_e) == len(tab_g) > 0
    for e, g in zip(tab_e, tab_g):
        for k in ("indptr", "last", "indices", "groups"):
            assert e[k] == g[k], k
        if e["groups"]:
            assert e["gindptr"] == g["gindptr"] and e["members"] == g["members"] and e["shared"] == g["shared"]
            assert g["bounds"] == (len(e["last"]), maxp) and e["bounds"] is None
    assert any(t["groups"] for t in tab_g) == (shared >= block)
    # one graph entry per (batch size, number of groups); without groups the buffer has today's layout
    r = tg.DecodeGraphRunner(None, KvPoolInt4(1, 2, 128, 8, block, torch.device("cpu")), "cpu", max_pages_per_seq=maxp, capture=False)
    assert r._layout(3)[-1] == 3 * 3 + 1 + 3 * maxp and r._layout(3, 1)[-1] == 3 * 3 + 1 + 3 * maxp + 2 + 2 * 3
