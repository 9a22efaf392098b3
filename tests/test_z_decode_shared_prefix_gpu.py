"""GPU suite: shared-prefix decode.  Sequences forked from one root share its full INT4 pages (kvcache.py), and the cascade
(ops.batch_decode_i4 on a batch with prefix groups) attends each group's shared pages once per KV head on tensor cores, then
each row's private pages with the decode kernel.

  1. accuracy: every G x page size x RoPE base and the score regimes of test_z_attention_accuracy_gpu, groups of 2 to 32
     members (more rows than one 64-row tile), prefixes from one page to 32k tokens, suffixes from one token to several pages,
     groups and lone rows interleaved; every row within tests/attn_cascade_ref64.cascade_bound, lone rows bit-identical to the
     existing kernel (kv_split=1) and within decode_bound;
  2. determinism: identical bytes on a dirty pool, under another page placement and on a repeated call;
  3. the existing kernel on shared pages: kv_split=1 on a forked pool is bit-identical to the same rows on a pool where the
     prefix pages are physically duplicated;
  4. the automatic choice follows ops.decode_cascade on both sides of its threshold;
  5. a CUDA graph of append + cascade decode with PDL replays bit for bit against eager, across a page boundary.
"""
import numpy as np
import pytest
import torch

from tests import attn_ref64 as R
from tests.attn_cascade_ref64 import cascade_bound
from tests.test_z_attention_accuracy_gpu import SIGMA_Q, _centred, _check

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
PAGES = [8, 16, 24, 32, 64]
THETAS = [1e4, 5e5, 1e6]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint16)


class Case:
    """A forked batch on a real KvPoolInt4: groups = [(prefix tokens, [suffix lengths])], lone = [lengths].  Each group is a root
    prefilled with `prefix` tokens (not in the batch) and one fork per suffix, grown by it; rows interleave group members and
    lone sequences.  The pool's bytes are written from the host: every row's whole sequence, so shared pages get the same bytes
    from each member.  place: seed of the page placement (the pool's stack is shuffled); dirty: unused slots hold 0xFF / NaN."""

    def __init__(self, rng, P, hkv, groups, lone, L=1, layer=0, place=0, dirty=False, kscale=(0.1, 1.0), vscale=(0.1, 1.0),
                 duplicate=False):
        from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
        self.P, self.hkv, self.layer = P, hkv, layer
        cap = sum(-(-(p + s) // P) + 1 for p, ss in groups for s in ss) + sum(-(-n // P) for n in lone) \
            + sum(-(-p // P) for p, _ in groups) + 5
        self.pool = pool = KvPoolInt4(L, hkv, 128, cap, P, torch.device(DEV))
        pages = [pool.alloc_block() for _ in range(cap)]
        for i in np.random.default_rng(place).permutation(cap):
            pool.free_block(pages[i])
        content, members, self.roots = [], [], []
        for p, ss in groups:
            pre = _centred(rng, hkv, p, kscale, vscale)
            if duplicate:            # the same bytes on pages of each member's own
                mem = [KvCacheInt4(pool, p + s) for s in ss]
            else:
                root = KvCacheInt4(pool, p)
                self.roots.append(root)
                mem = [root.fork() for _ in ss]
                for m, s in zip(mem, ss):
                    m.acquire(s)
            for s in ss:
                suf = _centred(rng, hkv, s, kscale, vscale)
                content.append(tuple(np.concatenate([a, b], 1) for a, b in zip(pre, suf)))
            members.append(mem)
        lone_seqs = [KvCacheInt4(pool, n) for n in lone]
        lone_content = [_centred(rng, hkv, n, kscale, vscale) for n in lone]
        # interleave: member 0 of every group, a lone row, member 1 of every group, ...
        rows, rc, self.lone_rows = [], [], []
        queues = [list(zip(m, content[sum(len(x) for x in members[:gi]):][:len(m)])) for gi, m in enumerate(members)]
        lq = list(zip(lone_seqs, lone_content))
        while any(queues) or lq:
            for qu in queues:
                if qu:
                    s, c = qu.pop(0); rows.append(s); rc.append(c)
            if lq:
                s, c = lq.pop(0); self.lone_rows.append(len(rows)); rows.append(s); rc.append(c)
        self.rows = rows
        data = np.full(tuple(pool.buf.shape), 0xFF if dirty else 0, np.uint8)
        param = np.full(tuple(pool.param.shape), np.nan if dirty else 0, np.float16)
        for s, (kn, kp, vn, vp) in zip(rows, rc):
            n = kn.shape[1]
            for j, pg in enumerate(s.indicies):
                a, e = j * P, min(n, (j + 1) * P)
                for which, (nib, par) in enumerate(((kn, kp), (vn, vp))):
                    data[pg, layer, which, :, :e - a] = R.pack(nib[:, a:e])
                    param[pg, layer, which, :, :e - a] = par[:, a:e]
        pool.buf.copy_(torch.from_numpy(data))
        pool.param.copy_(torch.from_numpy(param))
        self.batch = BatchedKvCacheInt4(rows)
        self.data, self.param = data, param

    def table(self):
        b = self.batch
        shared = b.shared_pages.cpu().numpy() if b.shared_pages is not None else np.zeros(len(self.rows), np.int32)
        return b.indptr.cpu().numpy(), b.indicies.cpu().numpy(), b.last_page_offset.cpu().numpy(), shared

    def release(self):
        for s in self.rows + self.roots:
            s.release()
        assert self.pool.num_free_blocks == self.pool.capacity


def cascade(q, case, theta):
    """The cascade, whatever the automatic rule would pick."""
    from atom_b200 import ops
    b = case.batch
    L, H, P = ops._kv_dims(b)
    qt = torch.from_numpy(q).to(DEV)
    o = torch.empty_like(qt)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    return ops._batch_decode_shared(o, qt, b, b.groups, L, H, P, case.layer, theta, sms).cpu().numpy()


def plain(q, case, theta, split=1):
    from atom_b200 import ops
    return ops.batch_decode_i4(torch.from_numpy(q).to(DEV), case.batch, case.layer, rope_theta=theta, kv_split=split).cpu().numpy()


def check_case(case, q, theta, what):
    got = cascade(q, case, theta)
    indptr, indices, last, shared = case.table()
    hq = q.shape[1]
    ref, bnd = cascade_bound(q, case.data, case.param, indptr, indices, last, case.layer, hq, theta, shared)
    worst = _check(got, ref, bnd, what)
    if case.lone_rows:
        lone = plain(q, case, theta)
        assert np.array_equal(_bits(got[case.lone_rows]), _bits(lone[case.lone_rows])), f"{what}: lone rows differ from kv_split=1"
        ref_d, bnd_d = R.decode_bound(q, case.data, case.param, indptr, indices, last, case.layer, hq, theta)
        _check(got[case.lone_rows], ref_d[case.lone_rows], bnd_d[case.lone_rows], what + " (lone rows, decode_bound)")
    return got, worst


# ------------------------------------------------------------------------------------------------ 1. accuracy
@pytest.mark.parametrize("P", PAGES)
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_cascade_every_group_and_page_size_within_bound(G, P):
    theta = THETAS[(G + P) % 3]
    seed = 1000 * G + P
    rng = np.random.default_rng(seed)
    hkv = 2 if G < 8 else 1
    # a one-page prefix, a prefix with a partial page (its last page is copied: private), a several-tile prefix; suffixes of one
    # token to several pages; two lone rows
    groups = [(P, [1, P - 1, 2 * P + 3]), (3 * P + P // 2, [1, 5]), (5 * 64 + 2 * P, [P, 3 * P + 1, 7])]
    case = Case(rng, P, hkv, groups, [P + 3, 130], L=2, layer=1, place=seed)
    assert [len(m) for m, _ in case.batch.groups] == [3, 2, 3]
    assert [n for _, n in case.batch.groups] == [1, 3, (5 * 64 + 2 * P) // P]
    q = (rng.standard_normal((len(case.rows), G * hkv, 128)) * SIGMA_Q["moderate"]).astype(np.float16)
    check_case(case, q, theta, f"cascade G={G} P={P} theta={theta:g}")
    case.release()


REGIMES = list(SIGMA_Q) + ["one-hot", "vscale16"]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("G,P", [(1, 16), (4, 32), (8, 64), (2, 24)])
def test_cascade_score_regimes_within_bound(G, P, regime):
    theta = THETAS[P % 3]
    rng = np.random.default_rng(100 * G + P + 10000 * REGIMES.index(regime))
    hkv = 2
    vscale = (16.0, 16.0) if regime == "vscale16" else (0.1, 1.0)
    groups = [(8 * P, [2, P + 1, 3 * P]), (2 * P, [1, 1, 1, 1])]
    case = Case(rng, P, hkv, groups, [3 * P], vscale=vscale, place=G + P)
    sigma = SIGMA_Q["moderate" if regime in ("one-hot", "vscale16") else regime]
    q = (rng.standard_normal((len(case.rows), G * hkv, 128)) * sigma).astype(np.float16)
    if regime == "one-hot":                     # all of q's weight on one pair: the scores follow one key component
        q[:] = 0
        q[:, :, 63] = 8.0
    check_case(case, q, theta, f"cascade {regime} G={G} P={P}")
    case.release()


@pytest.mark.parametrize("members,G,P", [(32, 4, 16), (17, 8, 32), (32, 1, 64), (9, 8, 8)])
def test_cascade_groups_with_more_rows_than_one_tile(members, G, P):
    rng = np.random.default_rng(members * 100 + G + P)
    groups = [(6 * P, list(rng.integers(1, 3 * P, members)))]
    case = Case(rng, P, 1, groups, [2 * P], place=members)
    assert len(case.batch.groups[0][0]) == members
    q = (rng.standard_normal((len(case.rows), G, 128)) * SIGMA_Q["moderate"]).astype(np.float16)
    check_case(case, q, 1e4, f"cascade {members} members G={G} P={P}")
    case.release()


@pytest.mark.parametrize("prefix,G,P,theta,regime", [(32768, 4, 32, 5e5, "moderate"), (32768, 8, 64, 1e6, "peaked"),
                                                     (8192, 1, 16, 1e4, "peaked"), (512, 2, 8, 1e4, "flat")])
def test_cascade_long_prefixes_within_bound(prefix, G, P, theta, regime):
    rng = np.random.default_rng(prefix + G + P)
    case = Case(rng, P, 1, [(prefix, [1, P + 5, 1000])], [700])
    q = (rng.standard_normal((len(case.rows), G, 128)) * SIGMA_Q[regime]).astype(np.float16)
    check_case(case, q, theta, f"cascade prefix {prefix} {regime} G={G} P={P}")
    case.release()


# ------------------------------------------------------------------------------------------------ 2. determinism
@pytest.mark.parametrize("G,P", [(4, 16), (8, 32), (1, 64)])
def test_cascade_is_deterministic_on_dirty_pools_and_under_other_placements(G, P):
    groups, lone = [(5 * P + 3, [1, 2 * P, 9]), (2 * P, [P - 1, 4])], [3, 2 * P + 1]
    rng = lambda: np.random.default_rng(G * 7 + P)
    q = (np.random.default_rng(1).standard_normal((7, G * 2, 128)) * 0.7).astype(np.float16)
    base = Case(rng(), P, 2, groups, lone, place=1)
    got = cascade(q, base, 5e5)
    assert np.array_equal(_bits(cascade(q, base, 5e5)), _bits(got))
    base.release()
    dirty = Case(rng(), P, 2, groups, lone, place=1, dirty=True)
    assert np.array_equal(_bits(cascade(q, dirty, 5e5)), _bits(got))
    dirty.release()
    other = Case(rng(), P, 2, groups, lone, place=2)
    assert [r.indicies for r in other.rows] != [r.indicies for r in base.rows]
    assert np.array_equal(_bits(cascade(q, other, 5e5)), _bits(got))
    other.release()


# ------------------------------------------------------------------------------------------------ 3. existing kernel, shared pages
@pytest.mark.parametrize("G,P", [(1, 16), (4, 32), (8, 64), (2, 24)])
def test_existing_kernel_on_shared_pages_equals_duplicated_pages(G, P):
    groups, lone = [(4 * P + 5, [1, P, 3 * P + 2]), (P, [2, 2])], [P + 1]
    q = (np.random.default_rng(3).standard_normal((6, G * 2, 128)) * 0.7).astype(np.float16)
    shared = Case(np.random.default_rng(G + P), P, 2, groups, lone, place=4)
    dup = Case(np.random.default_rng(G + P), P, 2, groups, lone, place=5, duplicate=True)
    assert shared.batch.groups and not dup.batch.groups
    for split in (1, 2):
        assert np.array_equal(_bits(plain(q, shared, 1e4, split)), _bits(plain(q, dup, 1e4, split))), split
    shared.release()
    dup.release()


# ------------------------------------------------------------------------------------------------ 4. the automatic choice
def test_auto_follows_the_rule_on_both_sides_of_its_threshold():
    from atom_b200 import ops
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    P, hkv, G = 32, 8, 4
    need = ops.DECODE_CASCADE_MIN_PER_SM * sms                     # token-heads the cascade must save
    pages_at = -(-need // (hkv * 3 * P))                           # a four-member group at the threshold
    rng = np.random.default_rng(5)
    for pages, lone, picked in ((pages_at - 1, [], False), (pages_at, [], True), (pages_at, [100] * 4, False)):
        case = Case(rng, P, hkv, [(pages * P, [3, 40, 1, 70])], lone)
        B = len(case.rows)
        assert ops.decode_cascade(case.batch.groups, B, P, hkv, G, sms) is picked
        q = (rng.standard_normal((B, G * hkv, 128)) * 0.7).astype(np.float16)
        auto = plain(q, case, 1e4, split=0)
        want = cascade(q, case, 1e4) if picked else plain(q, case, 1e4, split=ops.decode_kv_split(B, hkv, G))
        assert np.array_equal(_bits(auto), _bits(want)), (pages, lone)
        case.release()


# ------------------------------------------------------------------------------------------------ 5. graphs
def test_graph_of_append_and_cascade_decode_with_pdl_replays_bit_for_bit():
    """Append one token per row, then the cascade: captured once with PDL on, its page table in static buffers that are
    rewritten between replays, and replayed over three steps that cross a page boundary; every step equals the same calls made
    eagerly on an identical pool."""
    from atom_b200 import _lib, ops
    from atom_b200.kvcache import BatchedKvCacheInt4
    P, hkv, G = 16, 2, 4
    groups_in, lone = [(4 * P, [P - 2, 3]), (P, [5, P - 1, 1])], [P - 2]
    eager_case = Case(np.random.default_rng(11), P, hkv, groups_in, lone, place=3)
    graph_case = Case(np.random.default_rng(11), P, hkv, groups_in, lone, place=3)
    b = len(eager_case.rows)
    rng = np.random.default_rng(12)
    q = torch.from_numpy((rng.standard_normal((b, G * hkv, 128)) * 0.7).astype(np.float16)).to(DEV)
    k = torch.randint(0, 256, (b, hkv * 64), dtype=torch.uint8, device=DEV)
    v = torch.randint(0, 256, (b, hkv * 64), dtype=torch.uint8, device=DEV)
    kp = (torch.rand((b, hkv, 2), device=DEV) * torch.tensor([0.2, 1.5], device=DEV)).half()
    vp = (torch.rand((b, hkv, 2), device=DEV) * torch.tensor([0.2, 1.5], device=DEV)).half()
    L, H, _ = ops._kv_dims(eager_case.batch)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    groups = eager_case.batch.groups

    def grow(case):
        for r in case.rows:
            r.acquire_one()
        kv = BatchedKvCacheInt4(case.rows)
        assert kv.groups == groups
        return kv

    def step(kv, out):
        ops.append_kv_i4(kv, k, v, kp, vp, 0)
        out.copy_(ops._batch_decode_shared(torch.empty_like(q), q, kv, groups, L, H, P, 0, 1e4, sms))

    eager = []
    for _ in range(3):
        out = torch.empty_like(q)
        step(grow(eager_case), out)
        eager.append(out.cpu().numpy())

    names = ("indptr", "last_page_offset", "indicies", "group_indptr", "group_members", "shared_pages")
    kv = grow(graph_case)
    static = type("StaticKV", (), {})()
    static.data, static.param = kv.data, kv.param
    for n in names:
        t = getattr(kv, n)
        setattr(static, n, torch.zeros(t.numel() + (4 * b if n == "indicies" else 0), dtype=torch.int32, device=DEV))

    def load(kv):
        for n in names:
            t = getattr(kv, n)
            getattr(static, n)[:t.numel()].copy_(t)

    out = torch.empty_like(q)
    got = []
    _lib.check(_lib.lib().atom_set_pdl(1), "set_pdl")
    try:
        load(kv)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step(static, out)                                      # step 1, eager with PDL: also warms every kernel up
        torch.cuda.current_stream().wait_stream(s)
        got.append(out.cpu().numpy())
        g = torch.cuda.CUDAGraph()
        # the capture records the launches without running them: the pool is left as step 1 left it
        with torch.cuda.graph(g):
            step(static, out)
        for _ in range(2):
            load(grow(graph_case))
            g.replay()
            torch.cuda.synchronize()
            got.append(out.cpu().numpy())
    finally:
        _lib.check(_lib.lib().atom_set_pdl(0), "set_pdl")
    assert any(r.seqlen % P == 1 for r in graph_case.rows), "no row crossed a page boundary"
    for i in range(3):
        assert np.array_equal(_bits(got[i]), _bits(eager[i])), f"step {i}"
    eager_case.release()
    graph_case.release()


# ------------------------------------------------------------------------------------------------ 6. graphed serving steps
class _AttnStep:
    """A stand-in decode step for DecodeGraphRunner: decode attention of fixed q over the table it is handed; the output is kept."""

    def __init__(self, q, theta):
        self.q, self.theta, self.out = q, theta, torch.zeros_like(q)

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        from atom_b200 import ops
        o = ops.batch_decode_i4(self.q, decode_kv, 0, rope_theta=self.theta)
        self.out.copy_(o)
        return o.reshape(o.size(0), -1)[:, :64].float(), None


def test_decode_graph_runner_replays_the_cascade_as_members_join_and_leave(monkeypatch):
    """One graph key (6 rows, 1 group): the graph is captured with four members and two lone rows, then replayed as a fifth
    member joins, as a member leaves, and as every row grows across a page boundary; each replay equals the eager cascade over
    the same pool, bit for bit.  The cascade is what the capture recorded."""
    from atom_b200 import ops
    from atom_b200 import textgen as tg
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    P, hkv, G, theta = 32, 2, 8, 5e5
    shared = 180 * P                                               # 2 KV heads x 3 extra members x 5760 tokens: over the rule's bar
    pool = KvPoolInt4(1, hkv, 128, 260, P, torch.device(DEV))
    pool.buf.random_(0, 256)
    pool.param[..., 0].uniform_(0.01, 0.05)
    pool.param[..., 1].uniform_(0.0, 0.4)
    root = KvCacheInt4(pool, shared)
    forks = [root.fork() for _ in range(6)]
    for i, f in enumerate(forks):
        f.acquire(3 + 11 * i)
    lone = [KvCacheInt4(pool, n) for n in (70, 31, 200)]
    q = torch.from_numpy((np.random.default_rng(9).standard_normal((6, G * hkv, 128)) * 0.7).astype(np.float16)).to(DEV)
    model = _AttnStep(q, theta)
    calls = []
    real = ops._batch_decode_shared
    monkeypatch.setattr(ops, "_batch_decode_shared", lambda *a, **k: calls.append(1) or real(*a, **k))
    runner = tg.DecodeGraphRunner(model, pool, DEV, max_pages_per_seq=200)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    batches = [forks[:4] + lone[:2], forks[:5] + lone[:1], [forks[0], forks[2], forks[3], forks[5]] + lone[1:3]]
    batches += [batches[0]] * 2
    crossed = False
    for step, rows in enumerate(batches):
        for r in rows:
            crossed |= r.seqlen % P == 0                           # this step's token opens a page
            r.acquire_one()
        runner.run([0] * 6, rows)
        torch.cuda.synchronize()
        got = model.out.cpu().numpy()
        kv = BatchedKvCacheInt4(rows)
        assert len(kv.groups) == 1 and ops.decode_cascade(kv.groups, 6, P, hkv, G, sms), step
        want = ops.batch_decode_i4(q, kv, 0, rope_theta=theta).cpu().numpy()
        assert np.array_equal(_bits(got), _bits(want)), f"step {step}"
        if step == 0:
            assert len(calls) >= 1                                 # warm-up and capture ran the cascade
            captured = len(calls)
    assert len(runner._entries) == 1 and list(runner._entries) == [(6, 1)]
    assert len(calls) == captured + 4                              # the eager references only: replays make no host calls
    assert crossed


# ------------------------------------------------------------------------------------------------ 7. decoder-layer steps
@pytest.mark.timeout(900)
def test_decoder_layer_decode_step_on_forked_rows_runs_the_cascade(monkeypatch):
    """LlamaDecoderLayer steps (8 query heads, 2 KV heads, P = 32), each checked stage by stage by tests/layer_ref64.ModelRef with
    pool audits: a 3072-token root prefilled, 8 forks of it with continuation prompts beside 2 lone prompts, then two decode steps
    in which ops.decode_cascade picks the cascade, which runs inside LlamaAttention and is held to cascade_bound over the
    reference's shadow of the pool."""
    from atom_b200 import ops
    from atom_b200.kvcache import KvPoolInt4
    from tests import layer_ref64 as LR
    from tests.test_layer_ref64_cpu import Driver
    from tests.test_z_layer_ref64_gpu import _layer
    P, theta = 32, 5e5
    layer = _layer(1024, 1024, 8, 2, theta=theta)
    pool = KvPoolInt4(1, 2, 128, 140, P, torch.device(DEV))
    pool.buf.random_(0, 256)
    pool.param.view(torch.int16).random_(-32768, 32767)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    calls = []
    real = ops._batch_decode_shared
    monkeypatch.setattr(ops, "_batch_decode_shared", lambda *a, **k: calls.append(1) or real(*a, **k))
    ref = LR.ModelRef([LR.LayerParams(layer, 0)], P, prefill_rows={0: [0, 1, 31, 32, 33, 1500, 3071]}, sm_count=sms)
    d = Driver(monkeypatch, layer, pool, ref, ids=False)
    d.step([("R", 3072, None)])
    ref.prefill_rows = None
    for i in range(8):
        d.fork(f"F{i}", "R", total=1 + 9 * i)
    d.step([(f"F{i}", 1 + 9 * i, 1 + 9 * i) for i in range(8)] + [("L0", 45, 45), ("L1", 300, 300)])
    rows = [f"F{i}" for i in range(3)] + ["L0"] + [f"F{i}" for i in range(3, 8)] + ["L1"]
    d.step([], rows)
    d.step([], rows)
    assert len(calls) == 2 and ref.calls["cascade decode"] == 2 and "decode" not in ref.calls     # the cascade ran, twice
    print({k: round(v, 4) for k, v in sorted(ref.worst.items())})
