"""CPU suite: prefix sharing in the paged INT4 KV cache (reference counts, fork, the prefix groups of a batch and their bytes in
the page table) and the two host-side rules of the shared-prefix decode: when ops.batch_decode_i4 picks the cascade, and how many
chunks its prefix pass takes.  Pools live on the CPU; no kernel is launched."""
import itertools

import numpy as np
import pytest
import torch

from atom_b200 import _lib, ops
from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4

CPU = torch.device("cpu")


def _pool(capacity=64, block_len=16, layers=2, heads=2):
    p = KvPoolInt4(layers, heads, 128, capacity, block_len, CPU)
    g = torch.Generator().manual_seed(0)
    p.buf.copy_(torch.randint(0, 256, p.buf.shape, dtype=torch.uint8, generator=g))
    p.param.copy_(torch.randn(p.param.shape, generator=g).half())
    return p


def _legacy_table(kv):
    """The page table as the batch built it before prefix groups: [indptr | last_page_offset | indicies]."""
    counts = [len(c.indicies) for c in kv]
    return np.concatenate([np.cumsum([0] + counts), [c.last_page_offset for c in kv],
                           [p for c in kv for p in c.indicies]]).astype(np.int32)


def test_fork_shares_full_pages_and_copies_the_partial_page_of_every_layer():
    pool = _pool()
    root = KvCacheInt4(pool, 40)                                   # pages: 16 + 16 + 8 tokens
    free = pool.num_free_blocks
    child = root.fork()
    assert child.seqlen == 40 and child.indicies[:2] == root.indicies[:2]
    assert child.indicies[2] != root.indicies[2]
    assert pool.num_free_blocks == free - 1                        # only the partial page is new
    assert [pool.refcount(p) for p in root.indicies] == [2, 2, 1]
    src, dst = root.indicies[2], child.indicies[2]
    assert torch.equal(pool.buf[src], pool.buf[dst]) and torch.equal(pool.param[src].view(torch.int16), pool.param[dst].view(torch.int16))
    assert pool.buf[dst].shape[:2] == (pool.num_layers, 2)         # every layer, K and V

    half = root.fork(16)                                           # a page boundary: nothing copied
    assert half.indicies == root.indicies[:1] and pool.num_free_blocks == free - 1
    none = root.fork(0)
    assert none.indicies == [] and none.seqlen == 0
    with pytest.raises(ValueError):
        root.fork(41)


def test_release_order_does_not_matter_and_the_pool_ends_full():
    for order in itertools.permutations(range(4)):
        pool = _pool()
        root = KvCacheInt4(pool, 37)
        seqs = [root, root.fork(), root.fork(32), root.fork(5)]
        seqs[1].acquire(20)
        seqs[2].acquire_one()
        for i in order:
            seqs[i].release()
        assert pool.num_free_blocks == pool.capacity, order
        assert sorted(pool._stack) == list(range(pool.capacity))


def test_double_release_raises():
    pool = _pool()
    root = KvCacheInt4(pool, 32)
    child = root.fork()
    page = root.indicies[0]
    pool.free_block(page)                                          # the root's hold
    pool.free_block(page)                                          # the child's hold: back on the stack
    with pytest.raises(ValueError):
        pool.free_block(page)
    with pytest.raises(ValueError):
        pool.share_block(page)
    with pytest.raises(ValueError):
        pool.free_block(pool.capacity)
    del child


def test_pages_handed_out_for_writing_are_never_shared():
    pool = _pool()
    root = KvCacheInt4(pool, 40)
    kids = [root.fork() for _ in range(3)] + [root.fork(32), root.fork(16), root.fork(21)]
    for s in [root] + kids:
        for n in (1, 7, 16, 33):
            first_written = s.seqlen
            s.acquire(n)
            for t in range(first_written, s.seqlen):
                assert pool.refcount(s.indicies[t // pool.block_len]) == 1
    # a sequence whose last page is shared and partly filled cannot be grown: the host check fires before any write
    pool2 = _pool()
    a = KvCacheInt4(pool2, 20)
    b = KvCacheInt4(pool2, 0)
    pool2.share_block(a.indicies[1])
    b._pages.append(a.indicies[1])
    b._seqlen = 20
    with pytest.raises(AssertionError):
        b.acquire_one()


def test_batch_without_forks_builds_todays_table_byte_for_byte():
    pool = _pool(capacity=256)
    for lens in ([1], [5, 16, 17], [40, 1, 64, 33, 0 + 3]):
        kv = [KvCacheInt4(pool, n) for n in lens]
        b = BatchedKvCacheInt4(kv)
        assert b.groups == [] and b.group_indptr is None and b.group_members is None and b.shared_pages is None
        assert b._table.numpy().tobytes() == _legacy_table(kv).tobytes()
        assert b.indicies.numel() == sum(len(c.indicies) for c in kv)
        for c in kv:
            c.release()
    # two sequences forked from one root but not in the same batch form no group either
    root = KvCacheInt4(pool, 48)
    kid = root.fork()
    kid.acquire(3)
    for kv in ([root, KvCacheInt4(pool, 9)], [kid]):
        b = BatchedKvCacheInt4(kv)
        assert b.groups == [] and b._table.numpy().tobytes() == _legacy_table(kv).tobytes()


def test_group_tables_of_a_mixed_batch():
    pool = _pool(capacity=256)
    r1 = KvCacheInt4(pool, 40)        # 2 full pages + 8 tokens
    r2 = KvCacheInt4(pool, 64)        # 4 full pages
    lone_a, lone_b = KvCacheInt4(pool, 30), KvCacheInt4(pool, 3)
    g1 = [r1.fork() for _ in range(3)]
    g2 = [r2.fork(), r2.fork(50), r2.fork(64)]
    for i, s in enumerate(g1 + g2):
        s.acquire(1 + 9 * i)
    rows = [lone_a, g1[0], g2[0], g1[1], lone_b, g2[1], g1[2], g2[2]]
    b = BatchedKvCacheInt4(rows)
    assert b.groups == [([1, 3, 6], 2), ([2, 5, 7], 3)]            # g2[1] forked at 50 tokens shares 3 pages
    t = b._table.numpy()
    legacy = _legacy_table(rows)
    assert t[:len(legacy)].tobytes() == legacy.tobytes()           # today's table first, unchanged
    assert b.group_indptr.tolist() == [0, 3, 6]
    assert b.group_members.tolist() == [1, 3, 6, 2, 5, 7]
    assert b.shared_pages.tolist() == [0, 2, 3, 2, 0, 3, 2, 3]
    assert len(t) == len(legacy) + 3 + 6 + 8
    # the views are the table's own storage (one copy to the device)
    for v in (b.indptr, b.last_page_offset, b.indicies, b.group_indptr, b.group_members, b.shared_pages):
        assert v.untyped_storage().data_ptr() == b._table.untyped_storage().data_ptr()
    # the shared pages are full and identical for every member
    for members, n in b.groups:
        pages = [rows[m].indicies[:n] for m in members]
        assert all(p == pages[0] for p in pages) and all(rows[m].seqlen >= n * pool.block_len for m in members)
    # the group's root in the batch joins it
    b2 = BatchedKvCacheInt4([r1, g1[0]])
    assert b2.groups == [([0, 1], 2)]


def _cascade_rule(groups, batch, page_size, kv_heads, g, sms):
    """The cascade runs when more than half of the rows are group members, every group has at least 16 query rows per KV head
    (members x G), and num_kv_heads x sum over groups of (members - 1) x shared tokens >= 256 x SMs."""
    members = sum(len(r) for r, _ in groups)
    saved = kv_heads * sum((len(r) - 1) * n * page_size for r, n in groups)
    return bool(groups) and 2 * members > batch and min(len(r) for r, _ in groups) * g >= 16 and saved >= 256 * sms


def test_cascade_rule_matches_its_statement_over_a_grid():
    seen = set()
    for sms, kvh, g, p in itertools.product((1, 66, 132, 133), (1, 8, 32), (1, 2, 4, 8), (8, 16, 32, 64)):
        for members, pages in itertools.product((2, 3, 4, 8, 16, 32), (1, 2, 16, 33, 512)):
            for ngroups, lone in itertools.product((1, 2, 5), (0, 1, 8)):
                groups = [(list(range(k * members, (k + 1) * members)), pages) for k in range(ngroups)]
                batch = members * ngroups + lone * members * ngroups // 4 + lone
                got = ops.decode_cascade(groups, batch, p, kvh, g, sms)
                assert got == _cascade_rule(groups, batch, p, kvh, g, sms), (sms, kvh, g, p, members, pages, ngroups, lone)
                seen.add(got)
    assert seen == {True, False}
    assert not ops.decode_cascade([], 4, 32, 8, 4, 132)
    # the thresholds on a 132-SM card, 8 KV heads, G = 4, 32-token pages: 33792 token-heads saved
    four = list(range(4))
    assert not ops.decode_cascade([(four, 43)], 4, 32, 8, 4, 132) and ops.decode_cascade([(four, 44)], 4, 32, 8, 4, 132)
    assert not ops.decode_cascade([(four, 44)], 8, 32, 8, 4, 132) and ops.decode_cascade([(four, 44)], 7, 32, 8, 4, 132)
    assert not ops.decode_cascade([(four[:3], 4096)], 3, 32, 8, 4, 132)          # 12 rows per KV head
    assert ops.decode_cascade([(four[:2], 4096)], 2, 32, 8, 8, 132)              # 16 rows per KV head
    assert not ops.decode_cascade([(four, 512), (four[:2], 512)], 6, 32, 8, 4, 132)   # one group of 8 rows


def test_prefix_chunk_count_rule():
    l = _lib.lib()
    for sms, ng, b, g, kvh in itertools.product((1, 131, 132, 133), (1, 2, 3, 32), (2, 16, 17, 32, 64), (1, 4, 8), (1, 2, 8, 32)):
        assert l.atom_decode_shared_chunks(ng, b, g, kvh, sms) == -(-2 * sms // (ng * -(-b * g // 64) * kvh))
    assert l.atom_decode_shared_chunks(1, 32, 4, 8, 132) == 17 and l.atom_decode_shared_chunks(16, 32, 4, 8, 132) == 2
    for bad in ((0, 1, 1, 1, 1), (1, 0, 1, 1, 1), (1, 1, 0, 1, 1), (1, 1, 1, 0, 1), (1, 1, 1, 1, 0)):
        assert l.atom_decode_shared_chunks(*bad) < 0
