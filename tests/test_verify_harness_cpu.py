"""CPU checks of the host side of a verify step: BatchLenInfo with decode_len, and KvCacheInt4.truncate (pages returned,
reference counts consistent, no cut into a shared page)."""
import pytest
import torch

from atom_b200.cat_tensor import BatchLenInfo
from atom_b200.kvcache import KvCacheInt4, KvPoolInt4

CPU = torch.device("cpu")


def test_batch_len_info_default_is_unchanged_and_decode_len_sets_the_stride():
    a = BatchLenInfo([3, 4], 5, CPU)
    assert (a.decode, a.decode_len, a.doff, a.decode_indptr) == (5, 1, 7, None)
    b = BatchLenInfo([], 3, CPU, decode_len=4)
    assert (b.decode, b.decode_len, b.doff, b.indptr) == (3, 4, 0, None)
    assert b.decode_indptr.tolist() == [0, 4, 8, 12]
    assert b.max_len is None and BatchLenInfo([], 3, CPU, decode_len=4, max_len=700).max_len == 700
    with pytest.raises(ValueError):
        BatchLenInfo([], 3, CPU, decode_len=9)
    with pytest.raises(ValueError):
        BatchLenInfo([], 3, CPU, decode_len=4, max_len=3)


def _pool(capacity=12, P=4):
    return KvPoolInt4(1, 1, 128, capacity, P, CPU)


def test_truncate_returns_emptied_pages_and_keeps_refcounts():
    pool = _pool()
    c = KvCacheInt4(pool, 5)
    c.acquire(6)                                     # 11 tokens: 3 pages
    pages = list(c.indicies)
    free = pool.num_free_blocks
    assert c.truncate(11) == [] and c.seqlen == 11
    assert c.truncate(8) == [pages[2]] and c.seqlen == 8 and c.indicies == pages[:2]
    assert pool.num_free_blocks == free + 1
    assert c.truncate(6) == [] and c.indicies == pages[:2]
    for p in pages[:2]:
        assert pool.refcount(p) == 1
    c.acquire(3)                                     # grows into a fresh page again
    assert c.seqlen == 9 and len(c.indicies) == 3
    c.release()
    assert pool.num_free_blocks == pool.capacity
    with pytest.raises(ValueError):
        KvCacheInt4(pool, 2).truncate(3)


def test_truncate_never_cuts_into_a_shared_page():
    pool = _pool()
    root = KvCacheInt4(pool, 8)                      # two full pages
    child = root.fork()
    child.acquire(3)                                 # 11 tokens: the two shared pages and a private one
    shared = root.indicies[:2]
    dropped = child.truncate(8)
    assert dropped and child.seqlen == 8 and child.indicies == shared
    with pytest.raises(ValueError):
        child.truncate(6)                            # the next token would be written into a shared page
    assert child.truncate(4) == [shared[1]]          # a page boundary: the child just lets go of the second page
    assert pool.refcount(shared[1]) == 1 and pool.refcount(shared[0]) == 2
    child.release()
    root.release()
    assert pool.num_free_blocks == pool.capacity
