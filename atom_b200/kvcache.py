"""Paged INT4 KV cache: page pool, per-sequence page lists and the per-step page table.

API-compatible with /root/reference/e2e/punica-atom/punica/utils/kvcache.py:6-127 (class, property and method names are
what punica/models/llama.py and the benchmark harness touch), laid out for the CUDA kernels:

    pool.buf    uint8   [pages, num_layers, 2 (K|V), num_heads, block_len, head_dim // 2]   two INT4 per byte
    pool.param  float16 [pages, num_layers, 2,       num_heads, block_len, 2]               (scale, zero): x = nibble*scale - zero

so that one (page, layer, K-or-V, head) block is `block_len * 64` contiguous bytes -- exactly what the decode kernel
streams with one cp.async.bulk (kv_kernels.cuh).  Differences in mechanism, none in meaning:
  * pages are handed out from a LIFO stack (most recently freed first: still warm in L2), exhaustion raises;
  * the step's page table (CSR indptr / indicies / last_page_offset) is assembled in ONE int32 host buffer and shipped with
    ONE (blocking) host->device copy; the three tensors the kernels read are views into it.
Prefix sharing (EXTENSION): pages carry reference counts, and `KvCacheInt4.fork` starts a sequence on its parent's full pages.
RoPE is applied from page positions and K/V are quantised per token, so a shared page holds the same bytes for every holder;
a shared page is always full, so no holder ever writes into one.  A batch in which forked sequences meet records its prefix
groups (`BatchedKvCacheInt4.groups`) for the cascade decode (ops.batch_decode_i4).
"""
from typing import List, Sequence, Tuple

import numpy as np
import torch


class KvPoolInt4:
    def __init__(self, num_layers: int, num_heads: int, head_dim: int, capacity: int, block_len: int, device: torch.device):
        if head_dim % 2:
            raise ValueError("head_dim must be even (two INT4 per byte)")
        shape = (capacity, num_layers, 2, num_heads, block_len)
        self._buf = torch.empty(shape + (head_dim // 2,), dtype=torch.uint8, device=device)
        self._param = torch.empty(shape + (2,), dtype=torch.float16, device=device)
        self._stack: List[int] = list(range(capacity - 1, -1, -1))      # pop() hands out page 0 first
        self._refs = [0] * capacity                                       # holders of each page (0: on the stack)

    # ---- storage
    @property
    def buf(self) -> torch.Tensor:
        return self._buf

    @property
    def param(self) -> torch.Tensor:
        return self._param

    @property
    def device(self) -> torch.device:
        return self._buf.device

    @property
    def capacity(self) -> int:
        return self._buf.shape[0]

    @property
    def num_layers(self) -> int:
        return self._buf.shape[1]

    @property
    def block_len(self) -> int:
        return self._buf.shape[4]

    # ---- page accounting
    @property
    def num_free_blocks(self) -> int:
        return len(self._stack)

    def alloc_block(self) -> int:
        if not self._stack:
            raise RuntimeError(f"KvPoolInt4: out of pages (capacity {self.capacity})")
        page = self._stack.pop()
        self._refs[page] = 1
        return page

    def share_block(self, idx: int) -> None:
        """One more holder of an allocated page."""
        self.refcount(idx)
        self._refs[idx] += 1

    def free_block(self, idx: int) -> None:
        """Drop one holder; the page goes back to the stack with its last holder."""
        if self.refcount(idx) == 1:
            self._stack.append(idx)
        self._refs[idx] -= 1

    def refcount(self, idx: int) -> int:
        """Holders of an allocated page; raises for a page that is not allocated."""
        if not 0 <= idx < self.capacity or not self._refs[idx]:
            raise ValueError(f"KvPoolInt4: page {idx} is not allocated")
        return self._refs[idx]


class KvCacheInt4:
    """One sequence: the pages it owns, in order, and how many tokens they hold."""

    def __init__(self, pool: KvPoolInt4, init_len: int):
        if init_len < 0:
            raise ValueError("init_len must be non-negative")
        self._pool = pool
        self._pages: List[int] = []
        self._seqlen = 0
        self._grow_to(init_len)

    def _grow_to(self, seqlen: int) -> None:
        if seqlen > self._seqlen and self._seqlen % self._pool.block_len:
            # the next tokens are written into the partly filled last page: it must be this sequence's alone
            assert self._pool.refcount(self._pages[-1]) == 1, "KvCacheInt4: a shared page would be written"
        need = -(-seqlen // self._pool.block_len)
        while len(self._pages) < need:
            self._pages.append(self._pool.alloc_block())
        self._seqlen = seqlen

    @property
    def pool(self) -> KvPoolInt4:
        return self._pool

    @property
    def seqlen(self) -> int:
        return self._seqlen

    @property
    def indicies(self) -> List[int]:          # (sic) the reference's spelling is part of the interface
        return self._pages

    @property
    def last_page_offset(self) -> int:
        """Tokens in the last page, in [1, block_len] (the kernels' convention; 0 tokens also reports block_len)."""
        return (self._seqlen - 1) % self._pool.block_len + 1

    def acquire_one(self) -> None:
        """Make room for one more token; a page is added when the last one is full."""
        self._grow_to(self._seqlen + 1)

    def acquire(self, n: int) -> None:
        """Make room for n more tokens (a prompt chunk, a continuation); pages are added as the last one fills."""
        if n < 0:
            raise ValueError("acquire: n must be non-negative")
        self._grow_to(self._seqlen + int(n))

    def truncate(self, n: int) -> List[int]:
        """Drop the tokens past the first n (the rejected drafts of a verify step) and return the pages that no longer hold one
        of this sequence's tokens; this sequence's hold on each is given back to the pool.  The bytes past n stay as they are
        and are overwritten by the next write, as any slot past the length.  Refuses to leave the length inside a shared page:
        the next token would be written into it."""
        n = int(n)
        if not 0 <= n <= self._seqlen:
            raise ValueError(f"truncate: n={n} outside [0, {self._seqlen}]")
        P = self._pool.block_len
        keep = -(-n // P)
        if n % P and n < self._seqlen and self._pool.refcount(self._pages[keep - 1]) > 1:
            raise ValueError(f"truncate: n={n} cuts into shared page {self._pages[keep - 1]}")
        dropped = self._pages[keep:]
        del self._pages[keep:]
        for page in reversed(dropped):
            self._pool.free_block(page)
        self._seqlen = n
        return dropped

    def fork(self, n=None, copies=None) -> "KvCacheInt4":
        """A new sequence holding this one's first `n` tokens (default: all).  It shares the full pages among them; a partly
        filled last page is copied, every layer and K/V block, into a fresh page of its own (one device copy on the current
        stream).  Both sequences then grow independently.  copies: a list to defer that copy to, as (src page, dst page, slots),
        e.g. for ops.copy_kv_pages; it must then run before either sequence writes another token."""
        n = self._seqlen if n is None else int(n)
        if not 0 <= n <= self._seqlen:
            raise ValueError(f"fork: n={n} outside [0, {self._seqlen}]")
        pool = self._pool
        child = KvCacheInt4(pool, 0)
        full = n // pool.block_len
        for page in self._pages[:full]:
            pool.share_block(page)
            child._pages.append(page)
        if n % pool.block_len:
            page = pool.alloc_block()
            child._pages.append(page)
            if copies is not None:
                copies.append((self._pages[full], page, n % pool.block_len))
            else:
                pool.buf[page].copy_(pool.buf[self._pages[full]])
                pool.param[page].copy_(pool.param[self._pages[full]])
        child._seqlen = n
        return child

    def release(self) -> None:
        """Give every page back to the pool."""
        while self._pages:
            self._pool.free_block(self._pages.pop())
        self._seqlen = 0


class BatchedKvCacheInt4:
    """Page table of one step's batch, in the CSR form the kernels read (all int32, on the pool's device)."""

    def __init__(self, kv: Sequence[KvCacheInt4]):
        if len(kv) == 0:
            raise ValueError("empty batch")
        pool = kv[0].pool
        if any(c.pool is not pool for c in kv):
            raise ValueError("all sequences of a batch must live in the same pool")
        b = len(kv)
        counts = np.fromiter((len(c.indicies) for c in kv), dtype=np.int64, count=b)
        nnz = int(counts.sum())
        self.groups = prefix_groups(kv)
        ng = len(self.groups)
        extra = ng + 1 + sum(len(m) for m, _ in self.groups) + b if ng else 0
        # [indptr (b+1) | last_page_offset (b) | indicies (nnz)], and with prefix groups also
        # [group_indptr (ng+1) | group_members | shared_pages (b)]
        table = np.empty(2 * b + 1 + nnz + extra, dtype=np.int32)
        table[0] = 0
        np.cumsum(counts, out=table[1:b + 1])
        table[b + 1:2 * b + 1] = [c.last_page_offset for c in kv]
        pos = 2 * b + 1
        for c in kv:
            n = len(c.indicies)
            table[pos:pos + n] = c.indicies
            pos += n
        if ng:
            gi = pos
            table[gi] = 0
            table[gi + 1:gi + ng + 1] = np.cumsum([len(m) for m, _ in self.groups])
            pos = gi + ng + 1
            shared = np.zeros(b, dtype=np.int32)
            for members, n in self.groups:
                table[pos:pos + len(members)] = members
                pos += len(members)
                shared[members] = n
            table[pos:pos + b] = shared
        # a blocking copy: when the constructor returns the table is valid for every stream (callers hand the object to
        # side streams and CUDA-graph captures); the steady-state decode loop does not come through here at all
        # (textgen.DecodeGraphRunner keeps its table in a static buffer)
        dev = torch.from_numpy(table).to(pool.device)
        self._table = dev                                             # keeps the views alive
        self.data = pool.buf
        self.param = pool.param
        self.indptr = dev[:b + 1]
        self.last_page_offset = dev[b + 1:2 * b + 1]
        self.indicies = dev[2 * b + 1:2 * b + 1 + nnz]
        # prefix groups on the device (None without groups): members of group i are group_members[group_indptr[i] ..
        # group_indptr[i+1]], and shared_pages[r] is the number of leading pages row r shares with its group (0: no group)
        self.group_indptr = self.group_members = self.shared_pages = None
        if ng:
            gi = 2 * b + 1 + nnz
            self.group_indptr = dev[gi:gi + ng + 1]
            self.group_members = dev[gi + ng + 1:len(table) - b]
            self.shared_pages = dev[len(table) - b:]
        # host copy of every sequence's length at construction: the prefill over a cached prefix needs each prompt's position
        # in its sequence (seqlens[b] - prompt length) for the RoPE positions and the table size without reading the device
        self.seqlens: List[int] = [c.seqlen for c in kv]

    @property
    def page_size(self) -> int:
        return self.data.size(-2)


def prefix_groups(kv: Sequence[KvCacheInt4]) -> List[Tuple[List[int], int]]:
    """Prefix groups of a batch: (rows, shared page count) for every set of at least two rows that begin on the same page,
    which only a fork makes happen.  The count is the number of leading pages all members hold in common; those pages are
    full.  One level of sharing: a row is in at most one group, ordered by its first row."""
    by_first = {}
    for r, c in enumerate(kv):
        if c.indicies:
            by_first.setdefault(c.indicies[0], []).append(r)
    groups = []
    for rows in by_first.values():
        if len(rows) < 2:
            continue
        n = min(len(kv[r].indicies) for r in rows)
        first = kv[rows[0]].indicies
        for r in rows[1:]:
            pages = kv[r].indicies
            if pages[:n] != first[:n]:                  # (one list comparison when the members agree, as forks of one root do)
                n = next(i for i in range(n) if pages[i] != first[i])
        groups.append((rows, n))
    groups.sort(key=lambda g: g[0][0])
    return groups
