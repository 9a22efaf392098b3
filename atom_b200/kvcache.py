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
"""
from typing import List, Sequence

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
        self._in_use = bytearray(capacity)

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
        self._in_use[page] = 1
        return page

    def free_block(self, idx: int) -> None:
        if not 0 <= idx < self.capacity or not self._in_use[idx]:
            raise ValueError(f"KvPoolInt4: page {idx} is not allocated")
        self._in_use[idx] = 0
        self._stack.append(idx)


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
        table = np.empty(2 * b + 1 + nnz, dtype=np.int32)             # [indptr (b+1) | last_page_offset (b) | indicies (nnz)]
        table[0] = 0
        np.cumsum(counts, out=table[1:b + 1])
        table[b + 1:2 * b + 1] = [c.last_page_offset for c in kv]
        pos = 2 * b + 1
        for c in kv:
            n = len(c.indicies)
            table[pos:pos + n] = c.indicies
            pos += n
        # a blocking copy: when the constructor returns the table is valid for every stream (callers hand the object to
        # side streams and CUDA-graph captures); the steady-state decode loop does not come through here at all
        # (textgen.DecodeGraphRunner keeps its table in a static buffer)
        dev = torch.from_numpy(table).to(pool.device)
        self._table = dev                                             # keeps the views alive
        self.data = pool.buf
        self.param = pool.param
        self.indptr = dev[:b + 1]
        self.last_page_offset = dev[b + 1:2 * b + 1]
        self.indicies = dev[2 * b + 1:]
        # host copy of every sequence's length at construction: the prefill over a cached prefix needs each prompt's position
        # in its sequence (seqlens[b] - prompt length) for the RoPE positions and the table size without reading the device
        self.seqlens: List[int] = [c.seqlen for c in kv]

    @property
    def page_size(self) -> int:
        return self.data.size(-2)
