"""BatchLenInfo -- same surface as /root/reference/e2e/punica-atom/punica/utils/cat_tensor.py:26-66: a step's batch is the
concatenation of the prefill prompts' tokens followed by one token per decoding sequence.  EXTENSION (speculative decoding):
with decode_len = S > 1 every decoding sequence carries S tokens (its last token and its drafts), decode * S rows in all."""
from typing import Sequence

import torch


class BatchLenInfo:
    def __init__(self, prefills: Sequence[int], decode: int, indptr_device: torch.device, indptr_dtype: torch.dtype = torch.int32,
                 decode_len: int = 1, max_len=None):
        if not 1 <= decode_len <= 8:
            raise ValueError(f"decode_len={decode_len} must be in [1, 8]")
        if max_len is not None and int(max_len) < decode_len:
            raise ValueError(f"max_len={max_len} must be at least decode_len={decode_len}")
        self._max_len = None if max_len is None else int(max_len)
        self._prefills = list(prefills)
        self._decode = decode
        self._decode_len = decode_len
        # the verify step's K/V rows go to the cache with init_kv_i4 at stride decode_len
        self._decode_indptr = None if decode_len == 1 else \
            torch.arange(0, decode * decode_len + 1, decode_len, dtype=indptr_dtype, device=indptr_device)
        if len(self._prefills) > 0:
            cum = [0]
            for n in self._prefills:
                cum.append(cum[-1] + n)
            self._indptr = torch.tensor(cum, dtype=indptr_dtype, device=indptr_device)
            self._doff = cum[-1]
        else:
            self._indptr = None
            self._doff = 0

    @property
    def prefills(self) -> list:
        """Length of each prefill request."""
        return self._prefills

    @property
    def decode(self) -> int:
        """Number of decode requests."""
        return self._decode

    @property
    def decode_len(self) -> int:
        """Tokens each decode request carries (1: a plain decode step; S > 1: a verify step)."""
        return self._decode_len

    @property
    def decode_indptr(self):
        """[0, S, 2S, ..., decode * S] on the device for decode_len = S > 1; None for a plain decode step."""
        return self._decode_indptr

    @property
    def max_len(self):
        """A bound on every decoding sequence's length that a verify step sizes its RoPE table from (ops.batch_verify_i4's
        `max_len`).  A CUDA graph of the step stays valid while the lengths stay within it.  None: the verify step reads the
        lengths the page table recorded on the host (BatchedKvCacheInt4.seqlens), which holds only for the step it was built for."""
        return self._max_len

    @property
    def doff(self) -> int:
        """Index of the first decode token == total length of the prefills."""
        return self._doff

    @property
    def indptr(self):
        """indptr[i] = sum(prefills[:i]); None without prefill."""
        return self._indptr
