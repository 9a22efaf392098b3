"""Reference of speculative decoding's device side (include/atom_b200.h; DESIGN sections 5.7 and 5.8).

* `sample_draft_np` -- atom_sample_draft_f16's rule in numpy, built on tests/sample_ref64.py and tests/sample_penalty_ref64.py:
  the same keys, the same kept weights W (rules 1-4 and min-p, FP32 weights rounded to 2^-40, exact integer sums), Philox
  word 1 for the acceptance and word 0 for the draw after a rejection.  As sample_ref64.sample_np it is an exact sampler of the
  same semantics, not a bit model of the kernel (numpy's exp is not expf).
* `draft_ambiguous` -- whether a row's result could differ between two correct implementations of the rule: a top-p or min-p
  boundary, the acceptance test or the draw within sample_ref64.bound() of a decision.  Outside those regions the kernel and
  `sample_draft_np` must agree exactly.
* `propose_np` / `commit_propose_np` -- the prompt-lookup proposer and the commit, integers only, bit for bit the kernel's.
"""
import math

import numpy as np

from tests import sample_penalty_ref64 as RP
from tests import sample_ref64 as R


def _kept(row, T, k, p, m):
    """(order, W uint64 [V] with the non-kept tokens at 0) of a valid, non-greedy row: sample_penalty_ref64._sample_row's
    rules 3, min-p and 4, without the draw."""
    V = len(row)
    kk = R.order_keys(row)
    order = np.lexsort((np.arange(V), -kk))
    keep = np.ones(V, bool)
    if 0 < k < V:
        keep[:] = False
        keep[order[:k]] = True
    v32 = row.astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        x = ((v32 - v32[order[0]]).astype(np.float32) / np.float32(T)).astype(np.float32)
        w = np.exp(x).astype(np.float32)
    W = np.rint(w.astype(np.float64) * R.FIX)
    W[np.isneginf(row.astype(np.float64))] = 0
    if m > 0:
        keep &= W >= math.ceil(float(np.float32(m)) * R.FIX)
    W = W.astype(np.uint64) * keep
    if p < 1:
        tp = math.ceil(float(p) * float(int(W.sum())))
        Wo = W[order]
        M = np.concatenate([np.zeros(1, np.uint64), np.cumsum(Wo)[:-1]])
        n = int(np.count_nonzero(keep[order] & (M < np.uint64(tp))))
        keep2 = np.zeros(V, bool)
        keep2[order[:n]] = True
        W = W * keep2
    return order, W


def _invalid(row, T, k, p, m, d):
    kk = R.order_keys(row)
    return bool((kk > 0xFBFF).any() or (kk < 0x03FF).any() or (kk == 0x03FF).all() or R._bad_params(T, k, float(p)) or
                not 0 <= m <= 1 or d < -1 or d >= len(row))


def draft_row(row, T, k, p, key, ctr, d, m=0.0, faults=()):
    """One row of the rule.  faults (negative controls): 'accept_word0' (the acceptance reads word 0), 'keep_d' (the draw
    after a rejection keeps d), 'accept_le' (accept on <= instead of <)."""
    if _invalid(row, T, k, p, m, d):
        return -1
    if T == 0 or k == 1:
        return int(np.lexsort((np.arange(len(row)), -R.order_keys(row)))[0])
    _, W = _kept(row, T, k, p, m)
    if d >= 0:
        z = int(W.sum())
        wd = int(W[d])
        a = R.uniform53(key, ctr, 0 if "accept_word0" in faults else 1)
        t = (a * z) >> 53
        if t < wd or ("accept_le" in faults and t <= wd):
            return int(d)
        if "keep_d" not in faults:
            W = W.copy()
            W[d] = 0
    S = np.cumsum(W, dtype=np.uint64)
    t = (R.uniform53(key, ctr, 0) * int(S[-1])) >> 53
    return int(np.searchsorted(S, np.uint64(t), side="right"))


def sample_draft_np(logits, temperature, top_k, top_p, keys, counters, drafts, *, min_p=0.0, logprobs=None, faults=()):
    """ops.sample_tokens(..., drafts=) in numpy: int32 [B], or with logprobs (tokens, logprob, top_ids, top_logprobs)."""
    l16, T, K, P, KEY, CTR = R._params(logits, temperature, top_k, top_p, keys, counters)
    b = l16.shape[0]
    MP = R._rows(min_p, b, np.float32)
    D = R._rows(drafts, b, np.int64)
    n = 0 if logprobs is None else int(logprobs)
    out = np.empty(b, np.int32)
    lp = np.full(b, np.nan, np.float32)
    top_ids = np.full((b, n), -1, np.int32)
    top_lp = np.full((b, n), np.nan, np.float32)
    for i in range(b):
        out[i] = draft_row(l16[i], float(T[i]), int(K[i]), np.float32(P[i]), KEY[i], CTR[i], int(D[i]), float(MP[i]), faults)
        if out[i] >= 0 and logprobs is not None:
            lp[i], top_ids[i], top_lp[i] = RP._logprobs_row(l16[i], int(out[i]), n, ())
    return out if logprobs is None else (out, lp, top_ids, top_lp)


def sample_draft_tokens_np(logits, temperature, top_k, top_p, keys, counters, *, drafts, min_p=0.0, logprobs=None):
    """ops.sample_tokens' signature (with drafts) over sample_draft_np, for host-only tests: torch tensors on the logits'
    device."""
    import torch
    dev = logits.device if hasattr(logits, "device") else "cpu"
    r = sample_draft_np(logits, temperature, top_k, top_p, keys, counters, drafts, min_p=min_p, logprobs=logprobs)
    if isinstance(r, tuple):
        return tuple(torch.from_numpy(x).to(dev) for x in r)
    return torch.from_numpy(r).to(dev)


def draft_ambiguous(row, T, k, p, key, ctr, d, m=0.0):
    """True when a correct kernel may give another token than sample_draft_np on this row: the float64 weights
    w_i = exp((l_i - max) / T) put a top-p boundary, a min-p threshold, the acceptance test floor(a Z) < W_d or an edge of the
    draw's inverse CDF within sample_ref64.bound() (in units of the top weight, 2^40) of the value it is compared with."""
    if _invalid(row, T, k, p, m, d) or T == 0 or k == 1:
        return False
    v = row.astype(np.float64)
    V = len(v)
    order = R.total_order(v)
    nk = V if k == 0 or k >= V else k
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        w = np.exp((v[order[:nk]] - v[order[0]]) / T)
    w[np.isneginf(v[order[:nk]])] = 0.0
    if m > 0:
        mm = float(np.float32(m))
        if np.any(np.abs(w - mm) <= R.RHO * w + 2 * R.ALPHA):
            return True
        w = np.where(w >= mm, w, 0.0)
    z = float(w.sum())
    n = nk
    if p < 1:
        M = np.concatenate([[0.0], np.cumsum(w)[:-1]])
        bd = R.bound(z, nk)
        lo_, hi_ = int(np.count_nonzero(M < p * z - bd)), int(np.count_nonzero(M < p * z + bd))
        if lo_ != hi_:
            return True
        n = max(1, lo_)
        w = np.concatenate([w[:n], np.zeros(nk - n)])
        z = float(w.sum())
    full = np.zeros(V)
    full[order[:nk]] = w
    bd = R.bound(z, n)
    if d >= 0:
        x = R.uniform53(key, ctr, 1) * 2.0 ** -53 * z
        if abs(x - full[d]) <= bd:
            return True
        if x < full[d]:
            return False
        full[d] = 0.0
    S = np.cumsum(full)
    x = R.uniform53(key, ctr, 0) * 2.0 ** -53 * float(S[-1])
    return bool(np.any(np.abs(S[full > 0] - x) <= bd))


def propose_np(h, k, nmin, nmax):
    """The drafts prompt lookup proposes after history h (a sequence of ints): for n = nmax down to nmin, the latest p with
    p + n <= L - 1 and h[p:p+n] == h[L-n:L] gives h[p+n : min(p+n+k, L)]; the first n with a match wins; else []."""
    h = [int(t) for t in h]
    L = len(h)
    for n in range(nmax, nmin - 1, -1):
        if n > L:
            continue
        tail = h[L - n:]
        for q in range(L - 1 - n, -1, -1):
            if h[q:q + n] == tail:
                return h[q + n:min(q + n + k, L)]
    return []


def _np(x):
    return x.numpy() if hasattr(x, "numpy") else np.asarray(x)


def commit_propose_np(tokens, cands, row_indptr, slots, history, lengths, out, num_draft, ngram_min, ngram_max):
    """ops.spec_commit_propose in numpy: history / lengths / out are numpy arrays or CPU torch tensors, updated in place."""
    tok, cand, ip, sl = (np.asarray(_np(x)).astype(np.int64).reshape(-1) for x in (tokens, cands, row_indptr, slots))
    H, Ln, O = _np(history), _np(lengths), _np(out)
    k = int(num_draft)
    cap = H.shape[1]
    for i in range(len(ip) - 1):
        s = int(sl[i])
        o = O[i]
        o[:] = -1
        r0, last = int(ip[i]), min(int(ip[i + 1]) - int(ip[i]), k + 1) - 1
        m = 0
        while m < last and cand[r0 + m] >= 0 and tok[r0 + m] == cand[r0 + m]:
            m += 1
        e = 0 if last < 0 else m + 1
        L = int(Ln[s])
        for j in range(e):
            o[2 + j] = tok[r0 + j]
            if L < cap:
                H[s, L] = tok[r0 + j]
                L += 1
        Ln[s] = L
        dr = propose_np(H[s, :L], k, int(ngram_min), int(ngram_max))
        o[0], o[1] = e, len(dr)
        o[k + 3:k + 3 + len(dr)] = dr
    return out
