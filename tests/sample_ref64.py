"""Reference of atom_sample_f16 / ops.sample_tokens (include/atom_b200.h; DESIGN section 5.6).

Two things live here:

* `sample_np` -- the sampler's algorithm restated in numpy: the same keys, the same FP32 weight formula rounded to the same
  2^-40 fixed point, the same integer sums and the same draw.  numpy's float32 `exp` is not CUDA's `expf`, so it is not a bit
  model of the kernel; it is an exact sampler of the same semantics, used where the host logic needs a sampler without a GPU
  (the serving harness's CPU tests) and to show that the checker below rejects faulty samplers (`faults=`).

* `check_tokens` -- the float64 reference that every token the kernel returns must pass.  The kept sets of the greedy and
  top-k rules are exact (no tolerance).  The top-p boundary and the inverse-CDF intervals are computed in float64 from the
  exact probabilities p_i = exp((l_i - max) / T) and widened by `bound()`:

  The kernel's weight of token i is W_i = round(expf(fl(fl(l_i - m) / T)) * 2^40) (m the row maximum, exact in FP16).  In units
  of 2^40, |W_i - w_i| <= rho * w_i + alpha, w_i = exp((l_i - m) / T) exact:
    - fl(l_i - m): one FP32 rounding, relative u = 2^-24;  fl(. / T): one more.  So the exponent x carries |dx| <= (2u + u^2)|x|;
      while w_i is representable (x >= -104, below that expf is 0 or subnormal), |dx| <= 2.0000001 * 2^-24 * 104 = 1.2398e-5
      and exp turns it into a relative 1.2399e-5;
    - expf: at most 2 ulp (CUDA Programming Guide, maximum ulp errors), relative 2^-22;
    rho = (1 + 1.2399e-5)(1 + 2^-22) - 1 < 1.27e-5;
    - the integer rounding at 2^-40, half a unit, plus the subnormal/zero results of expf below 2^-126: alpha = 2^-40.
  Sums of W are exact integers.  A sum S' over n tokens of exact value S: |S' - S| <= rho * S + n * alpha.
    - top-p: the kernel keeps the token at place j of the order iff M'_j < ceil(fl(fl(p) * fl(Z'))) (M' the exclusive mass,
      Z' the top-k total; fl the double conversions and product, 3 roundings of 2^-53, and the ceil, one unit of 2^-40);
      so |(M'_j - p Z') - (M_j - p Z)| <= rho (M_j + p Z) + 2 n alpha + 2^-40 + 3 * 2^-53 Z;
    - draw: the kernel picks j with S'_{j-1} <= floor(u Z') < S'_j (the floor: one unit of 2^-40, the product is exact), so
      S_{j-1} - d <= u Z < S_j + d with d = rho (S + u Z) + 2 n alpha + 2^-40;
    - the float64 reference's own cumulative sums: n * 2^-53 * Z.
  Both rules use  bound(Z, n) = 2 rho Z + 2 n alpha + 2^-40 + (n + 3) * 2^-53 * Z  (S, M, p Z are all <= Z).
  A draw within bound() of another token's interval, or a top-p set whose boundary is within bound(), is *ambiguous*: the
  checker accepts any token consistent with some admissible set and counts the row, so the fraction can be reported.
"""
import math

import numpy as np

RHO = 1.27e-5
ALPHA = 2.0 ** -40
FIX = 2.0 ** 40

PHILOX_M = (0xD2E7470EE14C6C93, 0xCA5A826395121157)
PHILOX_W = (0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B)
_M64 = (1 << 64) - 1


def philox4x64_10(key, counter):
    """Philox4x64-10 (Salmon, Moraes, Dror, Shaw, SC'11; Random123's constants): the four 64-bit words of the block at
    `counter` (4 words) under `key` (2 words)."""
    k0, k1 = key
    c = list(counter)
    for r in range(10):
        if r:
            k0, k1 = (k0 + PHILOX_W[0]) & _M64, (k1 + PHILOX_W[1]) & _M64
        p0, p1 = PHILOX_M[0] * c[0], PHILOX_M[1] * c[2]
        c = [(p1 >> 64) ^ c[1] ^ k0, p1 & _M64, (p0 >> 64) ^ c[3] ^ k1, p0 & _M64]
    return c


def uniform53(key, counter, word=0):
    """The 53-bit integer a of the draw's u = a * 2^-53: word 0 of the block at counter (n, 0, 0, 0), shifted right by 11."""
    return philox4x64_10(key, (int(counter), 0, 0, 0))[word] >> 11


def bound(z, n):
    """Half-width of the top-p and draw acceptance regions for a total (exact) mass z over n tokens (module docstring)."""
    return 2 * RHO * z + 2 * n * ALPHA + 2.0 ** -40 + (n + 3) * 2.0 ** -53 * z


class SampleMismatch(AssertionError):
    pass


def _rows(x, b, dtype):
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    a = np.asarray(x)
    if a.ndim == 0:
        a = np.full((b,), a)
    return a.astype(dtype) if dtype is not None else a


def _u64(x, shape):
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    if isinstance(x, np.ndarray):
        a = x.view(np.uint64) if x.dtype == np.int64 else x
        return [int(v) for v in a.reshape(-1)], shape
    return [int(v) for v in np.array(x, dtype=object).reshape(-1)], shape     # Python ints: no trip through float64


def _params(logits, temperature, top_k, top_p, keys, counters):
    if hasattr(logits, "detach"):
        logits = logits.detach().cpu().float().numpy()
    l16 = np.asarray(logits).astype(np.float16)
    b = l16.shape[0]
    t = _rows(temperature, b, np.float32)
    k = _rows(top_k, b, np.int64)
    p = _rows(top_p, b, np.float32)
    kw, _ = _u64(keys, (b, 2))
    cw, _ = _u64(counters, (b,))
    return l16, t, k, p, [(kw[2 * i], kw[2 * i + 1]) for i in range(b)], cw


def order_keys(row16):
    """The sampler's 16-bit keys: key descending <=> value descending, -0 folded onto +0."""
    h = row16.view(np.uint16).astype(np.uint32)
    h = np.where(h == 0x8000, 0, h)
    return np.where(h & 0x8000, (~h) & 0xFFFF, h | 0x8000).astype(np.int64)


def total_order(v):
    """Indices of a row in the total order: value descending, then index ascending (float compare: -0 == +0)."""
    return np.lexsort((np.arange(len(v)), -np.asarray(v, dtype=np.float64)))


def _bad_params(T, k, p):
    return not (np.isfinite(T) and T >= 0) or k < 0 or not (0 < p <= 1)


def sample_np(logits, temperature, top_k, top_p, keys, counters, faults=()):
    """The sampler in numpy (module docstring).  faults: names of deliberate errors for the checker's negative controls --
    'tie_high' (ties toward the higher index), 'topk_after_t' (top-k on fp16(l / T)), 'topp_short' / 'topp_long' (one token
    fewer / more in the top-p set), 'counter+1', 'word1' (u from the block's word 1), 'cdf_next' (the kept token after the
    drawn one).  Returns int32 [B]."""
    l16, T, K, P, KEY, CTR = _params(logits, temperature, top_k, top_p, keys, counters)
    out = np.empty(l16.shape[0], np.int32)
    for b in range(l16.shape[0]):
        out[b] = _sample_row(l16[b], float(T[b]), int(K[b]), np.float32(P[b]), KEY[b], CTR[b], faults)
    return out


def _sample_row(row, T, k, p, key, ctr, faults):
    V = len(row)
    kk = order_keys(row)
    idx = np.arange(V)
    if (kk > 0xFBFF).any() or (kk < 0x03FF).any() or (kk == 0x03FF).all() or _bad_params(T, k, float(p)):
        return -1
    tie = -idx if "tie_high" in faults else idx
    order = np.lexsort((tie, -kk))
    if T == 0 or k == 1:
        return int(order[0])
    keep = np.ones(V, bool)
    if 0 < k < V:
        if "topk_after_t" in faults:
            scaled = (row.astype(np.float32) / np.float32(T)).astype(np.float16)
            o2 = np.lexsort((tie, -order_keys(scaled)))
            keep[:] = False
            keep[o2[:k]] = True
        else:
            keep[:] = False
            keep[order[:k]] = True
    v32 = row.astype(np.float32)
    vmax = v32[order[0]]
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        x = ((v32 - vmax).astype(np.float32) / np.float32(T)).astype(np.float32)
        w = np.exp(x).astype(np.float32)
    W = np.rint(w.astype(np.float64) * FIX)
    W[np.isneginf(row.astype(np.float64))] = 0
    W = W.astype(np.uint64) * keep
    if p < 1:
        zk = int(W.sum())
        tp = math.ceil(float(p) * float(zk))
        Wo = W[order]
        M = np.concatenate([np.zeros(1, np.uint64), np.cumsum(Wo)[:-1]])
        n = int(np.count_nonzero(keep[order] & (M < np.uint64(tp))))
        n += ("topp_long" in faults) - ("topp_short" in faults)
        keep2 = np.zeros(V, bool)
        keep2[order[:n]] = True
        keep &= keep2
    S = np.cumsum(W * keep, dtype=np.uint64)
    z = int(S[-1])
    a = uniform53(key, ctr + ("counter+1" in faults), 1 if "word1" in faults else 0)
    t = (a * z) >> 53
    tok = int(np.searchsorted(S, np.uint64(t), side="right"))
    if "cdf_next" in faults:
        nxt = np.nonzero(keep[tok + 1:])[0]
        tok = tok + 1 + int(nxt[0]) if len(nxt) else tok
    return tok


def sample_tokens_np(logits, temperature, top_k, top_p, keys, counters):
    """ops.sample_tokens' signature over sample_np, for host-only tests: returns an int32 torch tensor on the logits' device."""
    import torch
    dev = logits.device if hasattr(logits, "device") else "cpu"
    return torch.from_numpy(sample_np(logits, temperature, top_k, top_p, keys, counters)).to(dev)


def _fail(b, rule, msg):
    raise SampleMismatch(f"row {b}: rule {rule}: {msg}")


def check_row(b, row, T, k, p, key, ctr, tok):
    """Accept or reject one token; returns True when the row's draw was ambiguous (module docstring)."""
    v = row.astype(np.float64)
    V = len(v)
    T, k, p = float(T), int(k), float(np.float32(p))
    if np.isnan(v).any() or np.isposinf(v).any() or np.isneginf(v).all() or _bad_params(T, k, p):
        if tok != -1:
            _fail(b, "invalid", f"an invalid row (NaN / +inf / all -inf / parameters) must give -1, got {tok}")
        return False
    if not (0 <= tok < V):
        _fail(b, "range", f"token {tok} outside [0, {V})")
    if T == 0 or k == 1:
        want = int(np.argmax(v))
        if tok != want:
            _fail(b, "greedy", f"T={T}, top_k={k}: the first index of the maximum is {want}, got {tok}")
        return False
    order = total_order(v)
    nk = V if k == 0 or k >= V else k
    rank = np.empty(V, np.int64)
    rank[order] = np.arange(V)
    if rank[tok] >= nk:
        _fail(b, "top-k", f"token {tok} is at place {rank[tok]} of the order on the raw logits, top_k={k}")
    m = v[order[0]]
    with np.errstate(over="ignore", invalid="ignore"):
        w_order = np.exp((v[order[:nk]] - m) / T)
    w_order[np.isneginf(v[order[:nk]])] = 0.0
    z = float(w_order.sum())
    if p < 1:
        M = np.concatenate([[0.0], np.cumsum(w_order)[:-1]])
        d = bound(z, nk)
        l_lo = max(1, int(np.count_nonzero(M < p * z - d)))
        l_hi = max(1, int(np.count_nonzero(M < p * z + d)))
    else:
        l_lo = l_hi = nk
    if rank[tok] >= l_hi:
        _fail(b, "top-p", f"token {tok} is at place {rank[tok]}, the top-p={p} set holds at most {l_hi} tokens")
    u = uniform53(key, ctr) * 2.0 ** -53
    ok, amb = False, l_hi > l_lo
    for n in range(l_lo, l_hi + 1):
        if rank[tok] >= n:
            continue
        kept = np.sort(order[:n])
        S = np.cumsum(w_order[rank[kept]])
        zl = float(S[-1])
        d = bound(zl, n)
        x = u * zl
        j = int(np.searchsorted(kept, tok))
        lo_, hi_ = (float(S[j - 1]) if j else 0.0), float(S[j])
        if lo_ - d <= x < hi_ + d:
            ok = True
        j0 = min(int(np.searchsorted(S, x, side="right")), n - 1)
        edges = [float(S[j0 - 1]) if j0 else 0.0, float(S[j0])]
        if any(abs(x - e) <= d for e in edges):
            amb = True
    if not ok:
        _fail(b, "draw", f"token {tok}: u*Z = {u:.9f}*Z does not fall in its inverse-CDF interval (counter {ctr}, key {key})")
    return amb


def check_tokens(logits, temperature, top_k, top_p, keys, counters, tokens):
    """Check every row; returns the number of ambiguous rows.  Raises SampleMismatch naming the row and the rule."""
    l16, T, K, P, KEY, CTR = _params(logits, temperature, top_k, top_p, keys, counters)
    tokens = np.asarray(tokens.detach().cpu().numpy() if hasattr(tokens, "detach") else tokens).astype(np.int64)
    amb = 0
    for b in range(l16.shape[0]):
        amb += check_row(b, l16[b], T[b], K[b], P[b], KEY[b], CTR[b], int(tokens[b]))
    return amb


def probabilities(row, T, k, p):
    """The exact (float64) sampling distribution of a row whose top-p boundary is unambiguous: [V] probabilities."""
    v = row.astype(np.float64)
    V = len(v)
    order = total_order(v)
    nk = V if k == 0 or k >= V else k
    w = np.exp((v[order[:nk]] - v[order[0]]) / T)
    z = w.sum()
    n = nk
    if p < 1:
        M = np.concatenate([[0.0], np.cumsum(w)[:-1]])
        n = max(1, int(np.count_nonzero(M < p * z)))
    out = np.zeros(V)
    out[order[:n]] = w[:n] / w[:n].sum()
    return out
