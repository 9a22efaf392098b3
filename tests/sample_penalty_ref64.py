"""Reference of atom_sample_ex_f16 / ops.sample_tokens with penalties, min-p and log-probabilities (include/atom_b200.h;
DESIGN section 5.6).  It extends tests/sample_ref64.py, whose Philox, keys, total order, weights and `bound()` it uses as they
are; everything below applies rules 1-5 of that module to the penalised logits l'.

* `penalise` computes the penalised logits l' bit for bit: every step is one IEEE FP32 operation, which numpy float32 rounds
  the same way.  The invalid-row test stays on the raw row.

* `sample_np` -- the sampler of sample_ref64.sample_np with the options of ops.sample_tokens: penalties read from a table (and
  the drawn tokens recorded in it), min-p, and the log-probability outputs.  Like the base one it is an exact sampler of the
  semantics, not a bit model of the kernel (numpy's exp is not CUDA's expf); the serving harness's CPU tests substitute it for
  the kernel, and `faults=` shows that the checker rejects faulty samplers.

* `check_tokens` -- the float64 checker, extended:
  - min-p keeps the tokens with W_i >= ceil(m * 2^40).  With W_i within rho * w_i + alpha of w_i (units of 2^40; sample_ref64's
    docstring), a token is kept for certain when w_i (1 - rho) - alpha >= c and dropped for certain when
    w_i (1 + rho) + alpha < c, c = ceil(m 2^40) 2^-40; in between it is ambiguous.  The exact weights are monotone in l', so
    the admissible min-p sets are prefixes of the order.
  - log-probabilities: lp_i = (l'_i - max) - ln(Z1 2^-40), Z1 = sum of round(expf(l'_j - max) 2^40) over the whole row, against
    the exact (l'_i - max) - ln Z, Z = sum exp(l'_j - max).  The kernel's error is at most
        2^-24 |d|                 the FP32 difference d = fl(l'_i - max),
      + delta / (1 - delta)       ln(Z1' / Z), |Z1' - Z| <= rho Z + V alpha, delta = rho + V alpha / Z (Z >= 1),
      + 2^-50 (|ln Z| + |d| + 1)  the double log and subtraction (a few units of 2^-53),
      + 2^-24 |lp|                the conversion to FP32,
    and the float64 reference's own sum adds V 2^-53.  That is `lp_bound`.  The top-n ids are exact: a top-k set on the keys.
"""
import math

import numpy as np

from tests.sample_ref64 import (ALPHA, FIX, RHO, SampleMismatch, _fail, _params, _rows, bound, order_keys,  # noqa: F401
                                total_order, uniform53)


def _bad_params(T, k, p, m=0.0, r=1.0, f=0.0, q=0.0):
    return not (np.isfinite(T) and T >= 0) or k < 0 or not (0 < p <= 1) or not (0 <= m <= 1) or \
        not (np.isfinite(r) and r > 0) or not np.isfinite(f) or not np.isfinite(q)


TOP_N_MAX = 20
KEY_NEG_INF = 0x03FF


def lp_bound(d, lp, z, V):
    """Half-width of the acceptance region of a log-probability (module docstring): d = l'_i - max, lp the exact value, z the
    exact Z over V tokens."""
    delta = RHO + V * ALPHA / z
    return 2.0 ** -24 * abs(d) + delta / (1 - delta) + 2.0 ** -50 * (abs(math.log(z)) + abs(d) + 1) + 2.0 ** -24 * abs(lp) + \
        V * 2.0 ** -53


def penalise(row16, entries, r, f, q, faults=()):
    """The penalised logits l' (FP16) of one row from its table entries (u16: bit 15 prompt, bits 0-14 count): -inf stays;
    repetition r on prompt or generated tokens (l > 0: l / r, else l * r); frequency fl(c * f); presence q if c > 0; FP16 of the
    result saturated to +-65504.  faults: 'presence_on_prompt', 'neginf_penalised' (no -inf pass-through), 'rep_divide_all'
    (l / r whatever the sign), 'order' (frequency and presence before repetition)."""
    row16 = np.asarray(row16, np.float16)
    e = np.asarray(entries).astype(np.uint32)
    c = (e & 0x7FFF).astype(np.float32)
    prompt, gen = (e & 0x8000) != 0, c > 0
    r, f, q = np.float32(r), np.float32(f), np.float32(q)
    l = row16.astype(np.float32)
    with np.errstate(all="ignore"):
        def rep(l):
            return np.where(prompt | gen, l / r if "rep_divide_all" in faults else np.where(l > 0, l / r, l * r), l).astype(np.float32)

        def freq_pres(l):
            l = (l - c * f).astype(np.float32)
            return np.where((gen | prompt) if "presence_on_prompt" in faults else gen, l - q, l).astype(np.float32)
        l = rep(freq_pres(l)) if "order" in faults else freq_pres(rep(l))
        out = np.fmin(np.fmax(l, np.float32(-65504)), np.float32(65504)).astype(np.float16)
    if "neginf_penalised" not in faults:
        out[np.isneginf(row16)] = -np.inf
    return out


def _table_np(table):
    if table is None:
        return None
    if hasattr(table, "detach"):
        table = table.detach()
        return (table.cpu() if table.is_cuda else table).numpy().view(np.uint16)
    return np.asarray(table).view(np.uint16)


def _penalised(l16, table, slots, r, f, q, faults=()):
    """l' of every row (rows without a slot keep their raw logits)."""
    if table is None:
        return l16
    tab = _table_np(table)
    b, V = l16.shape
    sl = _rows(slots, b, np.int64)
    R, F, Q = (_rows(x, b, np.float32) for x in (r, f, q))
    out = l16.copy()
    for i in range(b):
        if sl[i] >= 0:
            out[i] = penalise(l16[i], tab[sl[i], :V], R[i], F[i], Q[i], faults)
    return out


def _ext_params(b, min_p, r, f, q):
    return [_rows(x, b, np.float32) for x in (min_p, r, f, q)]


def sample_np(logits, temperature, top_k, top_p, keys, counters, faults=(), *, min_p=0.0, repetition_penalty=1.0,
              frequency_penalty=0.0, presence_penalty=0.0, penalty_table=None, slots=None, logprobs=None):
    """The sampler in numpy (module docstring).  faults: names of deliberate errors for the checker's negative controls --
    'tie_high' (ties toward the higher index), 'topk_after_t' (top-k on fp16(l / T)), 'topp_short' / 'topp_long' (one token
    fewer / more in the top-p set), 'counter+1', 'word1' (u from the block's word 1), 'cdf_next' (the kept token after the
    drawn one); with the options below also `penalise`'s faults, 'minp_short' / 'minp_long' (one token fewer / more in the
    min-p set), 'no_saturate' (the count wraps into the prompt bit), 'logprob_off' (every log-probability 1e-3 too high),
    'topn_tie_high' (top-n ties toward the higher index).  Returns int32 [B].

    The keyword options are ops.sample_tokens': penalty_table (a numpy uint16 / int16 array or a CPU torch tensor, [slots, ld])
    is read for l' and then records the drawn tokens in place; with logprobs = n it returns (tokens, logprob float32 [B],
    top_ids int32 [B, n], top_logprobs float32 [B, n])."""
    l16, T, K, P, KEY, CTR = _params(logits, temperature, top_k, top_p, keys, counters)
    b = l16.shape[0]
    MP, RP, FP, QP = _ext_params(b, min_p, repetition_penalty, frequency_penalty, presence_penalty)
    lp16 = _penalised(l16, penalty_table, slots, RP, FP, QP, faults)
    n = 0 if logprobs is None else int(logprobs)
    out = np.empty(b, np.int32)
    lp = np.full(b, np.nan, np.float32)
    top_ids = np.full((b, n), -1, np.int32)
    top_lp = np.full((b, n), np.nan, np.float32)
    for i in range(b):
        bad = _bad_params(float(T[i]), int(K[i]), float(P[i]), float(MP[i]), float(RP[i]), float(FP[i]), float(QP[i]))
        out[i] = -1 if bad else _sample_row(lp16[i], float(T[i]), int(K[i]), np.float32(P[i]), KEY[i], CTR[i], faults, float(MP[i]),
                                            raw=l16[i])
        if out[i] >= 0 and logprobs is not None:
            lp[i], top_ids[i], top_lp[i] = _logprobs_row(lp16[i], int(out[i]), n, faults)
    if penalty_table is not None:
        tab = _table_np(penalty_table)
        sl = _rows(slots, b, np.int64)
        for i in range(b):
            if sl[i] >= 0 and out[i] >= 0:
                e = int(tab[sl[i], out[i]])
                if (e & 0x7FFF) != 0x7FFF or "no_saturate" in faults:
                    tab[sl[i], out[i]] = (e + 1) & 0xFFFF
    return out if logprobs is None else (out, lp, top_ids, top_lp)


def _logprobs_row(row, tok, n, faults):
    kk = order_keys(row)
    v32 = row.astype(np.float32)
    order = np.lexsort((-np.arange(len(row)) if "topn_tie_high" in faults else np.arange(len(row)), -kk))
    vmax = v32[order[0]]
    with np.errstate(all="ignore"):
        d = (v32 - vmax).astype(np.float32)
        W = np.rint(np.exp(d).astype(np.float64) * FIX)
    W[np.isneginf(row)] = 0
    lnz = math.log(float(int(W.astype(np.uint64).sum())) * 2.0 ** -40)
    lps = (d.astype(np.float64) - lnz + (1e-3 if "logprob_off" in faults else 0.0)).astype(np.float32)
    lps[np.isneginf(row)] = -np.inf
    ids = np.full(n, -1, np.int32)
    lpn = np.full(n, -np.inf, np.float32)
    top = [int(j) for j in order[:n] if kk[j] > KEY_NEG_INF]
    ids[:len(top)] = top
    lpn[:len(top)] = lps[top]
    return lps[tok], ids, lpn


def _sample_row(row, T, k, p, key, ctr, faults, m=0.0, raw=None):
    V = len(row)
    kk = order_keys(row)
    kr = kk if raw is None else order_keys(raw)
    idx = np.arange(V)
    if (kr > 0xFBFF).any() or (kr < 0x03FF).any() or (kr == 0x03FF).all() or _bad_params(T, k, float(p)):
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
    if m > 0:
        keep_m = W >= math.ceil(float(np.float32(m)) * FIX)
        nm = int(np.count_nonzero(keep_m[order] & keep[order]))
        nm = max(1, nm + ("minp_long" in faults) - ("minp_short" in faults))
        if "minp_long" in faults or "minp_short" in faults:
            keep_m[:] = False
            keep_m[order[:nm]] = True
        keep &= keep_m
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


def sample_tokens_np(logits, temperature, top_k, top_p, keys, counters, **options):
    """ops.sample_tokens' signature over sample_np, for host-only tests: returns an int32 torch tensor on the logits' device (with
    logprobs, the four tensors).  A CPU torch penalty_table is updated in place."""
    import torch
    dev = logits.device if hasattr(logits, "device") else "cpu"
    r = sample_np(logits, temperature, top_k, top_p, keys, counters, **options)
    if isinstance(r, tuple):
        return tuple(torch.from_numpy(x).to(dev) for x in r)
    return torch.from_numpy(r).to(dev)


def init_penalty_slot_np(table, slot, prompt):
    """ops.init_penalty_slot over a numpy array or a CPU torch tensor: zero the slot's row, mark the prompt's tokens."""
    tab = _table_np(table)
    tab[slot] = 0
    tab[slot, np.asarray(prompt, dtype=np.int64)] = 0x8000


def check_row(b, row, T, k, p, key, ctr, tok, m=0.0, raw=None):
    """Accept or reject one token; returns True when the row's draw was ambiguous (module docstring).  row: the (penalised)
    logits; raw: the raw ones, for the invalid-row test (default: row); m: min-p."""
    v = row.astype(np.float64)
    vr = v if raw is None else raw.astype(np.float64)
    V = len(v)
    T, k, p, m = float(T), int(k), float(np.float32(p)), float(np.float32(m))
    if np.isnan(vr).any() or np.isposinf(vr).any() or np.isneginf(vr).all() or _bad_params(T, k, p, m):
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
        _fail(b, "top-k", f"token {tok} is at place {rank[tok]} of the order on the logits, top_k={k}")
    mx = v[order[0]]
    with np.errstate(over="ignore", invalid="ignore"):
        w_all = np.exp((v[order[:nk]] - mx) / T)
    w_all[np.isneginf(v[order[:nk]])] = 0.0
    if m > 0:                                         # the admissible min-p sets: prefixes of the order
        c = math.ceil(m * FIX) / FIX
        m_lo = max(1, int(np.count_nonzero(w_all * (1 - RHO) - ALPHA >= c)))
        m_hi = max(1, int(np.count_nonzero(w_all * (1 + RHO) + ALPHA >= c)))
        if rank[tok] >= m_hi:
            _fail(b, "min-p", f"token {tok} is at place {rank[tok]}, the min-p={m} set holds at most {m_hi} tokens")
    else:
        m_lo = m_hi = nk
    u = uniform53(key, ctr) * 2.0 ** -53
    ok, amb, most = False, m_hi > m_lo, 0
    for nm in range(m_lo, m_hi + 1):
        w_order = w_all[:nm]
        z = float(w_order.sum())
        if p < 1:
            M = np.concatenate([[0.0], np.cumsum(w_order)[:-1]])
            d = bound(z, nm)
            l_lo = max(1, int(np.count_nonzero(M < p * z - d)))
            l_hi = max(1, int(np.count_nonzero(M < p * z + d)))
        else:
            l_lo = l_hi = nm
        most = max(most, l_hi)
        amb |= l_hi > l_lo
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
    if rank[tok] >= most:
        _fail(b, "top-p", f"token {tok} is at place {rank[tok]}, the top-p={p} set holds at most {most} tokens")
    if not ok:
        _fail(b, "draw", f"token {tok}: u*Z = {u:.9f}*Z does not fall in its inverse-CDF interval (counter {ctr}, key {key})")
    return amb


def check_logprobs_row(b, row, tok, lp, top_ids, top_lp):
    """The log-probability of the chosen token and the top-n list of one row of l' (module docstring)."""
    n = len(top_ids)
    if tok < 0:
        if not np.isnan(lp) or (np.asarray(top_ids) != -1).any() or not np.isnan(top_lp).all():
            _fail(b, "logprob", "an invalid row must give logprob NaN, top ids -1 and top logprobs NaN")
        return
    v = row.astype(np.float64)
    finite = ~np.isneginf(v)
    mx = v.max()
    z = float(np.exp(v[finite] - mx).sum())
    lnz = math.log(z)

    def want(i):
        return -math.inf if not finite[i] else (v[i] - mx) - lnz

    def close(i, got, what):
        w = want(i)
        if w == -math.inf:
            if got != -math.inf:
                _fail(b, "logprob", f"{what}: token {i} has logit -inf, logprob must be -inf, got {got}")
            return
        d = bound_ = lp_bound(v[i] - mx, w, z, len(v))
        if not abs(float(got) - w) <= d:
            _fail(b, "logprob", f"{what}: token {i}: {float(got)!r} is {abs(float(got) - w):.3g} from {w!r}, bound {bound_:.3g}")
    close(tok, lp, "chosen")
    order = [int(j) for j in total_order(v)[:n] if finite[j]]
    ids = np.full(n, -1, np.int64)
    ids[:len(order)] = order
    if not np.array_equal(np.asarray(top_ids, np.int64), ids):
        _fail(b, "top-n", f"top ids {np.asarray(top_ids).tolist()}, the first {n} of the order are {ids.tolist()}")
    for j in range(n):
        if ids[j] < 0:
            if top_lp[j] != -np.inf:
                _fail(b, "top-n", f"padding {j} must have logprob -inf, got {top_lp[j]}")
        else:
            close(int(ids[j]), top_lp[j], f"top-n place {j}")


def _np(x):
    return np.asarray(x.detach().cpu().numpy() if hasattr(x, "detach") else x)


def check_tokens(logits, temperature, top_k, top_p, keys, counters, tokens, *, min_p=0.0, repetition_penalty=1.0,
                 frequency_penalty=0.0, presence_penalty=0.0, penalty_table=None, slots=None, logprob=None, top_ids=None,
                 top_logprobs=None):
    """Check every row; returns the number of ambiguous rows.  Raises SampleMismatch naming the row and the rule.  The options
    are ops.sample_tokens'; penalty_table is the table as it was *before* the call.  logprob / top_ids / top_logprobs: the
    log-probability outputs, checked when given."""
    l16, T, K, P, KEY, CTR = _params(logits, temperature, top_k, top_p, keys, counters)
    b = l16.shape[0]
    MP, RP, FP, QP = _ext_params(b, min_p, repetition_penalty, frequency_penalty, presence_penalty)
    lp16 = _penalised(l16, penalty_table, slots, RP, FP, QP)
    tokens = _np(tokens).astype(np.int64)
    amb = 0
    for i in range(b):
        bad = _bad_params(float(T[i]), int(K[i]), float(P[i]), float(MP[i]), float(RP[i]), float(FP[i]), float(QP[i]))
        if bad:
            if tokens[i] != -1:
                _fail(i, "invalid", f"parameters out of range must give -1, got {tokens[i]}")
        else:
            amb += check_row(i, lp16[i], T[i], K[i], P[i], KEY[i], CTR[i], int(tokens[i]), MP[i], raw=l16[i])
        if logprob is not None:
            n = 0 if top_ids is None else _np(top_ids).shape[1]
            check_logprobs_row(i, lp16[i], int(tokens[i]), float(_np(logprob)[i]),
                               _np(top_ids)[i] if n else np.zeros(0, np.int64), _np(top_logprobs)[i] if n else np.zeros(0))
    return amb
