"""Float64 reference of beam search (atom_b200.ops.beam_select, the beam requests of atom_b200.textgen; DESIGN section 5.9).

beam_select_np is one beam step over FP16 logits rows with the log-probability rule of sample_penalty_ref64._logprobs_row (the
one atom_sample_ex_f16 follows at T = 1) and its bound lp_bound.  BeamRequest is the host state machine of one request: live
beams, finished hypotheses and the rules that end it.  beam_search_ref runs a whole request against a Markov stand-in (the next
row depends on the last token only) and exhaustive_best enumerates every output for small vocabularies and lengths."""
import itertools
import math

import numpy as np

from tests.sample_penalty_ref64 import KEY_NEG_INF, _logprobs_row, lp_bound, order_keys  # noqa: F401


def row_candidates(row):
    """(lps float32 [V], the token ids in the row's order with -inf excluded), or None for a row without candidates (NaN, +inf
    or only -inf)."""
    row = np.asarray(row, np.float16)
    kk = order_keys(row)
    if (kk > 0xFBFF).any() or (kk < KEY_NEG_INF).any() or (kk == KEY_NEG_INF).all():
        return None
    V = len(row)
    lps = _logprobs_row(row, np.arange(V), 0, ())[0]
    order = np.lexsort((np.arange(V), -kk))
    return lps, [int(t) for t in order if kk[t] > KEY_NEG_INF]


def beam_select_np(logits, row_indptr, sums, width, stop_ids=(), lp_rows=None):
    """One beam step (ops.beam_select's contract) on host arrays: returns (live [B, W, 2], live_key [B, W], fin [B, W, 2],
    fin_key [B, W]) as numpy arrays padded with -1.  lp_rows: optional per-row {token: float32 lp} that replaces the reference's
    log-probabilities for the tokens it holds (so that a device's own values can be merged exactly)."""
    logits = np.asarray(logits, np.float16)
    ip = np.asarray(row_indptr, np.int64).reshape(-1)
    sums = np.asarray(sums, np.float32).reshape(-1)
    W, stops = int(width), [int(t) for t in stop_ids]
    B = len(ip) - 1
    live = np.full((B, W, 2), -1, np.int32)
    fin = np.full((B, W, 2), -1, np.int32)
    live_key = np.full((B, W), -1, np.float32)
    fin_key = np.full((B, W), -1, np.float32)
    for i in range(B):
        r0, r1 = int(ip[i]), int(ip[i + 1])
        if not 0 < r1 - r0 <= W:
            continue
        cands = []
        for j, r in enumerate(range(r0, r1)):
            rc = row_candidates(logits[r])
            if rc is None:
                continue
            lps, order = rc
            kept = [t for t in order if t not in stops][:W] + [t for t in order if t in stops]
            pos = {t: p for p, t in enumerate(order)}
            for t in kept:
                lp = np.float32(lps[t]) if lp_rows is None or t not in lp_rows[r] else np.float32(lp_rows[r][t])
                key = np.float32(sums[r] + lp)
                if not np.isnan(key):
                    cands.append((-float(key), j, pos[t], r, t, key))
        cands.sort(key=lambda c: c[:3])
        nl = nf = 0
        for rank, (_, _, _, r, t, key) in enumerate(cands):
            if nl == W:
                break
            if t in stops:
                if rank < W:
                    fin[i, nf], fin_key[i, nf] = (r, t), key
                    nf += 1
            else:
                live[i, nl], live_key[i, nl] = (r, t), key
                nl += 1
    return live, live_key, fin, fin_key


def near_tie(rows, sums, a, b, slack=1.0):
    """Whether candidates a and b, each (row, token), are ordered within the reference's uncertainty: the difference of their
    float64 keys is within the sum of their log-probabilities' bounds plus one FP32 rounding of each key."""
    def key_bound(c):
        r, t = c
        row = np.asarray(rows[r], np.float16)
        v32 = row.astype(np.float32)
        vmax = np.float32(v32[np.isfinite(v32)].max())
        d = np.float32(v32[t] - vmax)
        with np.errstate(all="ignore"):
            w = np.rint(np.exp((v32 - vmax).astype(np.float32)).astype(np.float64) * 2.0 ** 40)
        w[np.isneginf(row)] = 0
        z = float(w.sum()) * 2.0 ** -40
        lp = float(d) - math.log(z)
        return float(sums[r]) + lp, lp_bound(float(d), lp, z, len(row)) + 2.0 ** -23 * abs(float(sums[r]) + lp)
    ka, ba = key_bound(a)
    kb, bb = key_bound(b)
    return abs(ka - kb) <= slack * (ba + bb)


class BeamRequest:
    """The host state of one request (DESIGN section 5.9): live beams (tokens, FP32 sum), in selection order, and up to W finished
    hypotheses (tokens, sum, score = sum / len^alpha in float64, order of arrival)."""

    def __init__(self, width, alpha, n_out, stop_ids=()):
        self.W, self.alpha, self.n = int(width), float(alpha), int(n_out)
        self.stops = frozenset(int(t) for t in stop_ids)
        self.live = [([], np.float32(0))]
        self.finished = []                              # (score, arrival, tokens, sum)
        self.arrivals = 0
        self.done = False

    def score(self, tokens, s):
        return float(s) / float(len(tokens)) ** self.alpha

    def offer(self, tokens, s):
        h = (self.score(tokens, s), self.arrivals, list(tokens), np.float32(s))
        self.arrivals += 1
        if len(self.finished) < self.W:
            self.finished.append(h)
        else:
            worst = min(range(len(self.finished)), key=lambda k: (self.finished[k][0], -self.finished[k][1]))
            if h[0] > self.finished[worst][0]:
                self.finished[worst] = h

    def step(self, live, live_key, fin, fin_key, row_of_beam):
        """Apply one beam_select result for this request; row_of_beam maps a result row to the live beam it extends.  Returns
        the parent beam index of each new live beam."""
        for (r, t), k in zip(fin, fin_key):
            if r >= 0:
                self.offer(self.live[row_of_beam(r)][0] + [int(t)], k)
        new, parents = [], []
        for (r, t), k in zip(live, live_key):
            if r >= 0:
                b = row_of_beam(r)
                new.append((self.live[b][0] + [int(t)], np.float32(k)))
                parents.append(b)
        self.live = new
        if len(self.finished) >= self.W:
            self.done = True
        elif not new:
            self.done = True
        elif len(new[0][0]) >= self.n:
            for tokens, s in new:
                self.offer(tokens, s)
            self.done = True
        return parents

    def best(self):
        """(tokens, sum, score) of the output: the highest score, the earliest on a tie; ([], nan, -inf) with none."""
        if not self.finished:
            return [], np.float32(np.nan), -math.inf
        h = max(self.finished, key=lambda h: (h[0], -h[1]))
        return h[2], h[3], h[0]


def beam_search_ref(next_row, first_row, width, alpha, n_out, stop_ids=()):
    """A whole request: first_row is the prompt's last logits row, next_row(token) the row after a token (a Markov stand-in).
    Returns the BeamRequest when it is done."""
    req = BeamRequest(width, alpha, n_out, stop_ids)
    rows = [np.asarray(first_row, np.float16)]
    while True:
        sums = [s for _, s in req.live]
        ip = [0, len(rows)]
        res = beam_select_np(np.stack(rows), ip, sums, width, stop_ids)
        req.step(res[0][0], res[1][0], res[2][0], res[3][0], lambda r: r)
        if req.done:
            return req
        rows = [np.asarray(next_row(tokens[-1]), np.float16) for tokens, _ in req.live]


def exhaustive_best(next_row, first_row, alpha, n_out, stop_ids=()):
    """The best score over every output: each token sequence that ends on its first stop id, or reaches n_out tokens without
    one, scored sum(lp) / len^alpha with the reference's FP32 sums.  Returns (score, tokens)."""
    stops = frozenset(int(t) for t in stop_ids)
    first = np.asarray(first_row, np.float16)
    V = len(first)
    cache = {}

    def lps(tok):
        if tok not in cache:
            cache[tok] = row_candidates(next_row(tok))[0]
        return cache[tok]

    best = (-math.inf, None)
    for n in range(1, n_out + 1):
        for seq in itertools.product(range(V), repeat=n):
            if any(t in stops for t in seq[:-1]) or (n < n_out and seq[-1] not in stops):
                continue
            s = np.float32(0)
            row = row_candidates(first)[0]
            for k, t in enumerate(seq):
                s = np.float32(s + row[t])
                row = lps(t) if k + 1 < n else None
            if not np.isfinite(s):
                continue
            sc = float(s) / float(n) ** alpha
            if sc > best[0]:
                best = (sc, list(seq))
    return best


def beam_select_tokens_np(logits, row_indptr, sums, width, stop_ids=(), out=None, workspace=None):
    """ops.beam_select's signature on host tensors (a stand-in for CPU tests): the reference's result, written into `out` (the
    packed int32 buffer) when it is given."""
    import torch
    lg = logits.detach().cpu().numpy().astype(np.float16)
    res = beam_select_np(lg, row_indptr.cpu().numpy(), sums.cpu().numpy(), width, stop_ids)
    B, W = res[1].shape
    if out is not None:
        flat = np.concatenate([res[0].reshape(-1), res[1].view(np.int32).reshape(-1), res[2].reshape(-1),
                               res[3].view(np.int32).reshape(-1)])
        out.copy_(torch.from_numpy(flat))
        n = B * W
        return (out[:2 * n].view(B, W, 2), out[2 * n:3 * n].view(torch.float32).view(B, W), out[3 * n:5 * n].view(B, W, 2),
                out[5 * n:].view(torch.float32).view(B, W))
    return tuple(torch.from_numpy(x) for x in res)


class CopyLog:
    """ops.copy_kv_pages' signature on a host pool (a stand-in for CPU tests): copies the first `slots` token slots of every
    block, records each pair with the source page's holder count at the time, and skips src < 0."""

    def __init__(self):
        self.pairs = []

    def __call__(self, pool, src, dst, slots):
        to_list = lambda x: [int(v) for v in (x.tolist() if hasattr(x, "tolist") else x)]      # noqa: E731
        for s, d, n in zip(to_list(src), to_list(dst), to_list(slots)):
            if s < 0:
                continue
            assert s != d and 1 <= n <= pool.block_len
            self.pairs.append((s, d, n, pool.refcount(s), pool.refcount(d)))
            pool.buf[d, :, :, :, :n] = pool.buf[s, :, :, :, :n]
            pool.param[d, :, :, :, :n] = pool.param[s, :, :, :, :n]
