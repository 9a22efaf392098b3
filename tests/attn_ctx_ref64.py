"""Float64 reference and error bound of the prefill attention over a cached prefix (prefill_attn_kernel<true>): prompt chunks
that are the tails of sequences in a paged INT4 pool attend to the pool's earlier tokens and, causally, to themselves.

TEST INFRASTRUCTURE ONLY.  Built on tests/attn_ref64.py (same dequantisation, RoPE and float64 softmax; the bound is
prefill_bound's with the key count ctx + n in place of the prompt length).  With every prefix empty the reference and the bound
are attn_ref64.prefill_ref / prefill_bound exactly.
"""
import numpy as np

from tests.attn_ref64 import E, HD, U, _sequence, _softmax, dequant, freqs, make_pool, pack, unpack


def _prefill_ctx_heads(q, k4, kp, v4, vp, lens, hq, theta, data, param, indptr, indices, last, layer):
    """Like _prefill_heads for prompts that are the tails of cached sequences: prompt b's n_b tokens sit at positions ctx_b ..
    ctx_b + n_b - 1 of sequence b of the pool, ctx_b = its length - n_b.  Its keys are the pool's first ctx_b tokens (read from
    the pages) followed by its own (from k4 / v4); query r attends to keys 0 .. ctx_b + r."""
    q = np.asarray(q).astype(np.float64)
    T = q.shape[0]
    hkv = np.shape(k4)[1] // 64
    G = hq // hkv
    kn = unpack(np.asarray(k4).reshape(T, hkv, 64))
    vn = unpack(np.asarray(v4).reshape(T, hkv, 64))
    kpar = np.asarray(kp).astype(np.float64).reshape(T, hkv, 2)
    vpar = np.asarray(vp).astype(np.float64).reshape(T, hkv, 2)
    f = freqs(theta)
    off = 0
    for b, n in enumerate(lens):
        ckn, ckp, cvn, cvp = _sequence(data, param, indptr, indices, last, layer, b)
        ctx = ckn.shape[1] - n
        assert ctx >= 0, "a sequence shorter than its prompt"
        rq = np.exp(1j * np.multiply.outer(np.arange(ctx, ctx + n, dtype=np.float64), f))
        rk = np.exp(1j * np.multiply.outer(np.arange(ctx + n, dtype=np.float64), f))
        for h in range(hq):
            hk = h // G
            k = dequant(np.concatenate([ckn[hk, :ctx], kn[off:off + n, hk]]), np.concatenate([ckp[hk, :ctx], kpar[off:off + n, hk]]))
            v = dequant(np.concatenate([cvn[hk, :ctx], vn[off:off + n, hk]]), np.concatenate([cvp[hk, :ctx], vpar[off:off + n, hk]]))
            qq = q[off:off + n, h * HD:(h + 1) * HD]
            zq = (qq[:, :64] + 1j * qq[:, 64:]) * rq
            zk = (k[:, :64] + 1j * k[:, 64:]) * rk
            s = (zq @ np.conj(zk).T).real / np.sqrt(HD)
            s[np.triu_indices(n, ctx + 1, ctx + n)] = -np.inf
            w, z = _softmax(s)
            yield off, n, ctx, h, dict(q=qq, k=k, v=v, s=s, w=w, Z=z, o=w @ v, f=f)
        off += n


def prefill_ctx_ref(q, k4, kp, v4, vp, lens, hq, theta, data, param, indptr, indices, last, layer=0):
    """Attention of prompt chunks over their cached prefix and, causally, themselves: q, k4, kp, v4, vp, lens as for prefill_ref
    (the chunks' own tokens); data / param / indptr / indices / last: the paged pool whose sequence b ends with chunk b (what
    init_kv_i4 writes).  Returns float64 [T, Hq*128]; with every prefix empty it is prefill_ref."""
    out = np.zeros((np.shape(q)[0], hq * HD))
    for off, n, ctx, h, t in _prefill_ctx_heads(q, k4, kp, v4, vp, lens, hq, theta, data, param, indptr, indices, last, layer):
        out[off:off + n, h * HD:(h + 1) * HD] = t["o"]
    return out


def prefill_ctx_bound(q, k4, kp, v4, vp, lens, hq, theta, data, param, indptr, indices, last, layer=0, rows=None):
    """(float64 reference, bound) for prefill_attn_kernel<true>: prefill_bound's terms with L = ctx + n, the keys a query sees
    at most, in the angle term (positions up to L - 1, q and k rotated from the same FP32 table) and the accumulation terms (the
    context adds ctx / 64 tiles to the online softmax and to the P.V sums).  The context's K and V are dequantised, rotated and
    rounded inside the kernel exactly as kv_dequant_rope_kernel does for the chunk, so the per-key terms are unchanged.  rows:
    {prompt index: row indices} as for prefill_bound."""
    ref = np.zeros((np.shape(q)[0], hq * HD))
    bnd = np.zeros_like(ref)
    for pi, (off, n, ctx, h, t) in enumerate(_prefill_ctx_heads(q, k4, kp, v4, vp, lens, hq, theta, data, param, indptr, indices,
                                                                 last, layer)):
        prompt = pi // hq
        L = ctx + n
        q_, k, v, w, o = t["q"], t["k"], t["v"], t["w"], t["o"]
        aq = np.abs(q_[:, :64] + 1j * q_[:, 64:])
        ak = np.abs(k[:, :64] + 1j * k[:, 64:])
        eps = 5 * U + 2 * E * (16 * (L - 1) * t["f"] + 8)
        dl = (aq @ (ak * eps).T) / np.sqrt(HD) + 2.0 ** -21
        D = np.log((w * np.exp(dl)).sum(1))
        g = w * np.expm1(dl + D[:, None])
        av = np.abs(v)
        t1 = g @ av + g.sum(1, keepdims=True) * np.abs(o)
        sel = None if rows is None else rows.get(prompt)
        sel = range(n) if sel is None else sel
        for r in sel:
            t1[r] = g[r, :ctx + r + 1] @ np.abs(v[:ctx + r + 1] - o[r])
        acc = E * (L / 16 + 32)
        wk = w * np.exp(dl + D[:, None])
        tiny = np.tril(w * t["Z"][:, None] < 2.0 ** -14, ctx)                             # keys the query sees only
        t2 = (2 * U + acc) * (wk @ av) + (2.0 ** -25 * (1 + U)) * ((tiny / t["Z"][:, None]) @ av)
        t3 = (U + acc) * np.abs(o) + E
        ref[off:off + n, h * HD:(h + 1) * HD] = o
        bnd[off:off + n, h * HD:(h + 1) * HD] = t1 + t2 + t3
    return ref, bnd


def make_ctx_case(rng, ctxs, lens, hq, hkv, P, regime="moderate", dirty=False, L=1, layer=0):
    """Prompt chunks over cached prefixes: sequence b holds ctxs[b] + lens[b] tokens in a paged pool (make_pool), its last
    lens[b] being the chunk.  K/V are centred (scales in [0.1, 1], zero ~ 7.5 scale).  regime "moderate": q ~ N(0, 0.7^2);
    "sink": the sequence's first token and one token in every later 64-token tile of it carry a growing maximum through the
    lowest-frequency pair (q's element 63 is 24), so the softmax maximum moves on through the context and into the chunk.
    Returns (q f16 [T, hq*128], k4, kp, v4, vp of the chunks, pool = (data, param, indptr, indices, last))."""
    seqs, qs, ks, kps, vs, vps = [], [], [], [], [], []
    for ctx, n in zip(ctxs, lens):
        m = ctx + n
        kn, vn = rng.integers(0, 16, (hkv, m, 128)), rng.integers(0, 16, (hkv, m, 128))
        par = lambda: (lambda s: np.stack([s, s * rng.uniform(7.3, 7.7, s.shape)], -1))(rng.uniform(0.1, 1, (hkv, m)))
        kp, vp = par(), par()
        if regime == "moderate":
            q = rng.standard_normal((n, hq, 128)) * 0.7
        else:
            q = rng.standard_normal((n, hq, 128)) * 0.3
            q[:, :, 63] = 24.0
            kn[:, 0, 63] = 15; kp[:, 0, 0] = 1.0; kp[:, 0, 1] = 7.5
            for j in range(1, (m + 63) // 64):
                tok = min(64 * j + int(rng.integers(64)), m - 1)
                kn[:, tok, 63] = 15; kp[:, tok, 0] = 1.0 + 0.1 * j; kp[:, tok, 1] = 7.5 * kp[:, tok, 0]
        kp, vp = kp.astype(np.float16), vp.astype(np.float16)
        seqs.append((kn, kp, vn, vp))
        qs.append(q.astype(np.float16).reshape(n, hq * 128))
        ks.append(pack(kn[:, ctx:].transpose(1, 0, 2)).reshape(n, hkv * 64))
        kps.append(kp[:, ctx:].transpose(1, 0, 2).reshape(n, hkv * 2))
        vs.append(pack(vn[:, ctx:].transpose(1, 0, 2)).reshape(n, hkv * 64))
        vps.append(vp[:, ctx:].transpose(1, 0, 2).reshape(n, hkv * 2))
    pool = make_pool(seqs, P, hkv, L=L, layer=layer, rng=rng, dirty=dirty)
    cat = lambda xs: np.ascontiguousarray(np.concatenate(xs))
    return (cat(qs), cat(ks), cat(kps), cat(vs), cat(vps)), pool
