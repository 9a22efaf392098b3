"""Float64 reference and error bound of the verify attention (verify_attn_kernel, ops.batch_verify_i4): every sequence of a paged
INT4 pool ends with S query tokens that attend to the pool's earlier tokens and, causally, to each other.

TEST INFRASTRUCTURE ONLY.  The reference is attn_ctx_ref64.prefill_ctx_ref over each sequence's last S tokens: a verify step is a
prompt chunk of S tokens whose K/V are already in the pages.  The bound (verify_bound) is prefill_ctx_bound's with q rotated as
the cascade's prefix pass rotates it and the chunk merge added; every constant is counted from the kernel's roundings, none is
fitted to a GPU run.
"""
import numpy as np

from tests import attn_ref64 as R
from tests.attn_ctx_ref64 import _prefill_ctx_heads
from tests.attn_ref64 import E, HD, U

MAX_CHUNKS = 64         # atom_verify_chunks never cuts a sequence into more runs


def tails(data, param, indptr, indices, last, layer, S):
    """The last S tokens of every sequence of the pool as a prompt chunk: (k4, kp, v4, vp, lens) in prefill_ref's layout."""
    H = data.shape[3]
    ks, kps, vs, vps = [], [], [], []
    for b in range(len(last)):
        kn, kp, vn, vp = R._sequence(data, param, indptr, indices, last, layer, b)
        assert kn.shape[1] >= S, "a sequence shorter than its query tokens"
        ks.append(R.pack(kn[:, -S:].transpose(1, 0, 2)).reshape(S, H * 64))
        kps.append(kp[:, -S:].transpose(1, 0, 2).astype(np.float16).reshape(S, H * 2))
        vs.append(R.pack(vn[:, -S:].transpose(1, 0, 2)).reshape(S, H * 64))
        vps.append(vp[:, -S:].transpose(1, 0, 2).astype(np.float16).reshape(S, H * 2))
    return np.concatenate(ks), np.concatenate(kps), np.concatenate(vs), np.concatenate(vps), [S] * len(last)


def verify_ref(q, data, param, indptr, indices, last, layer, hq, theta, S):
    """q [B*S, Hq, 128] (pre-RoPE, row b*S + i = token i of sequence b); the pool as for attn_ref64.decode_ref.  Returns float64
    [B*S, Hq, 128]: prefill_ctx_ref over the sequences' last S tokens."""
    from tests.attn_ctx_ref64 import prefill_ctx_ref
    k4, kp, v4, vp, lens = tails(data, param, indptr, indices, last, layer, S)
    T = np.shape(q)[0]
    out = prefill_ctx_ref(np.asarray(q).reshape(T, hq * HD), k4, kp, v4, vp, lens, hq, theta, data, param, indptr, indices, last, layer)
    return out.reshape(T, hq, HD)


def verify_bound(q, data, param, indptr, indices, last, layer, hq, theta, S):
    """(float64 reference [B*S, Hq, 128], per-element bound of |kernel - reference|) for verify_attn_kernel and its chunk merge.

    Sequence b of length L attends with query token r (position L - S + r) to keys 0 .. L - S + r.  Score error per pair i (u, e
    as in attn_ref64):
      * q is rotated in FP32 at its position by sincosf of pos * exp2f(-i log2(theta) / 64) and rounded to FP16 once (u), as the
        cascade's prefix pass does: its angle carries decode_bound's c_theta,i (L-1) theta_i plus 8 (sincosf, rotation);
      * k = fp16(n s - z) (u), rotated in FP32 from the (cos, sin) table of ops.rope_table and rounded (u): prefill_bound's
        (2 + sqrt2) u and 16 (L-1) theta_i + 8 for the angle; the tensor-core FP32 sums of 128 exact products (< 2^-17): c_s = 5;
      => delta_rt = sum_i |zq_ri||zk_ti| (5u + e ((c_theta,i + 16) (L-1) theta_i + 16)) / sqrt(128) + 2^-21 (exp2f).
    T1 = sum_t w_t (e^{delta_t + D} - 1) |v_t - o| (exact spread, the keys the row sees).
    V path as in prefill_bound: v and the weight rounded to FP16 (2u relative), a weight subnormal in its tile's frame (w_t Z <
    2^-14) 2^-25 / Z absolute.  FP32 sums: the tile recurrence (L/16 + 32, prefill_bound's) and the chunk merge (at most
    MAX_CHUNKS partials, two roundings each: 2 MAX_CHUNKS), acc = e (L/16 + 32 + 2 MAX_CHUNKS).
    T3 = (u + acc) |o| + 2^-24: the denominator and the final FP16 rounding.
    Counted constants: 5u, c_theta,i + 16, 16, 2^-21, 2u, 2^-25 (1 + u), L/16 + 32 + 2 MAX_CHUNKS, u, 2^-24.
    """
    k4, kp, v4, vp, lens = tails(data, param, indptr, indices, last, layer, S)
    T = np.shape(q)[0]
    ref = np.zeros((T, hq * HD))
    bnd = np.zeros_like(ref)
    c_theta = 2.2 * np.arange(64) * np.log2(theta) / 64 + 6
    for off, n, ctx, h, t in _prefill_ctx_heads(np.asarray(q).reshape(T, hq * HD), k4, kp, v4, vp, lens, hq, theta, data, param, indptr,
                                                indices, last, layer):
        L = ctx + n
        q_, k, v, w, o = t["q"], t["k"], t["v"], t["w"], t["o"]
        aq = np.abs(q_[:, :64] + 1j * q_[:, 64:])
        ak = np.abs(k[:, :64] + 1j * k[:, 64:])
        eps = 5 * U + E * ((c_theta + 16) * (L - 1) * t["f"] + 16)
        dl = (aq @ (ak * eps).T) / np.sqrt(HD) + 2.0 ** -21
        D = np.log((w * np.exp(dl)).sum(1))
        g = w * np.expm1(dl + D[:, None])
        t1 = np.stack([g[r, :ctx + r + 1] @ np.abs(v[:ctx + r + 1] - o[r]) for r in range(n)])
        acc = E * (L / 16 + 32 + 2 * MAX_CHUNKS)
        wk = w * np.exp(dl + D[:, None])
        av = np.abs(v)
        tiny = np.tril(w * t["Z"][:, None] < 2.0 ** -14, ctx)
        t2 = 2 * U * (wk @ av) + (2.0 ** -25 * (1 + U)) * ((tiny / t["Z"][:, None]) @ av) + acc * (wk @ av)
        t3 = (U + acc) * np.abs(o) + E
        ref[off:off + n, h * HD:(h + 1) * HD] = o
        bnd[off:off + n, h * HD:(h + 1) * HD] = t1 + t2 + t3
    return ref.reshape(T, hq, HD), bnd.reshape(T, hq, HD)


def verify_variant(q, data, param, indptr, indices, last, layer, hq, theta, S, limit_shift=0, rotate_at_last=False, head_mod=False):
    """The verify attention computed directly in float64, with the defects the negative controls plant: limit_shift moves every
    row's causal limit by that many keys; rotate_at_last rotates every query at len - 1; head_mod reads KV head h % Hkv instead of
    h // G.  With none of them it is verify_ref."""
    q = np.asarray(q).astype(np.float64)
    H = data.shape[3]
    G = hq // H
    f = R.freqs(theta)
    out = np.zeros(q.shape)
    for b in range(len(last)):
        kn, kp, vn, vp = R._sequence(data, param, indptr, indices, last, layer, b)
        L = kn.shape[1]
        pos = np.full(S, L - 1.0) if rotate_at_last else np.arange(L - S, L, dtype=np.float64)
        rq = np.exp(1j * np.multiply.outer(pos, f))
        rk = np.exp(1j * np.multiply.outer(np.arange(L, dtype=np.float64), f))
        for h in range(hq):
            hk = h % H if head_mod else h // G
            k, v = R.dequant(kn[hk], kp[hk]), R.dequant(vn[hk], vp[hk])
            qq = q[b * S:(b + 1) * S, h]
            s = (((qq[:, :64] + 1j * qq[:, 64:]) * rq) @ np.conj((k[:, :64] + 1j * k[:, 64:]) * rk).T).real / np.sqrt(HD)
            lim = np.arange(L - S, L) + limit_shift
            s[np.arange(L)[None, :] > lim[:, None]] = -np.inf
            w, _ = R._softmax(s)
            out[b * S:(b + 1) * S, h] = w @ v
    return out
