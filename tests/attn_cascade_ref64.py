"""Float64 reference and error bound of the shared-prefix (cascade) decode attention, on top of tests/attn_ref64.py.

TEST INFRASTRUCTURE ONLY.  The reference of a row is ordinary decode attention over the row's whole page list -- shared prefix
pages first, then its private pages -- so it is attn_ref64.decode_ref itself: sharing changes where the bytes sit, never what a
row attends to.  The bound (cascade_bound) counts every constant from the two kernels' roundings, like decode_bound and
prefill_bound next to it; none is fitted to a GPU run.
"""
import numpy as np

from tests import attn_ref64 as R
from tests.attn_ref64 import E, FP16_RUN, HD, U


def cascade_ref(q, data, param, indptr, indices, last, layer, hq, theta):
    """Decode attention of every row over its full page list: float64 [B, Hq, 128]."""
    return R.decode_ref(q, data, param, indptr, indices, last, layer, hq, theta)


def cascade_bound(q, data, param, indptr, indices, last, layer, hq, theta, shared_pages):
    """(float64 reference [B, Hq, 128], per-element bound of |kernel - reference| [B, Hq, 128]) for the cascade:
    shared_prefix_attn_kernel over the first shared_pages[b] pages of row b (n_p = shared_pages[b] * P tokens), then
    batch_decode_kernel<..., DecPrefix> over the rest, merged in FP32.  A row with shared_pages 0 gets decode_bound's bound.

    Score error of token t, per pair i (u, e as in attn_ref64):
      * prefix tokens (prefill_bound's terms, with q rotated as the decode kernel rotates it): q rotated in FP32 at len - 1 by
        sincosf of pos * exp2f(-i log2(theta) / 64) and rounded to FP16 once (u); k = fp16(n s - z) (u), rotated in FP32 from the
        (cos, sin) table of ops.rope_table and rounded (u), the tensor-core FP32 sums of 128 exact products (< 2^-17): c_s = 5 as in
        prefill_bound.  Angles: q's carries decode_bound's c_theta,i (len-1) theta_i plus 8 (sincosf, rotation), k's
        prefill_bound's 16 t theta_i + 8 <= 16 (len-1) theta_i + 8.
      * private tokens: decode_bound's c_s = 7 and angle terms c_theta,i (len-1) theta_i + 10 ((len-1)/8 + 2).
      Both are covered by eps_i = 7u + e ((c_theta,i + 16) (len-1) theta_i + 10 ((len-1)/8 + 2) + 16), plus decode_bound's
      2^-22 sum_i |zq_i| / sqrt(128) (FP16 subnormals on the decode K path) and 2^-21 (exp2f).
    T1 = sum_t w_t (e^{delta_t + D} - 1) |v_t - o| as in decode_bound (the merged softmax is one softmax with perturbed scores).
    V path: prefix tokens as in prefill_bound (v and the weight rounded to FP16: 2u relative; a weight subnormal in its chunk's
    frame is subnormal in the global one, w_t Z < 2^-14, 2^-25 / Z absolute); private tokens as in decode_bound (c_v, 2^-21 / Z).
    The FP32 sums -- prefix tiles (n_p / 16 + 32), decode lanes and stripes (len/4 + 16) and the chunk merge (<= n_p / 64 partials,
    two roundings each) -- are all below e (len/4 + 16 + len/16 + 32) = acc relative to sum_t w~_t (|s_t| n_t + |z_t|).
    T3 = (u + acc) |o| + 2^-24.
    """
    P = data.shape[4]
    c_v = min(P // 8, FP16_RUN) + 2
    ref = np.zeros((np.shape(q)[0], hq, HD))
    bnd = np.zeros_like(ref)
    for b, h, G, t in R._decode_heads(q, data, param, indptr, indices, last, layer, hq, theta):
        n, zq, zk, w, o = t["n"], t["zq"], t["zk"], t["w"], t["o"]
        npre = int(shared_pages[b]) * P
        pre = np.arange(n) < npre
        c_theta = 2.2 * np.arange(64) * np.log2(theta) / 64 + 6
        eps = 7 * U + E * ((c_theta + 16 * (npre > 0)) * (n - 1) * t["f"] + 10 * ((n - 1) / 8 + 2) + 16 * (npre > 0))
        aq = np.abs(zq)
        dl = (aq @ (np.abs(zk) * eps).T + 2.0 ** -22 * aq.sum(1, keepdims=True)) / np.sqrt(HD) + 2.0 ** -21
        D = np.log((w * np.exp(dl)).sum(1))
        t1 = R._weight_term(w, dl, D, t["v"], o)
        wk = w * np.exp(dl + D[:, None])
        s_abs, z_abs = np.abs(t["vp"][:, 0]), np.abs(t["vp"][:, 1])
        acc = E * (n / 4 + 16 + (n / 16 + 32) * (npre > 0))
        av = np.abs(t["v"])
        wp, ws = wk * pre, wk * ~pre
        tiny = (w * t["Z"][:, None] < 2.0 ** -14) * pre
        t2 = 2 * U * (wp @ av) + (2.0 ** -25 * (1 + U)) * ((tiny / t["Z"][:, None]) @ av) \
            + c_v * (np.maximum(U * ws * s_abs, 2.0 ** -21 / t["Z"][:, None] * ~pre) @ t["vn"]) \
            + acc * ((wk * s_abs) @ t["vn"] + (wk @ z_abs)[:, None])
        t3 = (U + acc) * np.abs(o) + E
        ref[b, h * G:(h + 1) * G] = o
        bnd[b, h * G:(h + 1) * G] = t1 + t2 + t3
    return ref, bnd
