"""Float64 reference of the INT4 paged-KV decode attention and of the INT4 prefill attention, with a per-element error bound
derived from the kernels' arithmetic.

TEST INFRASTRUCTURE ONLY.  Plain numpy, independent of oracle/atom_oracle.c and tests/gqa_oracle.c: those restate the reference's
FP32 algorithm with its own roundings, so they cannot anchor an error bound.  Here every value is float64:
  * K/V are dequantised as n * s - z from the stored fp16 (scale, zero), n the nibble (element 2j in the low nibble of byte j);
  * RoPE rotates the pairs (i, i + 64) as the complex number z = x_i + j x_{i+64} by pos * theta^(-i/64), angles in float64;
    decode rotates q at len - 1 and k at its index, prefill rotates q and k at their positions in the prompt;
  * the softmax is exact; query head h reads KV head h // G (G = query heads per KV head).

The bounds (decode_bound, prefill_bound) are written down next to each function with every constant counted from the kernels'
roundings (u = 2^-11 is the FP16 unit roundoff, e = 2^-24 the FP32 one).  None of them is fitted to a GPU run.
"""
import numpy as np

HD = 128
U = 2.0 ** -11          # FP16 unit roundoff
E = 2.0 ** -24          # FP32 unit roundoff
FP16_RUN = 4            # tokens a decode lane accumulates in one half2 run before adding it to its FP32 accumulators


def unpack(b):
    """u8 [..., 64] (two INT4 per byte, element 2j in the low nibble) -> float64 nibbles [..., 128]."""
    b = np.asarray(b, np.uint8)
    n = np.empty(b.shape[:-1] + (2 * b.shape[-1],), np.float64)
    n[..., 0::2] = b & 15
    n[..., 1::2] = b >> 4
    return n


def pack(n):
    """Nibbles [..., 128] (integers 0..15) -> u8 [..., 64]."""
    n = np.asarray(n).astype(np.uint8)
    return (n[..., 0::2] | (n[..., 1::2] << 4)).astype(np.uint8)


def freqs(theta):
    """theta_i = theta^(-i/64), i < 64, float64."""
    return float(theta) ** (-np.arange(64) / 64.0)


def rotate(x, pos, theta):
    """RoPE of x [..., n, 128] at positions pos [n]: the pair (i, i + 64) is multiplied by e^{j pos theta_i}."""
    z = x[..., :64] + 1j * x[..., 64:]
    z = z * np.exp(1j * np.multiply.outer(np.asarray(pos, np.float64), freqs(theta)))
    return np.concatenate([z.real, z.imag], -1)


def dequant(n, par):
    """nibbles [..., n, 128], (scale, zero) fp16 [..., n, 2] -> n * s - z in float64."""
    par = np.asarray(par).astype(np.float64)
    return n * par[..., :1] - par[..., 1:2]


def _softmax(s):
    m = s.max(-1, keepdims=True)
    e = np.exp(s - m)
    z = e.sum(-1, keepdims=True)
    return e / z, z[..., 0]


def _sequence(data, param, indptr, indices, last, layer, b):
    """K nibbles, K (s, z), V nibbles, V (s, z) of sequence b: [Hkv, len, 128] / [Hkv, len, 2] in float64."""
    P, H = data.shape[4], data.shape[3]
    pages = np.asarray(indices[indptr[b]:indptr[b + 1]])
    n = (len(pages) - 1) * P + int(last[b])
    d = np.asarray(data)[pages, layer].transpose(1, 2, 0, 3, 4).reshape(2, H, -1, 64)[:, :, :n]
    p = np.asarray(param)[pages, layer].astype(np.float64).transpose(1, 2, 0, 3, 4).reshape(2, H, -1, 2)[:, :, :n]
    return unpack(d[0]), p[0], unpack(d[1]), p[1]


def _decode_heads(q, data, param, indptr, indices, last, layer, hq, theta):
    """Yields (b, hkv, G query rows) with everything the reference and the bound need."""
    q = np.asarray(q).astype(np.float64)
    B, H = q.shape[0], data.shape[3]
    assert q.shape == (B, hq, HD) and hq % H == 0
    G = hq // H
    f = freqs(theta)
    for b in range(B):
        kn, kp, vn, vp = _sequence(data, param, indptr, indices, last, layer, b)
        n = kn.shape[1]
        ang = np.multiply.outer(n - 1 - np.arange(n, dtype=np.float64), f)            # [len, 64]: (len-1-t) theta_i
        for h in range(H):
            k, v = dequant(kn[h], kp[h]), dequant(vn[h], vp[h])
            zq = q[b, h * G:(h + 1) * G, :64] + 1j * q[b, h * G:(h + 1) * G, 64:]
            zk = k[:, :64] + 1j * k[:, 64:]
            s = (zq @ np.conj(zk * np.exp(-1j * ang)).T).real / np.sqrt(HD)             # Re(zq conj(zk) e^{j(len-1-t)theta})
            w, z = _softmax(s)
            yield b, h, G, dict(zq=zq, zk=zk, s=s, w=w, Z=z, o=w @ v, v=v, vn=vn[h], vp=vp[h], n=n, f=f)


def decode_ref(q, data, param, indptr, indices, last, layer, hq, theta):
    """Decode attention over the paged INT4 cache: q [B, Hq, 128]; data u8 [pages, L, 2, Hkv, P, 64]; param f16
    [pages, L, 2, Hkv, P, 2]; indptr / indices / last: the page table.  Returns float64 [B, Hq, 128]."""
    out = np.zeros((np.shape(q)[0], hq, HD))
    for b, h, G, t in _decode_heads(q, data, param, indptr, indices, last, layer, hq, theta):
        out[b, h * G:(h + 1) * G] = t["o"]
    return out


def _weight_term(w, dl, D, v, o):
    """sum_t w_t (e^{dl_t + D} - 1) |v_t - o|, row by row (w, dl [R, n]; v [n, 128]; o [R, 128])."""
    g = w * np.expm1(dl + D[:, None])
    return np.stack([g[r] @ np.abs(v - o[r]) for r in range(w.shape[0])])


def decode_bound(q, data, param, indptr, indices, last, layer, hq, theta):
    """(float64 reference [B, Hq, 128], per-element bound of |kernel - reference| [B, Hq, 128]) for batch_decode_kernel and
    batch_decode_gqa_kernel.

    Score of token t (natural log units), s_t = sum_i Re(zq_i conj(zk_ti) e^{j(len-1-t)theta_i}) / sqrt(128).  Kernel error:
      * K path, packed FP16, per component of the rotated pair (re = kre c - kim s): the dequantising HFMA2 of kre and kim
        (u |kre| |c| + u |kim| |s|), the FP16 table (u |kre| |c| + u |kim| |s|), the HMUL2 (u |kim| |s|) and the HFMA2 (u |re|):
        <= 4u (|kre| |c| + |kim| |s|) <= 4u |zk| (Cauchy-Schwarz, c^2 + s^2 = 1), likewise for im; against |qre| + |qim| <=
        sqrt2 |zq| that is 4 sqrt2 u |zq||zk|.  The FP16 rounding of the FP32 query bracket adds u |zq||zk|, the FP32 q.k sums
        (<= 16 terms + 2 shuffles) < 2^-18 relative: 6.8u in all, c_s = 7.
      * RoPE angles: the kernel uses one FP32 frequency f~_i = exp2f(-i * log2(theta) / 64) for the bracket, its step and the
        table, so the angle of pair i carries (len-1-t) (f~_i - theta_i) plus the rounding of the FP32 products pos * f~_i.  The
        exponent e_i = i log2(theta) / 64 is a product of FP32 values with <= 3e relative error (log2 theta within 1 ulp, one
        product), so f~_i is off by <= ln2 * 3e * e_i + 4e (exp2f, 2 ulp) relative; with the product's 1e and slack,
        c_theta,i = 2.2 e_i + 6 on (len-1) theta_i (6 for pair 0, whose frequency is exact).  Each page step of the FP32 bracket
        (a complex multiply by a sincosf table entry, <= 3 roundings per component + 2 ulp of the table) moves its phase and
        magnitude by <= 10e; there are at most (len-1)/8 + 2 steps (a stripe advances once per page, P * stripes >= 8).
      * subnormal FP16 intermediates on the K path: absolute 2^-25 per operation, 4 per component: 2^-22 sum_i |zq_i| / sqrt(128);
        exp2f of the scores: 2 ulp, 2^-21 in log units.
      => delta_t = sum_i |zq_i||zk_ti| (7u + e (c_theta,i (len-1) theta_i + 10 ((len-1)/8 + 2))) / sqrt(128)
         + 2^-22 sum_i|zq_i|/sqrt(128) + 2^-21.
    Softmax: the kernel's weights are w~_t = w_t e^{x_t} / sum_u w_u e^{x_u} with |x_t| <= delta_t, so with D = log sum_u w_u e^{delta_u}
    |w~_t - w_t| <= w_t (e^{delta_t + D} - 1) and, because sum_t (w~_t - w_t) = 0, the output moves by at most
      T1_i = sum_t w_t (e^{delta_t + D} - 1) |v_ti - o_i|.
    V path: sum_t p_t (n_ti s_t) is accumulated in half2 within one page and lane (at most FP16_RUN tokens per run), sum_t p_t z_t,
    the page sums and the softmax denominator in FP32.  Per token: the FP16 rounding of p s (or p s / 16 for the odd nibble couples,
    whose 16 n is exact) and one HFMA2 rounding per token of the run, each <= u times the run's partial sum of p |s| n (non-negative
    terms), so c_v = run + 2 with run = min(P/8, FP16_RUN); a subnormal p s / 16 costs n 2^-21 absolute in the page's frame, which
    is <= n 2^-21 / Z once normalised (Z = sum_t e^{s_t - max s} <= the kernel's denominator in its final frame).  The FP32 sums
    (len/8 adds per lane at most, plus merges and rescales) cost e (len/4 + 16) relative to sum_t w_t (|s_t| n_ti + |z_t|):
      T2_i = c_v sum_t n_ti max(u w~_t |s_t|, 2^-21 / Z) + e (len/4 + 16) sum_t w~_t (|s_t| n_ti + |z_t|),  w~_t = w_t e^{delta_t + D}.
    Output: the denominator's FP32 sum and the final FP16 rounding: T3_i = (u + e (len/4 + 16)) |o_i| + 2^-24.
    bound_i = T1_i + T2_i + T3_i.
    """
    P = data.shape[4]
    c_v = min(P // 8, FP16_RUN) + 2
    ref = np.zeros((np.shape(q)[0], hq, HD))
    bnd = np.zeros_like(ref)
    for b, h, G, t in _decode_heads(q, data, param, indptr, indices, last, layer, hq, theta):
        n, zq, zk, w, o = t["n"], t["zq"], t["zk"], t["w"], t["o"]
        c_theta = 2.2 * np.arange(64) * np.log2(theta) / 64 + 6
        eps = 7 * U + E * (c_theta * (n - 1) * t["f"] + 10 * ((n - 1) / 8 + 2))               # [64]
        aq = np.abs(zq)
        dl = (aq @ (np.abs(zk) * eps).T + 2.0 ** -22 * aq.sum(1, keepdims=True)) / np.sqrt(HD) + 2.0 ** -21
        D = np.log((w * np.exp(dl)).sum(1))
        t1 = _weight_term(w, dl, D, t["v"], o)
        wk = w * np.exp(dl + D[:, None])                                                    # upper bound of the kernel's weights
        s_abs, z_abs = np.abs(t["vp"][:, 0]), np.abs(t["vp"][:, 1])
        acc = E * (n / 4 + 16)
        t2 = c_v * (np.maximum(U * wk * s_abs, 2.0 ** -21 / t["Z"][:, None]) @ t["vn"]) \
            + acc * ((wk * s_abs) @ t["vn"] + (wk @ z_abs)[:, None])
        t3 = (U + acc) * np.abs(o) + E
        ref[b, h * G:(h + 1) * G] = o
        bnd[b, h * G:(h + 1) * G] = t1 + t2 + t3
    return ref, bnd


# ------------------------------------------------------------------------------------------------------------------ prefill
def _prefill_heads(q, k4, kp, v4, vp, lens, hq, theta):
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
    for L in lens:
        pos = np.arange(L, dtype=np.float64)
        ang = np.multiply.outer(pos, f)
        rot = np.exp(1j * ang)
        for h in range(hq):
            hk = h // G
            k = dequant(kn[off:off + L, hk], kpar[off:off + L, hk])
            v = dequant(vn[off:off + L, hk], vpar[off:off + L, hk])
            qq = q[off:off + L, h * HD:(h + 1) * HD]
            zq = (qq[:, :64] + 1j * qq[:, 64:]) * rot
            zk = (k[:, :64] + 1j * k[:, 64:]) * rot
            s = (zq @ np.conj(zk).T).real / np.sqrt(HD)
            s[np.triu_indices(L, 1)] = -np.inf
            w, z = _softmax(s)
            yield off, L, h, dict(q=qq, k=k, v=v, s=s, w=w, Z=z, o=w @ v, f=f)
        off += L


def prefill_ref(q, k4, kp, v4, vp, lens, hq, theta):
    """Causal attention of every prompt over its own INT4 K/V: q f16 [T, Hq*128] (pre-RoPE); k4, v4 u8 [T, Hkv*64]; kp, vp f16
    [T, Hkv*2] (scale, zero); lens: prompt lengths.  Returns float64 [T, Hq*128]."""
    out = np.zeros((np.shape(q)[0], hq * HD))
    for off, L, h, t in _prefill_heads(q, k4, kp, v4, vp, lens, hq, theta):
        out[off:off + L, h * HD:(h + 1) * HD] = t["o"]
    return out


def prefill_bound(q, k4, kp, v4, vp, lens, hq, theta, rows=None):
    """(float64 reference [T, Hq*128], bound [T, Hq*128]) for kv_dequant_rope_kernel + prefill_attn_kernel.  rows: optional
    {prompt index: row indices} limiting where the exact spread term is evaluated (elsewhere it uses |v_t - o| <= |v_t| + |o|,
    which is a matrix product); the bound is valid either way.

    Score error, per pair i (u, e as in decode_bound):
      * q is rotated in FP32 from an FP32 (cos, sin) table and rounded to FP16 once: u per component, u |zq||zk| on the score;
      * k = n s - z is rounded to FP16 (u per component), rotated in FP32 and rounded again (u): <= (sqrt2 + 1) u |zk| per
        component, (2 + sqrt2) u |zq||zk| on the score; the tensor-core FP32 sums of 128 exact products: < 2^-17 relative.
        c_s = 5 (4.5 + slack).
      * the table's angle pos * f~_i, f~_i = 1 / theta^(i/64) in FP32 (pow, reciprocal: <= 10e) and one product: <= 16 e pos theta_i
        with slack, plus 2 ulp of cosf / sinf and 3 roundings of the FP32 rotation: 8e; q and k both carry it.
      => delta_rt = sum_i |zq_ri||zk_ti| (5u + 2e (16 (L-1) theta_i + 8)) / sqrt(128) + 2^-21.
    T1 as in decode_bound.  V path: v = n s - z rounded to FP16 (u |v_t|); the softmax weights exp2(s - running max) rounded to FP16
    for the P.V product (u relative; a weight below 2^-14 in its tile's frame is subnormal, 2^-25 absolute, and such a token has
    w_t Z < 2^-14) while the denominator sums them unrounded in FP32; P.V and the tile rescales accumulate in FP32:
      T2_i = (2u + e (L/16 + 32)) sum_t w~_t |v_ti| + 2^-25 / Z sum_{t: w_t Z < 2^-14} |v_ti| (1 + u).
    T3_i = (u + e (L/16 + 32)) |o_i| + 2^-24: the FP32 denominator and the final FP16 rounding.
    """
    ref = np.zeros((np.shape(q)[0], hq * HD))
    bnd = np.zeros_like(ref)
    for pi, (off, L, h, t) in enumerate(_prefill_heads(q, k4, kp, v4, vp, lens, hq, theta)):
        prompt = pi // hq
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
        sel = range(L) if sel is None else sel
        for r in sel:
            t1[r] = g[r, :r + 1] @ np.abs(v[:r + 1] - o[r])
        acc = E * (L / 16 + 32)
        wk = w * np.exp(dl + D[:, None])
        tiny = np.tril(w * t["Z"][:, None] < 2.0 ** -14)                                  # causal keys only
        t2 = (2 * U + acc) * (wk @ av) + (2.0 ** -25 * (1 + U)) * ((tiny / t["Z"][:, None]) @ av)
        t3 = (U + acc) * np.abs(o) + E
        ref[off:off + L, h * HD:(h + 1) * HD] = o
        bnd[off:off + L, h * HD:(h + 1) * HD] = t1 + t2 + t3
    return ref, bnd


def prefill_kv_ref(k4, kp, v4, vp, lens, theta):
    """The prefill's FP16 scratch in float64: kf = RoPE(fp16(n s - z)) at each token's position in its prompt (K is rounded to
    FP16 before the rotation: the K the decode kernel reads back), vf = n s - z.  Returns (kf, vf, |zk| per pair [T, Hkv, 64],
    position [T])."""
    T = np.shape(k4)[0]
    hkv = np.shape(k4)[1] // 64
    k = dequant(unpack(np.asarray(k4).reshape(T, hkv, 64)), np.asarray(kp).reshape(T, hkv, 2))
    v = dequant(unpack(np.asarray(v4).reshape(T, hkv, 64)), np.asarray(vp).reshape(T, hkv, 2))
    k = k.astype(np.float16).astype(np.float64)
    pos = np.concatenate([np.arange(L) for L in lens]).astype(np.float64)
    kf = rotate(k.transpose(1, 0, 2), pos, theta).transpose(1, 0, 2)
    return kf.reshape(T, hkv * HD), v.reshape(T, hkv * HD), np.abs(k[..., :64] + 1j * k[..., 64:]), pos


# ------------------------------------------------------------------------------------------------------------------ pools
def make_pool(seqs, P, hkv, L=1, layer=0, extra_pages=3, rng=None, dirty=False):
    """Paged INT4 pool holding the sequences `seqs` = [(k nibbles [Hkv, n, 128], k (s, z) [Hkv, n, 2], v nibbles, v (s, z))] in
    layer `layer`, on a shuffled page order with `extra_pages` pages no sequence references.  Slots no sequence owns (the tail of
    each last page, unreferenced pages, other layers) hold zeros, or with dirty=True the bytes 0xFF and fp16 NaN parameters:
    a valid input, the kernels never read them into a result.  Returns (data, param, indptr, indices, last)."""
    rng = rng if rng is not None else np.random.default_rng(0)
    npg = [(k.shape[1] + P - 1) // P for k, _, _, _ in seqs]
    pages = sum(npg) + extra_pages
    data = np.full((pages, L, 2, hkv, P, 64), 0xFF if dirty else 0, np.uint8)
    param = np.full((pages, L, 2, hkv, P, 2), np.nan if dirty else 0, np.float16)
    perm = rng.permutation(pages)
    indptr, indices, last, c = [0], [], [], 0
    for (kn, kpar, vn, vpar), m in zip(seqs, npg):
        n = kn.shape[1]
        own = perm[c:c + m]; c += m
        indices += list(own); indptr.append(len(indices)); last.append((n - 1) % P + 1)
        for j, pg in enumerate(own):
            a, e = j * P, min(n, (j + 1) * P)
            for which, (nib, par) in enumerate(((kn, kpar), (vn, vpar))):
                data[pg, layer, which, :, :e - a] = pack(nib[:, a:e])
                param[pg, layer, which, :, :e - a] = par[:, a:e]
    return data, param, np.array(indptr, np.int32), np.array(indices, np.int32), np.array(last, np.int32)
