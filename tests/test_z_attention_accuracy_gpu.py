"""GPU accuracy suite (-m gpu) of the attention kernels: batch_decode_kernel at every group size and the prefill kernels
against the float64 reference of tests/attn_ref64.py, element by element inside the bound derived there from the kernels'
arithmetic (|kernel - ref64| <= bound; the assert message gives the worst error-to-bound ratio, and every passing case prints it).

The inputs are the regimes a model produces rather than a flat softmax: centred K/V (zero ~ 7.5 * scale, scales in [0.1, 1])
with logit spreads from flat to one-hot; exact score patterns placed on chosen pages, stripes and tokens through the
lowest-frequency RoPE pair; page sizes 8, 16, 24, 32 and 64 and every group size, which reach every kernel instantiation;
contexts of 8k and 32k tokens; pools whose unused slots hold 0xFF bytes and NaN parameters; V page sums driven to the edge
of their FP16 range.  Fixed seeds, no retries."""
import numpy as np
import pytest
import torch

from tests import attn_ref64 as R

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
LN2 = np.log(2.0)
# kernel variant -> (query heads, KV heads, RoPE base or None = varies with the case, page stripes S)
VARIANTS = {
    "mha": (2, 2, 1e4, 4),       # batch_decode_kernel<1, ...>: one query head per KV head at base 1e4
    "g1": (2, 2, 5e5, 4),        # batch_decode_kernel<1, ...>: multi-head at another base
    "g2": (4, 2, None, 4),
    "g4": (8, 2, None, 2),
    "g8": (8, 1, None, 1),
}
PAGES = [8, 16, 24, 32, 64]
THETAS = [1e4, 5e5, 1e6]


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


class _KV:
    def __init__(self, data, param, indptr, indices, last):
        self.data, self.param, self.indptr, self.indicies, self.last_page_offset = T(data), T(param), T(indptr), T(indices), T(last)


def _theta(variant, P):
    t = VARIANTS[variant][2]
    return t if t is not None else THETAS[PAGES.index(P) % 3]


def _decode(q, pool, layer, theta):
    from atom_b200 import ops
    return ops.batch_decode_i4(T(q), _KV(*pool), layer, rope_theta=theta).cpu().numpy()


def _check(got, ref, bnd, what):
    got = got.astype(np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output ({np.count_nonzero(~np.isfinite(got))} elements)"
    ratio = np.abs(got - ref) / bnd
    worst = float(ratio.max())
    at = np.unravel_index(int(ratio.argmax()), ratio.shape)
    assert worst <= 1.0, f"{what}: |kernel - ref64| exceeds the bound, worst error/bound = {worst:.3f} at {at} " \
                         f"(kernel {got[at]:.6g}, ref {ref[at]:.6g}, bound {bnd[at]:.3g})"
    print(f"worst error/bound {what}: {worst:.4f}")
    return worst


def _centred(rng, hkv, n, kscale=(0.1, 1.0), vscale=(0.1, 1.0)):
    """Random K/V nibbles with scales in the given range and zero ~ 7.5 * scale: values centred on 0."""
    def part(lo, hi):
        s = rng.uniform(lo, hi, (hkv, n))
        return rng.integers(0, 16, (hkv, n, 128)), np.stack([s, s * rng.uniform(7.3, 7.7, (hkv, n))], -1).astype(np.float16)
    return part(*kscale) + part(*vscale)


# logit std ~ 2.8 * sigma_q for the centred K above: 0.25 (flat), 2 (moderate), 11 (peaked)
SIGMA_Q = {"flat": 0.09, "moderate": 0.7, "peaked": 4.0}


# ------------------------------------------------------------------------------------------------ 1. score regimes, dirty pool
@pytest.mark.parametrize("regime", list(SIGMA_Q))
@pytest.mark.parametrize("P", PAGES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_decode_regimes_within_bound_and_blind_to_unused_slots(variant, P, regime):
    hq, hkv, _, S = VARIANTS[variant]
    theta = _theta(variant, P)
    seed = 1000 * list(VARIANTS).index(variant) + 10 * P + list(SIGMA_Q).index(regime)
    rng = np.random.default_rng(seed)
    lens = [1, P - 1, P, P + 1, S * P - 1, S * P + 1, 2 * S * P + 3, 300]
    seqs = [_centred(rng, hkv, n) for n in lens]
    q = (rng.standard_normal((len(lens), hq, 128)) * SIGMA_Q[regime]).astype(np.float16)
    pool = R.make_pool(seqs, P, hkv, L=2, layer=1, rng=np.random.default_rng(seed))
    got = _decode(q, pool, 1, theta)
    ref, bnd = R.decode_bound(q, *pool, 1, hq, theta)
    _check(got, ref, bnd, f"{regime} {variant} P={P} theta={theta:g}")
    # the same call on a pool whose unused slots (tails of last pages, unreferenced pages, layer 0) are 0xFF / NaN
    dirty = R.make_pool(seqs, P, hkv, L=2, layer=1, rng=np.random.default_rng(seed), dirty=True)
    assert all(np.array_equal(a, b) for a, b in zip(dirty[2:], pool[2:]))           # the same page table
    assert np.array_equal(_decode(q, dirty, 1, theta).view(np.uint16), got.view(np.uint16))


# ------------------------------------------------------------------------------------------------ 2. exact score patterns
A63 = 8.0          # q's whole weight, on the lowest-frequency pair i = 63


def _pattern_seq(rng, levels, theta, nib_v=None, vscale=(0.1, 1.0)):
    """One KV head whose scores are `levels` (nats, >= 0): K is zero except element 63 = 15 * s_t (nibble 15, zero 0), so with
    q = A63 on element 63 the score is A63 * 15 s_t cos((len-1-t) theta_63) / sqrt(128), and s_t is solved for."""
    n = len(levels)
    cos = np.cos((n - 1 - np.arange(n)) * theta ** (-63 / 64))
    kn = np.zeros((1, n, 128)); kn[0, :, 63] = 15
    kp = np.zeros((1, n, 2)); kp[0, :, 0] = np.asarray(levels) * np.sqrt(128) / (A63 * 15 * cos)
    _, _, vn, vp = _centred(rng, 1, n, vscale=vscale)
    if nib_v is not None:
        vn = np.full_like(vn, nib_v)
    return kn, kp.astype(np.float16), vn, vp


def _scores(seqs, P, theta):
    """The float64 scores the reference sees for each pattern sequence (one KV head, q on pair 63)."""
    pool = R.make_pool(seqs, P, 1)
    q = np.zeros((len(seqs), 1, 128), np.float16); q[:, 0, 63] = A63
    return [t["s"][0] for _, _, _, t in R._decode_heads(q, *pool, 0, 1, theta)]


def _rise(rng, S, P, rises, base=4.5):
    """Every stripe sees page maxima rising by `rises` (log2 units) from one of its pages to the next; the other tokens of a
    page sit 1 to 4 nats below its maximum."""
    npg = S * (len(rises) + 1)
    top = base + LN2 * np.concatenate([[0], np.cumsum(rises)])
    lv = np.empty(npg * P)
    for pg in range(npg):
        lv[pg * P:(pg + 1) * P] = top[pg // S] - rng.uniform(1, 4, P)
        lv[pg * P + rng.integers(P)] = top[pg // S]
    return lv


@pytest.mark.parametrize("P", PAGES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_decode_exact_score_patterns(variant, P):
    """In one batch: the maximum on the first token; on the last token of a partial last page; on a page of each stripe; one
    token 45 nats above the rest; page maxima rising by 5.9 then 6.1 log2 units (the lazy rescale skipped, then taken) and by
    6.1 then 5.9."""
    _, _, _, S = VARIANTS[variant]
    hkv, theta = 1, _theta(variant, P)
    G = {"mha": 1, "g1": 1, "g2": 2, "g4": 4, "g8": 8}[variant]
    rng = np.random.default_rng(77 + P + 100 * G)
    low = lambda n: rng.uniform(0, 2, n)
    pats = []
    lv = low(S * P + P // 2 + 1); lv[0] = 12.0; pats.append(lv)                            # first token
    lv = low(2 * S * P + P // 2 + 1); lv[-1] = 12.0; pats.append(lv)                       # last token of a partial last page
    for s in range(S):                                                                     # a page of stripe s
        lv = low(2 * S * P + 3); lv[(S + s) * P + rng.integers(P)] = 12.0; pats.append(lv)
    lv = low(S * P + 5); lv[rng.integers(len(lv))] = 45.0; pats.append(lv)                 # one-hot
    pats.append(_rise(rng, S, P, [5.9, 6.1]))
    pats.append(_rise(rng, S, P, [6.1, 5.9]))
    seqs = [_pattern_seq(rng, lv, theta) for lv in pats]
    # the patterns as realised after FP16 rounding of the scales: the rises keep 0.05 log2 units from the threshold 6
    for lv, s in zip(pats[-2:], _scores(seqs[-2:], P, theta)):
        tops = [s[pg * P:(pg + 1) * P].max() for pg in range(len(s) // P)]
        steps = np.diff(np.array(tops).reshape(-1, S).T, axis=1) / LN2      # [stripe, rise]
        assert (np.abs(np.abs(steps - 6) - 0.1) < 0.05).all(), steps
    # G query heads per KV head: every query head carries the pattern, at its own amplitude
    q = np.zeros((len(seqs), G * hkv, 128), np.float16)
    q[:, :, 63] = A63 * (1 - 0.05 * np.arange(G))
    pool = R.make_pool(seqs, P, hkv, rng=np.random.default_rng(P))
    got = _decode(q, pool, 0, theta)
    ref, bnd = R.decode_bound(q, *pool, 0, q.shape[1], theta)
    _check(got, ref, bnd, f"patterns {variant} P={P} theta={theta:g}")


# ------------------------------------------------------------------------------------------------ 3. long contexts
@pytest.mark.parametrize("regime", ["moderate", "peaked"])
@pytest.mark.parametrize("n,variant,P,theta", [(8192, "mha", 16, 1e4), (32768, "g4", 32, 5e5), (32768, "g1", 64, 1e6),
                                               (8192, "g8", 24, 1e6), (32768, "mha", 8, 1e4)])
def test_decode_long_contexts(n, variant, P, theta, regime):
    hq, hkv, _, _ = VARIANTS[variant]
    hq, hkv = hq // hkv, 1                        # one KV head: the float64 reference stays cheap
    rng = np.random.default_rng(n + P)
    lens = [n, n - 37]
    seqs = [_centred(rng, hkv, m) for m in lens]
    q = (rng.standard_normal((2, hq, 128)) * SIGMA_Q[regime]).astype(np.float16)
    pool = R.make_pool(seqs, P, hkv, rng=rng)
    got = _decode(q, pool, 0, theta)
    ref, bnd = R.decode_bound(q, *pool, 0, hq, theta)
    _check(got, ref, bnd, f"long {regime} {variant} len={n} P={P} theta={theta:g}")


# ------------------------------------------------------------------------------------------------ 4. FP16 range of the V page sums
@pytest.mark.parametrize("vscale", [4.0, 12.0, 16.0])
@pytest.mark.parametrize("P", [32, 64])
@pytest.mark.parametrize("variant", ["mha", "g4"])
def test_decode_v_page_sums_stay_finite_at_large_v_scales(variant, P, vscale):
    """Every V nibble 15 and every token of a page 5.95 log2 units above the running maximum, which the lazy rescale keeps: the
    softmax weights reach 2^5.95 = 62 and a half2 run holds 4 tokens x 15 x 62 x scale, 59 000 at scale 16 (FP16 max 65 504).
    The next page rises by 8 more (rescaled).  Scales up to 16 are inside the documented range for every page size."""
    hq, _, _, S = VARIANTS[variant]
    G = hq // VARIANTS[variant][1]
    theta = _theta(variant, P)
    rng = np.random.default_rng(int(vscale) + P)
    lv = np.concatenate([np.full(S * P, base) for base in LN2 * np.array([0.5, 6.45, 14.45])])
    seqs = [_pattern_seq(rng, lv, theta, nib_v=15, vscale=(vscale, vscale))]
    top = [s.reshape(-1, P).max(1) for s in _scores(seqs, P, theta)][0]
    assert 5.9 < (top[S] - top[0]) / LN2 < 6.0
    q = np.zeros((1, G, 128), np.float16); q[0, :, 63] = A63
    pool = R.make_pool(seqs, P, 1)
    got = _decode(q, pool, 0, theta)
    ref, bnd = R.decode_bound(q, *pool, 0, G, theta)
    _check(got, ref, bnd, f"V envelope {variant} P={P} scale={vscale:g}")


# ------------------------------------------------------------------------------------------------ 5. prefill
def _prefill_case(rng, lens, hq, hkv, regime):
    t = sum(lens)
    kn = rng.integers(0, 16, (t, hkv, 128))
    vn = rng.integers(0, 16, (t, hkv, 128))
    par = lambda: (lambda s: np.stack([s, s * rng.uniform(7.3, 7.7, s.shape)], -1))(rng.uniform(0.1, 1, (t, hkv)))
    kp, vp = par(), par()
    if regime == "moderate":
        q = rng.standard_normal((t, hq, 128)) * SIGMA_Q["moderate"]
    else:
        # an attention sink (the first token of every prompt) and a maximum that moves on in every later 64-token tile: q has a
        # large lowest-frequency pair, and K's element 63 is 7.5 s (nibble 15) there with s growing from tile to tile
        q = rng.standard_normal((t, hq, 128)) * 0.3
        q[:, :, 63] = 24.0
        off = 0
        for L in lens:
            kn[off, :, 63] = 15; kp[off, :, 0] = 1.0; kp[off, :, 1] = 7.5
            for j in range(1, (L + 63) // 64):
                tok = off + min(64 * j + int(rng.integers(64)), L - 1)
                kn[tok, :, 63] = 15; kp[tok, :, 0] = 1.0 + 0.1 * j; kp[tok, :, 1] = 7.5 * kp[tok, :, 0]
            off += L
    return (q.astype(np.float16).reshape(t, hq * 128), R.pack(kn).reshape(t, hkv * 64), kp.astype(np.float16).reshape(t, 2 * hkv),
            R.pack(vn).reshape(t, hkv * 64), vp.astype(np.float16).reshape(t, 2 * hkv))


def _prefill(q, k4, kp, v4, vp, lens, hq, hkv, theta):
    from atom_b200 import _lib, ops
    t = sum(lens)
    args = [T(x) for x in (q, k4, kp, v4, vp)]
    ip = T(np.array([0] + list(np.cumsum(lens)), np.int32))
    pos = T(np.concatenate([np.arange(n) for n in lens]).astype(np.int32))
    table = ops.rope_table(max(lens), torch.device(DEV), theta)
    kf = torch.empty(t, hkv * 128, dtype=torch.float16, device=DEV)
    vf, out = torch.empty_like(kf), torch.empty(t, hq * 128, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().atom_prefill_attention_gqa_i4(*[a.data_ptr() for a in args], ip.data_ptr(), pos.data_ptr(), table.data_ptr(),
                                                        kf.data_ptr(), vf.data_ptr(), out.data_ptr(), t, len(lens), max(lens), hq, hkv,
                                                        torch.cuda.current_stream().cuda_stream), "prefill_attention_gqa_i4")
    return out.cpu().numpy(), kf.cpu().numpy(), vf.cpu().numpy()


def _check_scratch(kf, vf, k4, kp, v4, vp, lens, theta):
    """kf within one FP16 ulp (plus the FP32 RoPE angle error, 2^-24 (32 pos theta_i + 8) |zk|) of RoPE(fp16(n s - z)) at the
    token's position, pairs (i, i + 64); vf within one FP16 ulp of n s - z."""
    kr, vr, zk, pos = R.prefill_kv_ref(k4, kp, v4, vp, lens, theta)
    t, hkv = kf.shape[0], kf.shape[1] // 128
    ulp = lambda x: np.spacing(np.abs(x).astype(np.float16)).astype(np.float64)
    ang = R.E * (32 * np.multiply.outer(pos, R.freqs(theta)) + 8)[:, None, :] * zk            # [T, Hkv, 64]
    tol = ulp(kr) + np.concatenate([ang, ang], -1).reshape(t, hkv * 128) + 2.0 ** -24
    bad = np.abs(kf.astype(np.float64) - kr) > tol
    assert not bad.any(), f"kf: {np.count_nonzero(bad)} elements off, first at {np.argwhere(bad)[0]}"
    bad = np.abs(vf.astype(np.float64) - vr) > ulp(vr) + 2.0 ** -24
    assert not bad.any(), f"vf: {np.count_nonzero(bad)} elements off, first at {np.argwhere(bad)[0]}"


@pytest.mark.parametrize("theta", [1e4, 5e5])
@pytest.mark.parametrize("regime", ["sink", "moderate"])
@pytest.mark.parametrize("hq,hkv", [(2, 2), (8, 2), (8, 1)])
def test_prefill_within_bound(hq, hkv, regime, theta):
    lens = [1, 63, 64, 65, 127, 128, 129]
    rng = np.random.default_rng(hq * 10 + hkv + (regime == "sink"))
    case = _prefill_case(rng, lens, hq, hkv, regime)
    got, kf, vf = _prefill(*case, lens, hq, hkv, theta)
    _check_scratch(kf, vf, *case[1:], lens, theta)
    ref, bnd = R.prefill_bound(*case, lens, hq, theta)
    _check(got, ref, bnd, f"prefill {regime} G={hq // hkv} theta={theta:g}")


def test_prefill_4096_token_prompt_within_bound():
    lens, hq, hkv, theta = [4096], 2, 1, 5e5
    rng = np.random.default_rng(4096)
    case = _prefill_case(rng, lens, hq, hkv, "sink")
    got, kf, vf = _prefill(*case, lens, hq, hkv, theta)
    _check_scratch(kf, vf, *case[1:], lens, theta)
    # the exact spread term on 320 rows (the first and last tiles, both sides of every eighth tile boundary, random rows); the
    # looser form |v_t - o| <= |v_t| + |o| everywhere else
    rows = sorted(set(range(64)) | set(range(4032, 4096)) | {64 * j + d for j in range(1, 64, 8) for d in (-1, 0)}
                  | set(rng.choice(4096, 160, replace=False).tolist()))
    ref, bnd = R.prefill_bound(*case, lens, hq, theta, rows={0: rows})
    _check(got, ref, bnd, "prefill sink 4096 G=2")
