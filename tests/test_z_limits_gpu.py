"""GPU suite (-m gpu): the kernels at the edges of the ranges their C ABI entry points accept (ATOM_REQUIRE in
atom_b200/csrc/atom_b200.cu), where they take code paths the model-shaped suites never reach:

  * vocabularies that need clusters of 1 to 8 sampler CTAs, with the row maximum, exact top ties and -inf runs planted on the CTA
    boundaries, for the plain, extended (min-p, penalties, 20 log-probabilities) and draft samplers and the beam step at width 8
    with 8 stop ids;
  * the quantisers at hidden sizes up to 65536 (reorder indices >= 32768, 128 KB shared-memory rows, the rmsnorm scalar path
    with more than 16 groups), bit for bit or within 1 LSB of the oracle, and the dequantised codes within a float64 bound;
  * MoE routing, planning, gathering, combining and the whole block at top-8;
  * GEMMs with hundreds of K-groups per rank and the fused gate/up and q/k/v projections at Llama-3-70B / 405B widths;
  * the verify attention cut into 64 chunks.

The edge constants below are what tests/test_limits_cpu.py compares with the limits it reads from the sources, so raising a
limit fails the CPU suite until these tests follow it.  Fixed seeds, no retries."""
import math

import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import beam_ref as BR
from tests import moe_ref as MR
from tests import sample_penalty_ref64 as RP
from tests import sample_ref64 as RS
from tests import spec_ref as SR
from tests.test_gpu_parity import _cmp_quant, _zero_mask

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

# ------------------------------------------------------------------------------------------------ the edges tested here
SAMPLE_VOCABS = [1, 7, 32768, 32769, 131072, 131073, 151936, 256000, 262144]
SAMPLE_VOCAB_REJECTED = 262145
BEAM_VOCABS = [32768, 131073, 262144]
BEAM_SMALL_VOCABS = [5, 9]                 # width 8 against fewer (or barely more) tokens than beams
BEAM_WIDTH, BEAM_STOPS = 8, 8
REORDER_HIDDEN = [256, 2176, 16384, 32768, 40960, 65536]     # also activate_fp16_i4
RMSNORM_HIDDEN = [256, 2176, 16384, 32768]                   # also add_rmsnorm_fp16_i4
QUANT_HIDDEN_REJECTED = 65664
RMSNORM_HIDDEN_REJECTED = 32896
HIDDEN_TOO_SMALL = 128
ROUTE_HIDDEN = [256, 6144, 32768]
ROUTE_EXPERTS_TOPK = [(1, 1), (8, 8), (16, 5), (64, 6), (64, 8)]
MOE_EXPERTS, MOE_TOPK, MOE_TOPK_REJECTED = 64, 8, 9
VERIFY_NCHUNKS, VERIFY_NCHUNKS_REJECTED = 64, 65

U32 = 2.0 ** -24


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ================================================================================================ 1. vocabulary clusters
def cluster(V):
    """CTAs per sampler row and the logits each holds (sample_cluster / sample_slice): C = ceil(V / 32768) CTAs of
    slice = ceil(V / C) rounded up to a multiple of 8; the last CTA holds the rest."""
    C = -(-V // 32768)
    return C, (-(-V // C) + 7) & ~7


def boundaries(V):
    """The indices either side of every CTA boundary, and the row's ends."""
    C, s = cluster(V)
    return sorted({i for c in range(1, C) for i in (c * s - 1, c * s)} | {0, V - 1} | ({s - 1} if s - 1 < V else set()))


def _plant(l, rng):
    """In place, on FP16 rows [B, V]: row kinds by index -- the maximum on one boundary index; exact ties of the maximum on every
    boundary index; -inf runs across each boundary with the maximum just after one; the maximum at V - 1 with ties inside a
    slice.  Rows that hold NaN or only -inf are left as they are."""
    V = l.shape[1]
    bd = boundaries(V)
    for i in range(l.shape[0]):
        row = l[i].astype(np.float32)
        if np.isnan(row).any() or np.isneginf(row).all():
            continue
        top = np.float16(min(float(np.nanmax(row[np.isfinite(row)])) + 1.0, 65504.0) if np.isfinite(row).any() else 1.0)
        kind = i % 4
        if kind == 0:
            l[i, bd[(i // 4) % len(bd)]] = top
        elif kind == 1:
            l[i, bd] = top
        elif kind == 2:
            for b in bd:
                l[i, max(0, b - 3):b + 4] = -np.inf
            l[i, bd[-1]] = -np.inf
            l[i, min(V - 1, bd[len(bd) // 2] + 4)] = top
        else:
            l[i, V - 1] = top
            l[i, rng.integers(0, V, 3)] = top
    return l


def _sample_case(V, B, seed):
    from tests.test_z_sample_gpu import _logits, _params
    rng = np.random.default_rng(seed)
    l = _plant(_logits(rng, B, V), rng)
    return l, _params(rng, B, V), rng


@pytest.mark.parametrize("B", [1, 7, 33])
@pytest.mark.parametrize("V", SAMPLE_VOCABS)
def test_sampler_on_every_cluster_size(V, B):
    """Plain sampler and the extended one (min-p, penalties, logprobs = 20) against the float64 references: every token accepted,
    every log-probability and top-20 list within its bound; the penalty table incremented once per drawn token."""
    from tests.test_z_sample_gpu import _sample
    from tests.test_z_sample_penalty_gpu import _call, _options, _recorded, _table
    l, (Tm, K, P, keys, ctr), rng = _sample_case(V, B, 7 * V + B)
    RS.check_tokens(l, Tm, K, P, keys, ctr, _sample(l, Tm, K, P, keys, ctr))
    table = _table(rng, B + 3, V, saturate=True)
    opts = _options(rng, B, B + 3)
    (tok, lp, ids, lps), after = _call(l, Tm, K, P, keys, ctr, table, opts, 20)
    RP.check_tokens(l, Tm, K, P, keys, ctr, tok, penalty_table=table, logprob=lp, top_ids=ids, top_logprobs=lps, **opts)
    assert np.array_equal(after, _recorded(table, opts["slots"], tok))
    # greedy rows are the argmax of the planted rows (the first of the tied maxima), whatever CTA holds it
    g = _sample(l, np.zeros(B, np.float32), np.zeros(B, np.int32), np.ones(B, np.float32), keys, ctr)
    want = torch.argmax(T(l), dim=-1).cpu().numpy()
    finite = ~np.isnan(l.astype(np.float32)).any(1) & ~np.isneginf(l.astype(np.float32)).all(1)
    assert np.array_equal(g[finite], want[finite]), (g[finite], want[finite])


@pytest.mark.parametrize("B", [1, 7, 33])
@pytest.mark.parametrize("V", SAMPLE_VOCABS)
def test_draft_sampler_on_every_cluster_size(V, B):
    """The draft sampler against spec_ref outside its ambiguity regions; drafts on the CTA boundaries among the rest."""
    from atom_b200 import ops
    from tests.test_z_spec_gpu import _drafts, _logits, _params
    rng = np.random.default_rng(11 * V + B)
    l16 = _plant(_logits(B, V, V + B).numpy(), rng)
    Tm, K, P, M, keys, ctrs = _params(B, V + B)
    d = _drafts(l16, B, V, V + B) if V > 1 else np.where(np.arange(B) % 2, 0, -1).astype(np.int32)
    bd = boundaries(V)
    d[::4] = [bd[i % len(bd)] for i in range(len(d[::4]))]
    tok = ops.sample_tokens(T(l16), Tm, K, P, keys, ctrs, min_p=M, drafts=d.tolist()).cpu().numpy()
    ref = SR.sample_draft_np(l16, Tm, K, P, keys, ctrs, d, min_p=M)
    checked = 0
    for i in range(B):
        if SR.draft_ambiguous(l16[i], float(Tm[i]), int(K[i]), np.float32(P[i]), keys[i], ctrs[i], int(d[i]), float(M[i])):
            continue
        checked += 1
        assert tok[i] == ref[i], (i, Tm[i], K[i], P[i], M[i], d[i], tok[i], ref[i])
    assert checked >= B - max(1, B // 5)


def _stops(logits, V, W, n, rng):
    """n distinct stop ids: 0, V - 1, a CTA boundary, row 0's first and fourth tokens (inside its first W), its W-th and later
    tokens (outside), then random ones."""
    C, s = cluster(V)
    top = [int(t) for t in np.argsort(-logits[0].astype(np.float32), kind="stable")]
    want = [0, V - 1, s if s < V else V // 2, top[0], top[3 % V], top[W % V], top[(W + 5) % V]]
    out = []
    for t in want + [int(x) for x in rng.permutation(V)]:
        if t not in out:
            out.append(t)
        if len(out) == n:
            break
    return sorted(out)


def _beam_case(V, W, n_stop, seed):
    """Requests of 0 to W rows: peaked rows, exact ties of the maximum on the CTA boundaries, -inf runs over them, a NaN row."""
    rng = np.random.default_rng(seed)
    counts = [W, int(rng.integers(1, W + 1)), 0, 1, W]
    R = sum(counts)
    x = (rng.standard_normal((R, V)) * 2.5).astype(np.float32)
    bd = [b for b in boundaries(V) if b < V]
    for r in range(R):
        kind = r % 4
        if kind == 1:
            x[r, bd] = x[r].max() + 1
        elif kind == 2:
            for b in bd:
                x[r, max(0, b - 2):b + 3] = -np.inf
        elif kind == 3:
            x[r, bd[r % len(bd)]] += 12
    if R > 6:
        x[6, V // 2] = np.nan
    logits = x.astype(np.float16)
    logits[0, bd[-1]] = np.float16(np.nanmax(x[0][np.isfinite(x[0])]) + 12)   # row 0 leads its request, at V - 1
    ip = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    sums = (-rng.uniform(1, 30, R)).astype(np.float32)
    sums[0] = 0
    return logits, ip, sums, _stops(logits, V, W, n_stop, rng)


@pytest.mark.parametrize("V", BEAM_VOCABS + BEAM_SMALL_VOCABS)
def test_beam_select_at_width_8_with_8_stop_ids(V):
    """Bit for bit against beam_ref merged with the sampler's own log-probabilities; within near_tie of the float64 selection."""
    from atom_b200 import ops
    W = BEAM_WIDTH
    n_stop = min(BEAM_STOPS, V - 1)
    logits, ip, sums, stops = _beam_case(V, W, n_stop, V)
    assert len(stops) == n_stop
    R = len(logits)
    lg = T(logits)
    live, lk, fin, fk = (t.cpu().numpy() for t in ops.beam_select(lg, T(ip), T(sums), W, stops))
    n = min(ops.SAMPLE_TOP_N_MAX, V)      # W + 8 stop ids <= 16 <= 20: every candidate is among the row's first n tokens
    _, _, ids, lps = ops.sample_tokens(lg, [0.0] * R, [0] * R, [1.0] * R, [(0, r) for r in range(R)], [0] * R, logprobs=n)
    ids, lps = ids.cpu().numpy(), lps.cpu().numpy()
    lp_rows = [{int(t): lps[r, j] for j, t in enumerate(ids[r]) if t >= 0} for r in range(R)]
    exact = BR.beam_select_np(logits, ip, sums, W, stops, lp_rows=lp_rows)
    for name, got, want in zip(("live", "live_key", "fin", "fin_key"), (live, lk, fin, fk), exact):
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), (name, got, want)
    assert (live[:, :, 0] >= 0).sum() > 0 and (fin[:, :, 0] >= 0).sum() > 0
    ref = BR.beam_select_np(logits, ip, sums, W, stops)
    for i in range(len(ip) - 1):
        for a, b in zip(map(tuple, np.concatenate([live[i], fin[i]])), map(tuple, np.concatenate([ref[0][i], ref[2][i]]))):
            if a != b:
                assert a[0] >= 0 and b[0] >= 0 and BR.near_tie(logits, sums, a, b), (i, a, b)


def test_vocabulary_past_8_ctas_is_rejected():
    from atom_b200 import ops
    V = SAMPLE_VOCAB_REJECTED
    lg = torch.zeros((1, V), dtype=torch.float16, device=DEV)
    with pytest.raises(RuntimeError, match=f"vocab={V} in \\[1, {V - 1}\\]"):
        ops.sample_tokens(lg, 1.0, 0, 1.0, [(0, 0)], [0])
    with pytest.raises(RuntimeError, match=f"vocab={V}"):
        ops.beam_select(lg, torch.tensor([0, 1], dtype=torch.int32, device=DEV), torch.zeros(1, device=DEV), 2, ())


# ================================================================================================ 2. quantise kernels
def _half_ulp(x):
    return np.maximum(2.0 ** (np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -14))) - 11), 2.0 ** -25)


def dequant_check(out, X, rel, what, fp16_input=False):
    """Hold the quantiser's output `out` (o8, o4, s8, s4) to the float64 values X [m, h] it quantised (in quantiser order).

    Derivation.  The kernel quantises FP32 values x with |x - X| <= e = rel |X|, plus h(|X| (1 + rel)) when x was rounded to
    FP16 first (`fp16_input`, the rmsnorm path); `rel` bounds the relative error of the FP32 steps before the quantiser and h is
    half an FP16 ulp.  Per 128-group with divisor D (7 INT4, 127 INT8): s = fl(max|x| / D), s^ = fp16(s), r = fl(1 / s),
    q = clamp(roundf(fl(x r))).  |x / s| <= D (1 + u), so fl(x r) is within 3u D (1 + u)^2 of x / s and roundf adds half a
    step: |q s - x| <= s (1/2 + 3 D u + u) -- the clamp never binds (|q| <= D).  The stored scale is off s by at most h(s^),
    and q by at most Q = D + 1 (the code range) times that: so q s^, evaluated in float64, satisfies
        |q s^ - X| <= (s^ + h(s^)) (1/2 + (3 D + 2) u) + Q h(s^) + e.
    The scale itself: |s^ - max|X| / D| <= h(s^) + max e / D + 2 u s.  An all-zero group stores scale +0 and codes 0."""
    o8, o4, s8, s4 = [t.cpu().numpy() for t in out]
    m, h = X.shape
    g = h // 128
    q = np.concatenate([O.unpack_int4(o4.view(np.uint8)).astype(np.float64), o8.astype(np.float64)], 1).reshape(m, g, 128)
    sh = np.concatenate([O.a_scale_from_layout(s4, m).T, O.a_scale_from_layout(s8[None], m).T], 1).astype(np.float64)
    D = np.where(np.arange(g) == g - 1, 127.0, 7.0)
    Xg = X.reshape(m, g, 128)
    e = rel * np.abs(Xg) + (_half_ulp(np.abs(Xg) * (1 + rel)) if fp16_input else 0.0)
    hs = _half_ulp(sh)
    assert np.isfinite(sh).all() and (sh >= 0).all(), f"{what}: a scale is negative or not finite"
    bound = (sh + hs)[..., None] * (0.5 + (3 * D + 2)[None, :, None] * U32) + ((D + 1)[None, :, None] * hs[..., None]) + e
    err = np.abs(q * sh[..., None] - Xg)
    worst = np.unravel_index(int(np.argmax(err / bound)), err.shape)
    assert err[worst] <= bound[worst], (f"{what}: row {worst[0]} group {worst[1]} element {worst[2]}: code {q[worst]} x scale "
                                        f"{sh[worst[:2]]!r} is off X = {Xg[worst]!r} by x{err[worst] / bound[worst]:.3g} the bound")
    amax = np.abs(Xg).max(-1)
    sb = hs + e.max(-1) / D + 2 * U32 * sh
    bad = np.abs(sh - amax / D) > sb
    assert not bad.any(), f"{what}: scale of (row, group) {np.argwhere(bad)[0]} off max|X| / D beyond its bound"
    zero = amax == 0
    assert (sh[zero] == 0).all() and not q[zero].any(), f"{what}: an all-zero group must store scale 0 and codes 0"


def _quant_cases(hidden):
    return [(h, m, z) for h in hidden for m in (1, 17, 129) for z in ((False,) if m == 1 else (False, True))]


def _perm(rng, h):
    """A random reorder index of `h` columns as the kernels read it: u16 (indices >= 32768 included), passed as int16 bits."""
    return rng.permutation(h).astype(np.uint16)


def _x(rng, m, h):
    return (rng.standard_normal((m, h)) * np.where(rng.random((1, h)) > 0.97, 12.0, 1.0)).astype(np.float16)


@pytest.mark.parametrize("h,m,zeros", _quant_cases(REORDER_HIDDEN))
def test_reorder_at_every_hidden_size(h, m, zeros):
    from atom_b200 import ops
    rng = np.random.default_rng(h * 3 + m)
    x, idx = _x(rng, m, h), _perm(rng, h)
    if zeros:
        x[_zero_mask(m, h, idx)] = 0
    out = ops.reorder_fp16_i4(T(x), T(idx.view(np.int16)))
    _cmp_quant(out, O.reorder_fp16_i4(x, idx), exact=True)
    dequant_check(out, x[:, idx].astype(np.float64), 0.0, f"reorder h={h} m={m}")


@pytest.mark.parametrize("h,m,zeros", _quant_cases(REORDER_HIDDEN))
def test_activate_at_every_hidden_size(h, m, zeros):
    from atom_b200 import ops
    rng = np.random.default_rng(h * 5 + m)
    a = (rng.standard_normal((m, h)) * 2).astype(np.float16)
    b = (rng.standard_normal((m, h)) * 2).astype(np.float16)
    z = _zero_mask(m, h) if zeros else np.zeros((m, h), bool)
    a[z & (np.arange(m) % 2 == 1)[:, None]] = 0
    b[z & (np.arange(m) % 2 == 0)[:, None]] = 0
    out = ops.activate_fp16_i4(T(a), T(b))
    _cmp_quant(out, O.activate_fp16_i4(a, b), exact=False)
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    # silu(a) b in FP32: expf within 2 ulp, then 1 + e, the division and the product: 16 u is a generous relative bound
    dequant_check(out, a64 / (1 + np.exp(-a64)) * b64, 16 * U32, f"activate h={h} m={m}")


def _rms64(x, w, idx, eps):
    x64 = x.astype(np.float64)
    rstd = 1.0 / np.sqrt((x64 ** 2).mean(1, keepdims=True) + float(np.float32(eps)))
    return (x64 * w.astype(np.float64) * rstd)[:, idx]


def _rms_rel(h):
    """Relative FP32 error of fl(fl(x w) rstd) before its FP16 rounding: the sum of squares runs h/128 fmaf steps per thread and
    7 tree levels (positive terms: (h/128 + 7) u), the mean, + eps and rsqrtf (2 ulp) add 6 u; the square root halves the sum's
    part; two products add 2 u."""
    return ((h // 128 + 7) / 2 + 10) * U32


@pytest.mark.parametrize("h,m,zeros", _quant_cases(RMSNORM_HIDDEN))
def test_rmsnorm_and_fused_add_at_every_hidden_size(h, m, zeros):
    from atom_b200 import ops
    rng = np.random.default_rng(h * 7 + m)
    x, idx = _x(rng, m, h), _perm(rng, h)
    res = (rng.standard_normal((m, h)) * 2).astype(np.float16)
    if zeros:
        x[_zero_mask(m, h, idx)] = -res[_zero_mask(m, h, idx)]
    w = (1 + 0.2 * rng.standard_normal(h)).astype(np.float16)
    ti = T(idx.view(np.int16))
    s, fused = ops.add_rmsnorm_fp16_i4(T(x), T(res), T(w), ti, 1e-5)
    s_ref = T(res) + T(x)
    two = ops.rmsnorm_fp16_i4(s_ref, T(w), ti, 1e-5)
    assert torch.equal(s, s_ref)
    sel = torch.tensor([O.scale_index(r) + 2 * j for r in range(m) for j in range(4)], device=DEV)
    assert torch.equal(fused[0], two[0]) and torch.equal(fused[1], two[1])
    assert torch.equal(fused[2][sel], two[2][sel]) and torch.equal(fused[3][:, sel], two[3][:, sel])
    sn = s.cpu().numpy()
    _cmp_quant(two, O.rmsnorm_fp16_i4(sn, w, idx, 1e-5), exact=False)
    dequant_check(two, _rms64(sn, w, idx, 1e-5), _rms_rel(h), f"rmsnorm h={h} m={m}", fp16_input=True)


def test_quantisers_reject_hidden_sizes_outside_their_range():
    from atom_b200 import ops
    for h in (QUANT_HIDDEN_REJECTED, HIDDEN_TOO_SMALL):
        x = torch.zeros((2, h), dtype=torch.float16, device=DEV)
        idx = torch.zeros(h, dtype=torch.int16, device=DEV)
        with pytest.raises(RuntimeError, match=f"reorder_fp16_i4: hidden_dim={h} must be a multiple of 128 in \\[256, 65536\\]"):
            ops.reorder_fp16_i4(x, idx)
        with pytest.raises(RuntimeError, match=f"activate_fp16_i4: hidden_dim={h} must be a multiple of 128 in \\[256, 65536\\]"):
            ops.activate_fp16_i4(x, x)
    for h in (RMSNORM_HIDDEN_REJECTED, HIDDEN_TOO_SMALL):
        x = torch.zeros((2, h), dtype=torch.float16, device=DEV)
        w = torch.ones(h, dtype=torch.float16, device=DEV)
        idx = torch.zeros(h, dtype=torch.int16, device=DEV)
        msg = f"hidden_dim={h} > 32768 unsupported" if h > 256 else f"hidden_dim={h} must be a multiple of 128 in \\[256, 65536\\]"
        with pytest.raises(RuntimeError, match="rmsnorm_fp16_i4: " + msg):
            ops.rmsnorm_fp16_i4(x, w, idx, 1e-5)
        with pytest.raises(RuntimeError, match="add_rmsnorm_fp16_i4: " + msg):
            ops.add_rmsnorm_fp16_i4(x, x, w, idx, 1e-5)


# ================================================================================================ 3. MoE at top-8
def _bits(t):
    return t.contiguous().view(torch.int16) if t.dtype == torch.float16 else t.contiguous().view(torch.uint8)


def _sidx(rows):
    return torch.tensor([O.scale_index(r) for r in rows], dtype=torch.long, device=DEV)


@pytest.mark.parametrize("e,k", ROUTE_EXPERTS_TOPK)
@pytest.mark.parametrize("h", ROUTE_HIDDEN)
def test_route_at_top_8_and_every_hidden_size(h, e, k):
    """The checks of test_z_moe_gpu.test_route_matches_float64_topk.  Router rows are a spike on one channel per expert over
    small noise, so that the logits are spread far beyond the FP32 error bound at every hidden size."""
    from atom_b200 import ops
    t = 64
    g = torch.Generator(device=DEV).manual_seed(h + 100 * e + k)
    x = (torch.randn(t, h, device=DEV, generator=g) * 2).half()
    nw = (1 + 0.1 * torch.randn(h, device=DEV, generator=g)).half()
    idx_np = np.random.default_rng(h + e).permutation(h).astype(np.uint16)
    idx = T(idx_np.view(np.int16))
    wr = torch.randn(e, h, device=DEV, generator=g) / (4 * math.sqrt(h))
    wr[torch.arange(e, device=DEV), torch.randperm(h, device=DEV, generator=g)[:e]] += 2.0
    wr = wr.half()
    ids, w, lg, yn = ops.moe_route_f16(x, nw, idx, 1e-5, wr, k, router_logits=True, normed=True)
    a, b = ops.rmsnorm_fp16_i4(x, nw, idx, 1e-5), ops.reorder_fp16_i4(yn, torch.arange(h, device=DEV).to(torch.int16))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(_bits(a[2][_sidx(range(t))]), _bits(b[2][_sidx(range(t))]))
    y, wrn = yn.double().cpu().numpy(), wr.double().cpu().numpy()
    lg64 = y @ wrn.T
    bound = np.stack([MR.logit_error_bound(y[r], wrn) for r in range(t)])
    assert (np.abs(lg.double().cpu().numpy() - lg64) <= bound).all()
    ids, w = ids.cpu().numpy(), w.float().cpu().numpy()
    assert ((ids >= 0) & (ids < e)).all() and all(len(set(r)) == k for r in ids.tolist())
    srt = -np.sort(-lg64, axis=1)
    gap = srt[:, k - 1] - srt[:, k] if k < e else np.full(t, np.inf)
    ok = gap > 2 * bound.max(1)
    assert ok.mean() > 0.9
    for r in np.nonzero(ok)[0]:
        ref_ids, _ = MR.topk_f64(lg64[r], k)
        assert sorted(ids[r].tolist()) == sorted(ref_ids.tolist()), r
        p = np.exp(lg64[r] - lg64[r].max())
        w64 = p[ids[r]] / p[ids[r]].sum()
        ulp = 2.0 ** (np.floor(np.log2(np.maximum(w64, 2.0 ** -14))) - 10)
        assert (np.abs(w[r] - w64) <= ulp).all(), (r, w[r], w64)


@pytest.mark.parametrize("t", [1, 1000, 4096])
def test_plan_gather_and_combine_at_top_8(t):
    from atom_b200 import ops
    from tests.test_z_moe_gpu import _rows_equal, _scales_of
    e, k, h = MOE_EXPERTS, MOE_TOPK, 512
    rng = np.random.default_rng(t)
    ids_np = np.stack([rng.permutation(e)[:k] for _ in range(t)]).astype(np.int32)
    ids_np[: t // 3, 0] = 0                                     # a crowded expert: several tiles for one segment
    for r in range(t // 3):
        ids_np[r, 1:] = [x for x in rng.permutation(np.arange(1, e))[:k - 1]]
    ids = T(ids_np)
    bn, tmax, rows_cap = ops.moe_tiles(t, e, k)
    dest, tiles = ops.moe_plan(ids, e)
    rd, rt = MR.plan(ids_np, e, bn, tmax)
    assert np.array_equal(dest.cpu().numpy(), rd) and np.array_equal(tiles.cpu().numpy(), rt)
    x = ops.reorder_fp16_i4((torch.randn(t, h, device=DEV) * 3).half(), torch.randperm(h, device=DEV).to(torch.int16))
    ws = ops._quant_outputs(rows_cap, h, DEV)
    for a in ws:
        a.view(torch.uint8).fill_(0xFF)
    xp = ops.moe_gather_i4(x, dest, rows_cap, out=ws)
    tok = np.repeat(np.arange(t), k)
    _rows_equal(xp, rd.reshape(-1).tolist(), (x[0][T(tok)], x[1][T(tok)], *_scales_of(x, tok.tolist())), f"t={t}")
    # combine: 8 weighted summands per token, signed zeros included, against the index_add loop over experts
    y = (torch.randn(rows_cap, 256, device=DEV) * 4).half()
    y[:, :16] = -0.0
    w = torch.rand(t, k, device=DEV).half()
    w[::5, k - 1] = -0.0
    out = ops.moe_combine_f16(y, ids, w, dest)
    ref = torch.zeros(t, 256, device=DEV, dtype=torch.float16)
    for ex in range(e):
        tk, sl = np.nonzero(ids_np == ex)
        if len(tk):
            tt, ss = T(tk), T(sl)
            ref.index_add_(0, tt, (y[T(rd[tk, sl])] * w[tt, ss, None]).half())
    assert torch.equal(_bits(out), _bits(ref))
    assert (_bits(out[:, :16]) == 0).all()


@pytest.mark.parametrize("e", [8, 64])
def test_moe_block_at_top_8_equals_unfused_composition(e):
    from tests.test_z_moe_gpu import _block, _moe, _unfused
    moe = _moe(512, 256, e, MOE_TOPK, seed=e)
    for t in (1, 33, 300):
        hs = (torch.randn(t, 512, device=DEV) * 2).half()
        assert torch.equal(_bits(_block(moe, hs)), _bits(_unfused(moe, hs))), t


def test_top_k_past_8_is_rejected():
    from atom_b200 import ops
    e, k, h, t = MOE_EXPERTS, MOE_TOPK_REJECTED, 256, 4
    x = torch.zeros((t, h), dtype=torch.float16, device=DEV)
    with pytest.raises(RuntimeError, match=f"top_k={k} in \\[1, min\\(num_experts, 8\\)\\]"):
        ops.moe_route_f16(x, torch.ones(h, dtype=torch.float16, device=DEV), torch.arange(h, device=DEV).to(torch.int16), 1e-5,
                          torch.zeros((e, h), dtype=torch.float16, device=DEV), k)
    with pytest.raises(RuntimeError, match="moe_plan"):
        ops.moe_plan(torch.zeros((t, k), dtype=torch.int32, device=DEV), e, token_tile=16, tiles_max=t * k)


# ================================================================================================ 4. long-K and wide GEMMs
@pytest.mark.parametrize("n,k", [(256, 28672), (256, 53248), (1024, 16384)])
@pytest.mark.parametrize("m", [1, 16, 64])
def test_long_k_gemm_auto_dispatch(m, n, k):
    """Hundreds of K-groups per rank: bit for bit against the oracle at the split the automatic rule picks, and within the float64
    bound -- on uniform codes and on codes all at their extremes (the largest partial sums)."""
    from tests import gemm_ref64 as R
    from tests.test_z_gemm_configs_gpu import _o16
    bn, split = R.dispatch(m, n, k, 0)
    for j, regime in enumerate(("random", "extreme_mixed")):
        _o16(R.operands(regime, m, n, k, seed=m + n + k + j), 0, split, bn, f"auto {regime} {m}x{n}x{k} split {split}")


def _dev_operands(m, n, k, seed):
    """Random operands built on the device (the weights of these shapes are hundreds of MB): packed codes, keeper codes, and
    FP16 scales in the bands of make_gemm_inputs."""
    from atom_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(seed)
    G = k // 128 - 1
    u8 = lambda *s: torch.randint(0, 256, s, dtype=torch.uint8, device=DEV, generator=g)  # noqa: E731
    sc = lambda lo, hi, *s: (lo + (hi - lo) * torch.rand(s, device=DEV, generator=g)).half()  # noqa: E731
    a, b = u8(m, (k - 128) // 2), u8(n, (k - 128) // 2)
    ak, bk = u8(m, 128).view(torch.int8), u8(n, 128).view(torch.int8)
    a_s = torch.zeros((G, ops.scale_size(m)), dtype=torch.float16, device=DEV)
    aks = torch.zeros(ops.scale_size(m), dtype=torch.float16, device=DEV)
    s, sk = sc(0.02, 0.06, G, m), sc(0.05, 0.2, m)
    for j in range(4):
        a_s[:, _sidx(range(m)) + 2 * j], aks[_sidx(range(m)) + 2 * j] = s, sk
    return a, b, a_s, sc(0.005, 0.02, G, n), ak, bk, aks, sc(0.0005, 0.002, n)


def _rows(t, lo, hi):
    a, b, a_s, b_s, ak, bk, aks, bks = t
    return a, b[lo:hi], a_s, b_s[:, lo:hi].contiguous(), ak, bk[lo:hi], aks, bks[lo:hi]


def test_gateup_at_llama3_70b_width():
    """M = 16, I = 28672, K = 8192: the fused gate/up + activation equals gate, up (o16, unsplit) and activate_fp16_i4."""
    from atom_b200 import ops
    m, inter, k = 16, 28672, 8192
    t = _dev_operands(m, 2 * inter, k, 70)
    got = ops.dense_layer_gemm_i4_gateup_act(*t)
    gate = ops.dense_layer_gemm_i4_fp16(*_rows(t, 0, inter), flags=ops.GEMM_NO_SPLITK)
    up = ops.dense_layer_gemm_i4_fp16(*_rows(t, inter, 2 * inter), flags=ops.GEMM_NO_SPLITK)
    ref = ops.activate_fp16_i4(gate, up)
    sel = torch.cat([_sidx(range(m)) + 2 * j for j in range(4)])
    assert torch.equal(got[0], ref[0]), "INT8 outliers differ"
    assert torch.equal(got[1], ref[1]), f"packed INT4 differs in {int((got[1] != ref[1]).sum())} bytes"
    assert torch.equal(got[2][sel], ref[2][sel]) and torch.equal(got[3][:, sel], ref[3][:, sel]), "scales differ"


def test_qkv_gqa_at_llama3_405b_width():
    """Hq = 16384, Hkv = 2048, K = 16384: the fused q/k/v projection equals q (o16, unsplit) and k, v (o4) called alone."""
    from atom_b200 import ops
    m, hq, hkv, k = 16, 16384, 2048, 16384
    t = _dev_operands(m, hq + 2 * hkv, k, 405)
    q, (kk, ks), (vv, vs) = ops.dense_layer_gemm_i4_qkv(*t, kv_rows=hkv)
    assert torch.equal(_bits(q), _bits(ops.dense_layer_gemm_i4_fp16(*_rows(t, 0, hq), flags=ops.GEMM_NO_SPLITK))), "q differs"
    for name, d, ds, lo in (("k", kk, ks, hq), ("v", vv, vs, hq + hkv)):
        rd, rds = ops.dense_layer_gemm_i4_o4(*_rows(t, lo, lo + hkv))
        assert torch.equal(_bits(d), _bits(rd)) and torch.equal(_bits(ds), _bits(rds)), f"{name} differs"


# ================================================================================================ 5. verify in 64 chunks
def test_verify_in_64_chunks_within_bound():
    from tests.test_z_verify_gpu import _KV, _case, _run
    from atom_b200 import ops
    S, G, hkv, P = 4, 4, 2, 16
    q, pool = _case(64, [0, 37, 64 * 64 + 5, 9000], S, G * hkv, hkv, P)
    _run(q, pool, 0, S, G * hkv, f"nchunks={VERIFY_NCHUNKS}", nchunks=VERIFY_NCHUNKS)
    with pytest.raises(RuntimeError, match=f"nchunks={VERIFY_NCHUNKS_REJECTED} must be in \\[1, 64\\]"):
        ops.batch_verify_i4(T(q), _KV(*pool), 0, S, max_len=9000, nchunks=VERIFY_NCHUNKS_REJECTED)
