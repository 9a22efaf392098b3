"""CPU checks of tests/attn_ref64.py, the float64 attention reference the GPU accuracy suite measures the kernels against: it
agrees with the two FP32 oracles and with a torch float64 SDPA, it has the invariances of attention over a paged cache, and
its error bound is positive and finite wherever it is used."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import attn_ref64 as R
from tests import gqa_oracle as GO


def _flat(rng, hkv, P, lens, L=2):
    """The decode suites' flat fixture: K/V scales in [0.01, 0.05], zeros in [0, 0.4], q ~ N(0, 1)."""
    pages = sum((n + P - 1) // P for n in lens) + 3
    data = rng.integers(0, 256, (pages, L, 2, hkv, P, 64), dtype=np.uint8)
    param = np.stack([rng.uniform(0.01, 0.05, (pages, L, 2, hkv, P)), rng.uniform(0, 0.4, (pages, L, 2, hkv, P))], -1).astype(np.float16)
    perm = rng.permutation(pages)
    indptr, indices, last, c = [0], [], [], 0
    for n in lens:
        npg = (n + P - 1) // P
        indices += list(perm[c:c + npg]); c += npg
        indptr.append(len(indices)); last.append((n - 1) % P + 1)
    return data, param, np.array(indptr, np.int32), np.array(indices, np.int32), np.array(last, np.int32)


def _fp32_close(ref, orc):
    # the oracles compute in FP32 and round to FP16: half an FP16 ulp plus FP32 noise
    err = np.abs(ref - orc.astype(np.float64)) - (R.U * np.abs(ref) + 2e-6)
    assert err.max() <= 0, f"worst excess {err.max():.3e}"


@pytest.mark.parametrize("P,lens", [(16, [1, 37, 64, 499]), (8, [8, 9, 1, 100]), (32, [777, 33]), (24, [23, 25, 200]), (64, [1, 65, 300])])
def test_decode_ref_matches_the_multi_head_oracle(P, lens):
    rng = np.random.default_rng(P)
    data, param, indptr, indices, last = _flat(rng, 3, P, lens)
    q = rng.standard_normal((len(lens), 3, 128)).astype(np.float16)
    for layer in (0, 1):
        ref = R.decode_ref(q, data, param, indptr, indices, last, layer, 3, 1e4)
        _fp32_close(ref, O.batch_decode_i4(q, data, param, indptr, indices, last, layer))


@pytest.mark.parametrize("hq,hkv,theta", [(4, 2, 5e5), (8, 1, 1e6), (8, 4, 1e4)])
def test_decode_ref_matches_the_gqa_oracle(hq, hkv, theta):
    rng = np.random.default_rng(hq + hkv)
    lens = [1, 17, 300, 64]
    data, param, indptr, indices, last = _flat(rng, hkv, 16, lens)
    q = rng.standard_normal((len(lens), hq, 128)).astype(np.float16)
    ref = R.decode_ref(q, data, param, indptr, indices, last, 1, hq, theta)
    _fp32_close(ref, GO.batch_decode_gqa_i4(q, data, param, indptr, indices, last, 1, theta=theta))


def _prefill_inputs(rng, lens, hq, hkv):
    t = sum(lens)
    q = (rng.standard_normal((t, hq * 128)) * 1.5).astype(np.float16)
    k4, v4 = (rng.integers(0, 256, (t, hkv * 64), dtype=np.uint8) for _ in range(2))
    par = lambda: np.stack([rng.uniform(0.1, 1, (t, hkv)), rng.uniform(0, 7.5, (t, hkv))], -1).astype(np.float16).reshape(t, 2 * hkv)
    return q, k4, par(), v4, par()


@pytest.mark.parametrize("lens,hq,hkv,theta", [([5, 64, 70], 4, 2, 1e4), ([130, 1], 8, 1, 5e5), ([33], 2, 2, 1e6)])
def test_prefill_ref_matches_torch_sdpa(lens, hq, hkv, theta):
    rng = np.random.default_rng(sum(lens))
    q, k4, kp, v4, vp = _prefill_inputs(rng, lens, hq, hkv)
    ref = R.prefill_ref(q, k4, kp, v4, vp, lens, hq, theta)
    t = sum(lens)
    # the same attention written the other way round: real rotate-half RoPE (x cos + rotate_half(x) sin), torch SDPA
    deq = lambda x4, p: torch.from_numpy(R.unpack(x4.reshape(t, hkv, 64)) * p.astype(np.float64).reshape(t, hkv, 2)[..., :1]
                                        - p.astype(np.float64).reshape(t, hkv, 2)[..., 1:])
    k, v = deq(k4, kp), deq(v4, vp)
    qt = torch.from_numpy(q.astype(np.float64)).view(t, hq, 128)
    inv = 1.0 / (theta ** (torch.arange(0, 128, 2, dtype=torch.float64) / 128))
    off = 0
    for n in lens:
        ang = torch.outer(torch.arange(n, dtype=torch.float64), inv)
        cos, sin = torch.cat([ang.cos()] * 2, -1)[:, None], torch.cat([ang.sin()] * 2, -1)[:, None]
        rot = lambda x: x * cos + torch.cat([-x[..., 64:], x[..., :64]], -1) * sin
        qq = rot(qt[off:off + n]).transpose(0, 1)
        kk = rot(k[off:off + n]).transpose(0, 1).repeat_interleave(hq // hkv, 0)
        vv = v[off:off + n].transpose(0, 1).repeat_interleave(hq // hkv, 0)
        o = torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, is_causal=True).transpose(0, 1).reshape(n, hq * 128)
        np.testing.assert_allclose(ref[off:off + n], o.numpy(), rtol=1e-10, atol=1e-10)
        off += n


def test_permuting_the_physical_pages_changes_nothing():
    rng = np.random.default_rng(7)
    P, lens = 16, [40, 1, 100]
    data, param, indptr, indices, last = _flat(rng, 2, P, lens)
    q = rng.standard_normal((3, 4, 128)).astype(np.float16)
    ref = R.decode_ref(q, data, param, indptr, indices, last, 0, 4, 5e5)
    perm = rng.permutation(data.shape[0])                       # physical page p moves to slot perm[p]
    d2, p2 = np.empty_like(data), np.empty_like(param)
    d2[perm], p2[perm] = data, param
    assert np.array_equal(ref, R.decode_ref(q, d2, p2, indptr, perm[indices].astype(np.int32), last, 0, 4, 5e5))


def test_gqa_equals_multi_head_attention_on_the_repeated_cache():
    rng = np.random.default_rng(8)
    lens = [33, 7]
    data, param, indptr, indices, last = _flat(rng, 2, 8, lens)
    q = rng.standard_normal((2, 8, 128)).astype(np.float16)
    rd, rp = GO.repeat_heads(data, param, 4)
    np.testing.assert_allclose(R.decode_ref(q, data, param, indptr, indices, last, 1, 8, 1e6),
                               R.decode_ref(q, rd, rp, indptr, indices, last, 1, 8, 1e6), rtol=1e-12, atol=1e-15)


def test_a_token_dominant_by_more_than_40_nats_is_the_output():
    """q on the lowest-frequency pair only, K zero except that pair: the score of token t is q_63 k_t cos((len-1-t) theta_63) /
    sqrt(128); one token 45 nats above the rest leaves its own V (to e^-45 relative)."""
    rng = np.random.default_rng(9)
    P, n, star = 16, 70, 23
    kn = np.zeros((1, n, 128)); kn[0, :, 63] = 1
    kp = np.zeros((1, n, 2)); kp[0, :, 0] = 0.25
    kp[0, star, 0] = 0.25 + 45 * np.sqrt(128) / 16 / np.cos((n - 1 - star) * 1e4 ** (-63 / 64))    # 45 nats above the others
    vn = rng.integers(0, 16, (1, n, 128)).astype(np.float64)
    vp = np.stack([rng.uniform(0.1, 1, (1, n)), rng.uniform(0, 7, (1, n))], -1)
    seq = (kn, kp.astype(np.float16), vn, vp.astype(np.float16))
    data, param, indptr, indices, last = R.make_pool([seq], P, 1)
    q = np.zeros((1, 1, 128), np.float16); q[0, 0, 63] = 16
    s = None
    for _, _, _, t in R._decode_heads(q, data, param, indptr, indices, last, 0, 1, 1e4):
        s = t["s"][0]
    assert np.sort(s)[-1] - np.sort(s)[-2] > 40
    ref = R.decode_ref(q, data, param, indptr, indices, last, 0, 1, 1e4)[0, 0]
    v_star = R.dequant(vn[0, star], seq[3][0, star])
    np.testing.assert_allclose(ref, v_star, rtol=0, atol=1e-12 * np.abs(v_star).max())


@pytest.mark.parametrize("P", [8, 16, 24, 32, 64])
def test_bounds_are_positive_and_finite(P):
    rng = np.random.default_rng(P + 1)
    lens = [1, P - 1, P + 1, 300]
    data, param, indptr, indices, last = _flat(rng, 2, P, lens)
    q = rng.standard_normal((len(lens), 8, 128)).astype(np.float16)
    ref, bnd = R.decode_bound(q, data, param, indptr, indices, last, 1, 8, 5e5)
    assert np.isfinite(bnd).all() and (bnd > 0).all() and np.isfinite(ref).all()
    assert np.array_equal(ref, R.decode_ref(q, data, param, indptr, indices, last, 1, 8, 5e5))
    lens = [1, 63, 64, 65]
    qp, k4, kp, v4, vp = _prefill_inputs(rng, lens, 4, 1)
    ref, bnd = R.prefill_bound(qp, k4, kp, v4, vp, lens, 4, 1e4)
    assert np.isfinite(bnd).all() and (bnd > 0).all()
    assert np.array_equal(ref, R.prefill_ref(qp, k4, kp, v4, vp, lens, 4, 1e4))
    # the sampled-row form is looser elsewhere, never tighter
    _, loose = R.prefill_bound(qp, k4, kp, v4, vp, lens, 4, 1e4, rows={3: [0, 64]})
    assert (loose >= bnd * (1 - 1e-12)).all()
