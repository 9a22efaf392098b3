"""CPU suite: tests/attn_cascade_ref64.py on forked page tables -- the cascade's reference is attn_ref64's decode reference, its
bound is positive and finite everywhere, and a row without shared pages gets decode_bound's bound exactly."""
import numpy as np
import pytest

from tests import attn_ref64 as R
from tests.attn_cascade_ref64 import cascade_bound, cascade_ref


def forked_table(rng, P, hkv, groups, lone, vscale=1.0):
    """A pool whose groups [(shared pages, [private tokens per member])] begin on common pages, then lone rows [tokens]."""
    pages, indptr, indices, last, shared = 0, [0], [], [], []
    for n, suffixes in groups:
        common = list(range(pages, pages + n))
        pages += n
        for s in suffixes:
            own = list(range(pages, pages + -(-s // P)))
            pages += len(own)
            indices += common + own
            indptr.append(len(indices))
            last.append((s - 1) % P + 1)
            shared.append(n)
    for t in lone:
        own = list(range(pages, pages + -(-t // P)))
        pages += len(own)
        indices += own
        indptr.append(len(indices))
        last.append((t - 1) % P + 1)
        shared.append(0)
    data = rng.integers(0, 256, (pages, 1, 2, hkv, P, 64), dtype=np.uint8)
    s = rng.uniform(0.1, 1.0, (pages, 1, 2, hkv, P)) * np.array([1.0, vscale])[None, None, :, None, None]
    param = np.stack([s, s * rng.uniform(7.3, 7.7, s.shape)], -1).astype(np.float16)
    perm = rng.permutation(pages)                                     # shared pages anywhere in the pool
    return data[np.argsort(perm)], param[np.argsort(perm)], np.array(indptr, np.int32), perm[np.array(indices)].astype(np.int32), \
        np.array(last, np.int32), np.array(shared, np.int32)


@pytest.mark.parametrize("P,G,theta,groups,lone", [
    (16, 4, 1e4, [(1, [1, 5, 40])], [7]),
    (32, 1, 5e5, [(3, [32, 1]), (2, [9, 9, 70])], [1, 100]),
    (8, 8, 1e6, [(64, [3, 17])], []),
    (64, 2, 5e5, [(128, [1, 64, 65])], [8192]),                      # an 8k-token prefix and an 8k-token lone row
])
def test_reference_is_decode_attention_and_bound_is_positive_and_finite(P, G, theta, groups, lone):
    rng = np.random.default_rng(P * G)
    hkv = 2
    data, param, ip, ind, last, shared = forked_table(rng, P, hkv, groups, lone)
    q = (rng.standard_normal((len(last), G * hkv, 128)) * 0.7).astype(np.float16)
    ref = cascade_ref(q, data, param, ip, ind, last, 0, G * hkv, theta)
    assert np.array_equal(ref, R.decode_ref(q, data, param, ip, ind, last, 0, G * hkv, theta))
    ref2, bnd = cascade_bound(q, data, param, ip, ind, last, 0, G * hkv, theta, shared)
    assert np.array_equal(ref2, ref)
    assert np.isfinite(bnd).all() and (bnd > 0).all()
    # rows without shared pages get decode_bound's bound exactly
    _, dbnd = R.decode_bound(q, data, param, ip, ind, last, 0, G * hkv, theta)
    lone_rows = shared == 0
    assert np.array_equal(bnd[lone_rows], dbnd[lone_rows])


def test_bound_stays_finite_at_v_scale_16_and_with_every_row_grouped():
    rng = np.random.default_rng(3)
    data, param, ip, ind, last, shared = forked_table(rng, 32, 1, [(16, [1, 2, 3, 33])], [], vscale=16.0)
    q = (rng.standard_normal((4, 4, 128)) * 4.0).astype(np.float16)
    _, bnd = cascade_bound(q, data, param, ip, ind, last, 0, 4, 5e5, shared)
    assert np.isfinite(bnd).all() and (bnd > 0).all()
    zero = cascade_bound(q, data, param, ip, ind, last, 0, 4, 5e5, np.zeros_like(shared))[1]
    assert np.array_equal(zero, R.decode_bound(q, data, param, ip, ind, last, 0, 4, 5e5)[1])
