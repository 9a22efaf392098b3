"""CPU checks of the verify attention's float64 reference and bound (tests/attn_verify_ref64.py): at S = 1 the reference is the
decode reference, the bound is positive and finite, and three planted defects -- a causal limit one key off, every query rotated
at len - 1, and KV head h % Hkv in place of h // G -- each land outside the bound."""
import numpy as np
import pytest

from tests import attn_ref64 as R
from tests import attn_verify_ref64 as V
from tests.attn_ctx_ref64 import make_ctx_case


def _case(seed, ctxs, S, hq, hkv, P, regime="moderate"):
    rng = np.random.default_rng(seed)
    (q, *_), pool = make_ctx_case(rng, ctxs, [S] * len(ctxs), hq, hkv, P, regime=regime)
    return q.reshape(len(ctxs) * S, hq, 128), pool


@pytest.mark.parametrize("G", [1, 4])
def test_one_token_is_the_decode_reference(G):
    q, pool = _case(1, [0, 17, 70], 1, 2 * G, 2, 16)
    ref = V.verify_ref(q, *pool, 0, 2 * G, 1e4, 1)
    dec = R.decode_ref(q, *pool, 0, 2 * G, 1e4)
    assert np.allclose(ref, dec, rtol=0, atol=1e-12)


@pytest.mark.parametrize("S,G,P,regime", [(2, 1, 16, "moderate"), (5, 2, 8, "sink"), (8, 8, 32, "moderate")])
def test_bound_is_positive_and_finite_and_the_direct_form_agrees(S, G, P, regime):
    hq = 2 * G
    q, pool = _case(2, [0, 40, 130], S, hq, 2, P, regime)
    ref, bnd = V.verify_bound(q, *pool, 0, hq, 1e4, S)
    assert np.isfinite(bnd).all() and (bnd > 0).all()
    assert np.allclose(ref, V.verify_ref(q, *pool, 0, hq, 1e4, S), rtol=0, atol=1e-12)
    assert np.allclose(ref, V.verify_variant(q, *pool, 0, hq, 1e4, S), rtol=0, atol=1e-9)


@pytest.mark.parametrize("defect", [dict(limit_shift=1), dict(rotate_at_last=True), dict(head_mod=True)])
def test_negative_controls_exceed_the_bound(defect):
    S, hq, hkv = 4, 8, 4           # G = 2: h % Hkv and h // G differ
    q, pool = _case(3, [25, 60], S, hq, hkv, 16)
    ref, bnd = V.verify_bound(q, *pool, 0, hq, 1e4, S)
    bad = V.verify_variant(q, *pool, 0, hq, 1e4, S, **defect)
    assert (np.abs(bad - ref) / bnd).max() > 1.0, f"{defect} stays within the bound"
