"""GPU suite (-m gpu): the tensor-core attention kernels -- prefill_attn_kernel<false> / <true>, verify_attn_kernel (+ its merge)
and the cascade's shared_prefix_attn_kernel -- reproduce bit for bit the SHA-256 digests in tests/golden/attn_mma_h100.npz,
written by tools/attn_mma_digests.py from a library built before the four kernels shared one tile step.  The cases, all seeded:

  * prefill without a context: G in {1, 2, 4, 8}, prompts of 1, 63, 64, 65 and 300 tokens in one batch;
  * prefill over a cached context: contexts of 0 and of lengths that are not multiples of 64 in one batch, P in {8, 16, 24, 32, 64};
  * verify: S in {1, 2, 3, 5, 8} x G in {1, 2, 4, 8}, unsplit, the automatic chunk count and more chunks than tiles; and a sequence
    shorter than its query tokens (zero rows);
  * the cascade: groups of more than 64 query rows, chunk counts that leave chunks empty, lone rows between group members;
  * RoPE bases 1e4 and 5e5.
The automatic chunk counts follow the SM count: the digests hold for a 132-SM H100."""
import hashlib
import os

import numpy as np
import pytest

from tests.attn_ctx_ref64 import make_ctx_case

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "attn_mma_h100.npz")
DEV = "cuda:0"
THETAS = [1e4, 5e5]


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _T(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


class _KV:
    def __init__(self, data, param, indptr, indices, last):
        self.data, self.param, self.indptr, self.indicies, self.last_page_offset = (_T(x) for x in (data, param, indptr, indices, last))


def _prefill(G, P, ctxs, lens, seed):
    from atom_b200 import ops
    from tests.test_z_prefill_ctx_gpu import _Kv
    hkv = 2
    theta = THETAS[seed % 2]
    (q, k4, kp, v4, vp), pool = make_ctx_case(np.random.default_rng(seed), ctxs, lens, G * hkv, hkv, P, L=2, layer=1)
    ip = _T(np.array([0] + list(np.cumsum(lens)), np.int32))
    kv = dict(kv=_Kv(*pool), layer_idx=1) if any(ctxs) else {}
    return ops.prefill_attention_i4(*(_T(x) for x in (q, k4, kp, v4, vp)), ip, seqlens=list(lens), rope_theta=theta, **kv).cpu().numpy()


def _verify(G, S, nchunks, seed, short=False):
    from atom_b200 import ops
    hkv, P = 2, [8, 16, 24, 32, 64][(G + S) % 5]
    theta = THETAS[seed % 2]
    ctxs = [0, P - 2, 3 * P + 1, 200 + S]
    (q, *_), pool = make_ctx_case(np.random.default_rng(seed), ctxs, [S] * len(ctxs), G * hkv, hkv, P)
    data, param, indptr, indices, last = pool
    if short:                    # sequence 0 keeps one page holding 2 < S tokens
        pool = (data, param, np.concatenate([[0, 1], indptr[2:] - indptr[1] + 1]).astype(np.int32),
                np.concatenate([indices[:1], indices[indptr[1]:]]).astype(np.int32), np.concatenate([[2], last[1:]]).astype(np.int32))
    lens = [(pool[2][b + 1] - pool[2][b] - 1) * P + pool[4][b] for b in range(len(ctxs))]
    return ops.batch_verify_i4(_T(q.reshape(len(ctxs) * S, G * hkv, 128)), _KV(*pool), 0, S, rope_theta=theta, max_len=max(lens),
                               nchunks=nchunks).cpu().numpy()


def _cascade(G, hkv, P, groups, lone, seed):
    import torch
    from tests.test_z_decode_shared_prefix_gpu import Case, cascade
    theta = THETAS[seed % 2]
    rng = np.random.default_rng(seed)
    case = Case(rng, P, hkv, groups, lone, L=2, layer=1, place=seed)
    q = (rng.standard_normal((len(case.rows), G * hkv, 128)) * 0.7).astype(np.float16)
    try:
        return cascade(q, case, theta)
    finally:
        case.release()
        torch.cuda.synchronize()


CASES = {}
for _G in (1, 2, 4, 8):
    CASES[f"prefill_g{_G}"] = (_prefill, (_G, 16, [0] * 5, [1, 63, 64, 65, 300], _G))
for _i, _P in enumerate((8, 16, 24, 32, 64)):
    CASES[f"prefill_ctx_p{_P}"] = (_prefill, ((1, 2, 4, 8, 4)[_i], _P, [0, 37, 130, 0, 1 + 64 * _i + 3], [65, 1, 64, 17, 129], 100 + _P))
for _G in (1, 2, 4, 8):
    for _S in (1, 2, 3, 5, 8):
        for _n in (1, 0, 7):     # unsplit, automatic, more chunks than the longest sequence's tiles
            CASES[f"verify_g{_G}_s{_S}_n{_n}"] = (_verify, (_G, _S, _n, 10 * _G + _S))
for _n in (1, 3):
    CASES[f"verify_short_n{_n}"] = (_verify, (2, 4, _n, 51, True))
CASES["cascade_g8_rows80"] = (_cascade, (8, 1, 16, [(200, [1, 5, 17, 3, 9, 2, 40, 1, 8, 6]), (70, [3, 1])], [33, 5], 1))
CASES["cascade_g4_rows96"] = (_cascade, (4, 2, 32, [(1000, [2] * 24)], [7], 2))
CASES["cascade_g1_lone"] = (_cascade, (1, 4, 8, [(64, [1, 9]), (131, [4, 4, 4])], [1, 70, 200], 3))
CASES["cascade_g2_p64"] = (_cascade, (2, 2, 64, [(128, [63, 65]), (64 * 5, [1] * 40)], [64], 4))


def compute(name):
    fn, args = CASES[name]
    return fn(*args)


@pytest.mark.gpu
def test_attention_kernels_reproduce_the_digests():
    import torch
    if torch.cuda.get_device_properties(DEV).multi_processor_count != 132:
        pytest.skip("the digests were taken on a 132-SM H100; the automatic chunk counts follow the SM count")
    golden = np.load(GOLDEN)
    assert sorted(golden.files) == sorted(CASES), "the digest file and the cases differ"
    bad = [name for name in CASES if digest(compute(name)) != str(golden[name])]
    assert not bad, f"{len(bad)} of {len(CASES)} cases differ from the digests: {bad}"
