"""GPU suite (-m gpu): the beam step (ops.beam_select) against tests/beam_ref.py -- bit for bit once merged with the sampler's own
log-probabilities, and within the reference's bound of the float64 ones -- and the batched page copy (ops.copy_kv_pages), eager
and replayed from a CUDA graph with new pairs."""
import numpy as np
import pytest
import torch

from atom_b200 import ops
from tests import beam_ref as BR

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _case(V, W, seed):
    """Requests of 1 to W rows and empty ones; peaked rows, exact ties, -inf entries and a NaN row; stop ids inside and outside
    the rows' first W tokens."""
    rng = np.random.default_rng(seed)
    counts = [int(c) for c in rng.integers(0, W + 1, 6)] + [W, 1, 0]
    R = sum(counts)
    x = (rng.standard_normal((R, V)) * 2.5).astype(np.float32)
    for r in range(R):
        kind = r % 5
        if kind == 1:
            x[r, rng.integers(0, V)] += 12                          # peaked
        elif kind == 2:
            x[r, rng.choice(V, 6, replace=False)] = x[r].max() + 1  # exact ties at the top
        elif kind == 3:
            x[r, rng.choice(V, V // 3, replace=False)] = -np.inf
    if R > 4:
        x[4, 7] = np.nan
    logits = x.astype(np.float16)
    ip = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    # row 0 is peaked and has the largest sum: its argmax, a stop id, ranks first in its request
    logits[0, int(np.argmax(x[0]))] = np.float16(x[0].max() + 12)
    sums = (-rng.uniform(1, 30, R)).astype(np.float32)
    sums[0] = 0
    top = np.argsort(-logits[0].astype(np.float32), kind="stable")
    stops = sorted({int(top[0]), int(top[W]), int(rng.integers(0, V)), int(rng.integers(0, V))})
    return logits, ip, sums, stops


@pytest.mark.parametrize("V", [32000, 128256])
@pytest.mark.parametrize("W", [1, 2, 4, 8])
def test_beam_select_matches_the_reference(V, W):
    logits, ip, sums, stops = _case(V, W, V + W)
    R = len(logits)
    lg = torch.from_numpy(logits).to(DEV)
    live, lk, fin, fk = (t.cpu().numpy() for t in ops.beam_select(lg, torch.from_numpy(ip).to(DEV), torch.from_numpy(sums).to(DEV),
                                                                 W, stops))
    # the sampler's own log-probabilities of each row's first 20 tokens: every candidate the step can return is among them
    n = ops.SAMPLE_TOP_N_MAX
    _, _, ids, lps = ops.sample_tokens(lg, [0.0] * R, [0] * R, [1.0] * R, [(0, r) for r in range(R)], [0] * R, logprobs=n)
    ids, lps = ids.cpu().numpy(), lps.cpu().numpy()
    lp_rows = [{int(t): lps[r, j] for j, t in enumerate(ids[r]) if t >= 0} for r in range(R)]
    exact = BR.beam_select_np(logits, ip, sums, W, stops, lp_rows=lp_rows)
    for got, want in zip((live, lk, fin, fk), exact):
        assert np.array_equal(got.view(np.int32), want.view(np.int32))
    # every key is fl32(sum + lp) with lp bit for bit the sampler's
    for sel, key in ((live, lk), (fin, fk)):
        for (r, t), k in zip(sel.reshape(-1, 2), key.reshape(-1)):
            if r >= 0:
                assert k == np.float32(sums[r] + lp_rows[r][int(t)])
    assert (live[:, :, 0] >= 0).sum() > 0 and (fin[:, :, 0] >= 0).sum() > 0
    # against the float64 reference: the same selections except at near-ties within its bound
    ref = BR.beam_select_np(logits, ip, sums, W, stops)
    near = 0
    for i in range(len(ip) - 1):
        for a, b in zip(map(tuple, np.concatenate([live[i], fin[i]])), map(tuple, np.concatenate([ref[0][i], ref[2][i]]))):
            if a != b:
                assert a[0] >= 0 and b[0] >= 0 and BR.near_tie(logits, sums, a, b), (i, a, b)
                near += 1
    print(f"V={V} W={W}: {near} near-tie differences from the float64 reference")


def test_beam_select_without_rows_pads_every_request():
    lg = torch.zeros((4, 1000), dtype=torch.float16, device=DEV)
    ip = torch.zeros(4, dtype=torch.int32, device=DEV)
    for t in ops.beam_select(lg[:0], ip, torch.zeros(4, device=DEV)[:0], 4, (3,)):
        assert (t.cpu() == -1).all()


def test_beam_select_rejects_bad_arguments():
    lg = torch.zeros((2, 100), dtype=torch.float16, device=DEV)
    ip = torch.tensor([0, 2], dtype=torch.int32, device=DEV)
    s = torch.zeros(2, dtype=torch.float32, device=DEV)
    for kw in (dict(width=0), dict(width=9), dict(width=2, stop_ids=(1, 1)), dict(width=2, stop_ids=(100,)),
               dict(width=2, stop_ids=tuple(range(9)))):
        with pytest.raises(RuntimeError):
            ops.beam_select(lg, ip, s, **kw)


def _pool(P):
    from atom_b200.kvcache import KvPoolInt4
    pool = KvPoolInt4(3, 2, 128, 10, P, DEV)
    g = torch.Generator(device=DEV).manual_seed(P)
    pool.buf.copy_(torch.randint(0, 256, pool.buf.shape, dtype=torch.uint8, device=DEV, generator=g))
    pool.param.copy_(torch.randn(pool.param.shape, device=DEV, generator=g).half())
    return pool


def _expect(before, pairs):
    buf, param = before
    buf, param = buf.clone(), param.clone()
    for s, d, n in pairs:
        if s >= 0:
            buf[d, :, :, :, :n] = buf[s, :, :, :, :n]
            param[d, :, :, :, :n] = param[s, :, :, :, :n]
    return buf, param


@pytest.mark.parametrize("P", [16, 32])
def test_copy_kv_pages_is_exact_and_leaves_the_rest(P):
    pool = _pool(P)
    pairs = [(1, 2, 1), (3, 4, P - 1), (5, 6, P)]
    before = (pool.buf.clone(), pool.param.clone())
    ops.copy_kv_pages(pool, *([p[k] for p in pairs] for k in range(3)))
    buf, param = _expect(before, pairs)
    assert torch.equal(pool.buf, buf) and torch.equal(pool.param.view(torch.int16), param.view(torch.int16))
    for bad in ([(1, 1, 1)], [(1, 2, 0)], [(1, 2, P + 1)], [(1, 10, 1)]):
        with pytest.raises(RuntimeError):
            ops.copy_kv_pages(pool, *([p[k] for p in bad] for k in range(3)))


def test_copy_kv_pages_replays_from_a_graph():
    P = 16
    pool = _pool(P)
    src, dst, slots = (torch.full((4,), -1, dtype=torch.int32, device=DEV) for _ in range(3))
    ops.copy_kv_pages(pool, src, dst, slots)                 # warm-up: all padding, a no-op
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.copy_kv_pages(pool, src, dst, slots)
    for pairs in ([(0, 1, 5), (2, 3, P), (-1, 0, 0), (-1, 0, 0)], [(7, 8, 1), (4, 9, P - 1), (5, 2, 3), (-1, 0, 0)]):
        before = (pool.buf.clone(), pool.param.clone())
        for k, t in enumerate((src, dst, slots)):
            t.copy_(torch.tensor([p[k] for p in pairs], dtype=torch.int32))
        g.replay()
        torch.cuda.synchronize()
        buf, param = _expect(before, pairs)
        assert torch.equal(pool.buf, buf) and torch.equal(pool.param.view(torch.int16), param.view(torch.int16))
