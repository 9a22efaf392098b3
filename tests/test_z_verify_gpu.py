"""GPU suite (-m gpu) of the verify attention (verify_attn_kernel + verify_merge_kernel, ops.batch_verify_i4): element by element
inside tests/attn_verify_ref64.verify_bound over every group size, S in {1, 2, 3, 5, 8}, every page size the decode kernel
instantiates, batches of 1 to 64, contexts from S to 32k tokens, tails straddling page boundaries, layers > 0, dirty pools and
the `sink` regime, split and unsplit; and bit-for-bit determinism under other page placements, repeated calls and CUDA-graph
replays as lengths grow.  Fixed seeds, no retries."""
import numpy as np
import pytest
import torch

from tests import attn_verify_ref64 as V
from tests.attn_ctx_ref64 import make_ctx_case
from tests.test_z_attention_accuracy_gpu import DEV, T, _check

pytestmark = pytest.mark.gpu

PAGES = [8, 16, 24, 32, 64]


class _KV:
    def __init__(self, data, param, indptr, indices, last):
        self.data, self.param, self.indptr, self.indicies, self.last_page_offset = T(data), T(param), T(indptr), T(indices), T(last)


def _case(seed, ctxs, S, hq, hkv, P, regime="moderate", dirty=False, L=1, layer=0):
    rng = np.random.default_rng(seed)
    (q, *_), pool = make_ctx_case(rng, ctxs, [S] * len(ctxs), hq, hkv, P, regime=regime, dirty=dirty, L=L, layer=layer)
    return q.reshape(len(ctxs) * S, hq, 128), pool


def _verify(q, pool, layer, S, theta=1e4, nchunks=0):
    from atom_b200 import ops
    lens = [(pool[2][b + 1] - pool[2][b] - 1) * pool[0].shape[4] + pool[4][b] for b in range(len(pool[4]))]
    return ops.batch_verify_i4(T(q), _KV(*pool), layer, S, rope_theta=theta, max_len=max(lens), nchunks=nchunks).cpu().numpy()


def _run(q, pool, layer, S, hq, what, theta=1e4, nchunks=0):
    ref, bnd = V.verify_bound(q, *pool, layer, hq, theta, S)
    return _check(_verify(q, pool, layer, S, theta, nchunks), ref, bnd, what)


@pytest.mark.parametrize("nchunks", [1, 0, 5])
@pytest.mark.parametrize("S", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_every_group_and_token_count_within_bound(G, S, nchunks):
    P = PAGES[(G + S) % len(PAGES)]
    hkv = 2
    # contexts: none, a tail straddling a page boundary (ctx = P - 2), a few pages, several tiles
    ctxs = [0, P - 2, 3 * P + 1, 200 + S]
    q, pool = _case(10 * G + S, ctxs, S, G * hkv, hkv, P)
    _run(q, pool, 0, S, G * hkv, f"G={G} S={S} P={P} nchunks={nchunks}", nchunks=nchunks)


@pytest.mark.parametrize("P", PAGES)
def test_every_page_size_dirty_pool_later_layer_sink(P):
    S, G, hkv = 4, 4, 2
    q, pool = _case(100 + P, [5, P, 2 * P - 3, 300], S, G * hkv, hkv, P, regime="sink", dirty=True, L=3, layer=2)
    _run(q, pool, 2, S, G * hkv, f"P={P} dirty layer 2 sink", theta=5e5)
    _run(q, pool, 2, S, G * hkv, f"P={P} dirty layer 2 sink split", theta=5e5, nchunks=3)


def test_batch_of_64():
    S, G, hkv, P = 3, 2, 2, 16
    rng = np.random.default_rng(7)
    ctxs = [int(c) for c in rng.integers(0, 300, 64)]
    q, pool = _case(7, ctxs, S, G * hkv, hkv, P)
    _run(q, pool, 0, S, G * hkv, "B=64")


@pytest.mark.parametrize("ctx,G,hkv,regime", [(8192 - 5, 4, 2, "sink"), (32768 - 8, 8, 1, "moderate")])
def test_long_contexts_within_bound(ctx, G, hkv, regime):
    S = 8 if ctx % 2 == 0 else 5
    q, pool = _case(ctx, [ctx], S, G * hkv, hkv, 32, regime=regime)
    _run(q, pool, 0, S, G * hkv, f"ctx={ctx} G={G} auto split", theta=5e5)
    _run(q, pool, 0, S, G * hkv, f"ctx={ctx} G={G} unsplit", theta=5e5, nchunks=1)


@pytest.mark.parametrize("nchunks", [1, 4])
def test_bit_identical_under_other_placements_and_repeated_calls(nchunks):
    S, G, hkv, P = 5, 4, 2, 16
    ctxs = [3, 40, 100]
    q, pool = _case(21, ctxs, S, G * hkv, hkv, P, dirty=True)
    a = _verify(q, pool, 0, S, nchunks=nchunks)
    assert np.array_equal(a.view(np.uint16), _verify(q, pool, 0, S, nchunks=nchunks).view(np.uint16)), "repeated call differs"
    # the same sequences on another page order (make_pool shuffles with its rng)
    data, param, indptr, indices, last = pool
    perm = np.random.default_rng(5).permutation(data.shape[0])
    inv = np.argsort(perm)
    pool_p = (data[perm], param[perm], indptr, inv[indices].astype(np.int32), last)
    b = _verify(q, pool_p, 0, S, nchunks=nchunks)
    assert np.array_equal(a.view(np.uint16), b.view(np.uint16)), "the result depends on where the pages sit"


def test_graph_replay_equals_eager_as_lengths_grow():
    """One graph captured with a length bound replays over a page table rewritten in place: every replay equals the eager call on
    the same table bit for bit, as the sequences grow across page and tile boundaries."""
    from atom_b200 import ops
    S, G, hkv, P = 4, 2, 4, 16
    full = [150, 90]
    q, pool = _case(31, [n - S for n in full], S, G * hkv, hkv, P)
    data, param, indptr, indices, last = pool
    kv = _KV(*pool)
    qd = T(q)
    bound = max(full)

    def set_lens(lens):
        ip, lp = [0], []
        for b, n in enumerate(lens):
            pages = -(-n // P)
            ip.append(ip[-1] + pages)
            lp.append((n - 1) % P + 1)
        # sequence b keeps its own leading pages: the first `pages` entries of its page list
        idx = np.concatenate([indices[indptr[b]:indptr[b] + ip[b + 1] - ip[b]] for b in range(len(lens))])
        kv.indptr.copy_(T(np.array(ip, np.int32)))
        kv.indicies[:len(idx)].copy_(T(idx.astype(np.int32)))
        kv.last_page_offset.copy_(T(np.array(lp, np.int32)))

    steps = [[60, 30], [64, 33], [65, 48], [128, 49], [150, 90]]
    set_lens(steps[0])
    for nchunks in (1, 4):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ops.batch_verify_i4(qd, kv, 0, S, max_len=bound, nchunks=nchunks)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = ops.batch_verify_i4(qd, kv, 0, S, max_len=bound, nchunks=nchunks)
        for lens in steps:
            set_lens(lens)
            g.replay()
            eager = ops.batch_verify_i4(qd, kv, 0, S, max_len=bound, nchunks=nchunks)
            torch.cuda.synchronize()
            assert torch.equal(out.view(torch.int16), eager.view(torch.int16)), f"replay differs at lengths {lens} nchunks {nchunks}"


def test_rejects_bad_arguments():
    from atom_b200 import ops
    q, pool = _case(41, [10], 2, 4, 2, 16)
    with pytest.raises(RuntimeError):
        ops.batch_verify_i4(T(q), _KV(*pool), 0, 9, max_len=64)
    with pytest.raises(RuntimeError):
        ops.batch_verify_i4(T(q)[:1], _KV(*pool), 0, 2, max_len=64)
    with pytest.raises(RuntimeError):
        ops.batch_verify_i4(torch.from_numpy(q), _KV(*pool), 0, 2, max_len=64)


@pytest.mark.parametrize("nchunks", [1, 4])
def test_a_sequence_shorter_than_its_query_tokens_gets_zero_rows(nchunks):
    """A malformed page table (len_b < S) is not read: that sequence's rows are zeros, the others are unaffected."""
    S, G, hkv, P = 4, 2, 2, 16
    q, pool = _case(51, [20, 37], S, G * hkv, hkv, P)
    good = _verify(q, pool, 0, S, nchunks=nchunks)
    data, param, indptr, indices, last = pool
    short = (data, param, np.array([0, 1, indptr[2] - indptr[1] + 1], np.int32),
             np.concatenate([indices[:1], indices[indptr[1]:indptr[2]]]).astype(np.int32), np.array([2, last[1]], np.int32))
    from atom_b200 import ops
    got = ops.batch_verify_i4(T(q), _KV(*short), 0, S, max_len=64, nchunks=nchunks).cpu().numpy()
    assert not got[:S].any(), "rows of a sequence shorter than S must be zeros"
    assert np.array_equal(got[S:].view(np.uint16), good[S:].view(np.uint16))
