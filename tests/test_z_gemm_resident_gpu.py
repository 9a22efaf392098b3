"""The resident-slice decode GEMM (-m gpu): gemm_i4_kernel<16, split, EPI_O16 | EPI_RESIDENT>, which gemm_dispatch picks for
16-token tiles split over K when every rank holds at most PACK = 8 INT4 groups.  Each rank loads all its token tiles and
scales in one burst after griddepcontrol.wait and pushes its split-K partials to the ranks that store them.

Every case is held bit for bit against the split-aware oracle (`ksplit`) and within the float64 bound of tests/gemm_ref64.py:
M over the 8-row halves of the scale layout, K with empty, uneven and keeper-only ranks, N with channel tails.  A chain in one
CUDA graph in which the quantiser writes the activations and token scales right before each GEMM (programmatic dependent
launch on) must equal eager launches with a synchronise between them, and a graph over rotating operand sets must replay bit
for bit."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import gemm_ref64 as R

pytestmark = pytest.mark.gpu

SPLIT_FLAG = {2: 16, 4: 32, 8: 64}                # GEMM_SPLITK2, GEMM_SPLITK4, GEMM_SPLITK8
PACK = 8                                          # GemmCfg<16, ...>::PACK: INT4 groups a resident rank may hold
MS = (1, 7, 8, 9, 15, 16)
KS = (256, 512, 1152, 4096)
NS = (8, 120, 4096, 8448)


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _resident(k, split):
    return -(-(k // 128) // split) <= PACK


def _check(t, flags, split, what):
    from atom_b200 import ops
    m, n, k = t[0].shape[0], t[1].shape[0], t[0].shape[1] * 2 + 128
    got = ops.dense_layer_gemm_i4_fp16(*[T(x) for x in t], flags=flags).cpu().numpy()
    rows = None if m * n * k <= 1 << 28 else sorted({0, m - 1, m // 2})
    if rows is not None:
        got = got[rows]
    ref = O.gemm_i4_o16(*t, rows=rows, ksplit=split)
    bad = np.argwhere(got.view(np.uint16) != ref.view(np.uint16))
    assert len(bad) == 0, f"{what}: {len(bad)} outputs differ from the oracle, first at {tuple(bad[0])}"
    S, Tabs = R.ref64(*t, rows=rows)
    R.check_o16(got, S, Tabs, k // 128 - 1, split, what)


@pytest.mark.parametrize("k,split", [(k, s) for k in KS for s in (2, 4, 8) if _resident(k, s)])
def test_resident_against_oracle(k, split):
    for i, m in enumerate(MS):
        assert R.dispatch(m, 8, k, SPLIT_FLAG[split]) == (16, split)
        n = NS[(i + KS.index(k)) % len(NS)]
        regime = R.REGIMES[i % len(R.REGIMES)]
        _check(R.operands(regime, m, n, k, seed=10 * m + split), SPLIT_FLAG[split], split, f"{regime} {m}x{n}x{k} split {split}")


@pytest.mark.parametrize("n", NS)
def test_resident_every_n(n):
    """The automatic rule: K = 4096 splits 4-way (8 groups per rank), K = 1152 2-way (5 groups)."""
    for m, k in ((16, 4096), (9, 1152), (1, 4096)):
        split = R.dispatch(m, n, k)[1]
        assert split > 1 and _resident(k, split)
        _check(R.operands("random", m, n, k, seed=n + m), 0, split, f"auto {m}x{n}x{k} split {split}")


def _chain(graph, steps=6, k=1024):
    """x -> (reorder+quantise -> resident GEMM, split 4) x steps: each GEMM reads what the quantiser just wrote."""
    from atom_b200 import ops, synth
    dev = torch.device("cuda:0")
    w = synth.gemm_operands(16, k, k, dev, seed=7)
    idx = torch.randperm(k, generator=torch.Generator().manual_seed(0)).to(torch.int16).to(dev)
    x0 = torch.randn(16, k, generator=torch.Generator().manual_seed(1)).half().to(dev)

    def run(x, sync):
        for _ in range(steps):
            o8, o4, s8, s4 = ops.reorder_fp16_i4(x, idx)
            if sync:
                torch.cuda.synchronize()
            x = ops.dense_layer_gemm_i4_fp16(o4.view(torch.uint8), w[1], s4, w[3], o8, w[5], s8, w[7], flags=SPLIT_FLAG[4])
            if sync:
                torch.cuda.synchronize()
            x = x / x.float().abs().amax().clamp(min=1e-3).half()
        return x
    if not graph:
        return run(x0, True).clone()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        run(x0, False)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            y = run(x0, False)
        outs = []
        for _ in range(3):
            g.replay()
            outs.append(y.clone())
        st.synchronize()
    return outs


@pytest.mark.timeout(300)
def test_resident_pdl_chain_graph_matches_eager():
    from atom_b200 import _lib
    lib = _lib.lib()
    torch.cuda.synchronize()
    ref = _chain(graph=False)
    assert torch.isfinite(ref).all()
    _lib.check(lib.atom_set_pdl(1), "atom_set_pdl")
    try:
        for y in _chain(graph=True):
            assert torch.equal(y, ref)
    finally:
        torch.cuda.synchronize()
        _lib.check(lib.atom_set_pdl(0), "atom_set_pdl")


def test_resident_graph_over_rotating_sets():
    from atom_b200 import ops, synth
    dev = torch.device("cuda:0")
    sets = [synth.gemm_operands(16, 4096, 4096, dev, seed=50 + i) for i in range(6)]
    ref = [ops.dense_layer_gemm_i4_fp16(*s).clone() for s in sets]
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            outs = [ops.dense_layer_gemm_i4_fp16(*s) for s in sets]
        for _ in range(5):
            g.replay()
            st.synchronize()
            for o, r in zip(outs, ref):
                assert torch.equal(o, r)
