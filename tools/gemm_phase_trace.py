"""Where the time of one W4A4 GEMM launch goes after griddepcontrol.wait, from the kernel's clock64 stamps (the slot layout is
documented at trace_stamp in atom_b200/csrc/gemm_i4_sm90.cuh).

python tools/gemm_phase_trace.py [--m 16 --n 4096 --k 4096] [--mhz MHZ] [--sets N] [--groups]

The launches run as bench.py runs them: one CUDA graph of back-to-back launches over operand sets larger than L2, with
programmatic dependent launch, warmed up first.  The stamps of the last launch are read back.  clock64 counts per SM, so
only differences inside one CTA are used; each phase is printed as median and max over the CTAs, in SM cycles and in us at
`--mhz` (default: the card's maximum SM clock).  A phase whose stamps the library does not write prints as "-".

--groups compiles a copy of the library with the per-group stamps (-DATOM_GEMM_TRACE_GROUPS) into a temporary directory
and also prints, per INT4 group, the median over the CTAs that own it of each per-group stamp after griddepcontrol.wait.
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from atom_b200 import _lib, ops, synth  # noqa: E402

L2_BYTES = 50e6
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRACE_GROUPS = 16        # gemm_i4_sm90.cuh: group s stamps slot 8 + kind * TRACE_GROUPS + s
GROUP_KINDS = ("prod pack_full", "prod slot free", "prod scales", "prod exp_full", "cons pack_full", "cons exp_full",
               "cons dequant")


def build_traced_lib(out_dir):
    """libatom_b200.so with the per-group stamps compiled in (the Makefile's flags + -DATOM_GEMM_TRACE_GROUPS)."""
    so = os.path.join(out_dir, "libatom_b200_trace.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler",
                           "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr", "-DATOM_GEMM_TRACE_GROUPS", "-shared",
                           "-o", so, os.path.join(ROOT, "atom_b200", "csrc", "atom_b200.cu"), "-lcudart"])
    return so


def max_sm_mhz():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.split()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def phases(tr):
    """Per-CTA phase durations (cycles) from one CTA's 128 stamps; None where a stamp is missing."""
    s = [int(x) for x in tr]

    def d(a, b):
        return b - a if a and b else None
    return {
        "setup (start -> barriers initialised)": d(s[0], s[1]),
        "griddepcontrol.wait (overlaps the previous launch)": d(s[1], s[5]),
        "wait -> INT4 groups and keeper done": d(s[5], s[2]),
        "tile staged + cluster barrier": d(s[2], s[3]),
        "split-K reduction + output stores": d(s[3], s[6]),
        "final cluster barrier": d(s[6], s[7]),
        "post-wait total (wait -> consumers leave)": d(s[5], s[7]),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--k", type=int, default=4096)
    ap.add_argument("--mhz", type=float, default=None, help="SM clock for the us column (default: nvidia-smi clocks.max.sm)")
    ap.add_argument("--sets", type=int, default=0, help="operand sets per graph (default: enough to exceed L2, as bench.py)")
    ap.add_argument("--groups", action="store_true", help="per-group stamps from a library built with -DATOM_GEMM_TRACE_GROUPS")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_phase_trace.py needs a CUDA device")
    if a.groups:
        _lib.LIB_PATH = build_traced_lib(tempfile.mkdtemp(prefix="atom_trace_"))
    dev = torch.device("cuda:0")
    one = synth.gemm_operands(a.m, a.n, a.k, dev, seed=1234)
    per_set = sum(t.numel() * t.element_size() for t in one)
    nsets = a.sets or int(2.4 * L2_BYTES // per_set) + 1
    sets = [one] + [tuple(t.clone() for t in one) for _ in range(nsets - 1)]
    # every CTA of the launch owns 128 slots: no grid exceeds the channel tiles x 16-token tiles x the 8-way split
    max_ctas = -(-a.n // 128) * -(-a.m // 16) * 8
    trace = torch.zeros((max_ctas, 128), dtype=torch.int64, device=dev)
    st = torch.cuda.Stream(dev)
    lib = _lib.lib()
    with torch.cuda.stream(st):
        for i in range(nsets):
            ops.dense_layer_gemm_i4_fp16(*sets[i])
        st.synchronize()
        lib.atom_gemm_set_trace(trace.data_ptr())        # read at launch: the captured launches carry the buffer
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g, stream=st):
                for i in range(nsets):
                    ops.dense_layer_gemm_i4_fp16(*sets[i])
        finally:
            lib.atom_gemm_set_trace(None)
        for _ in range(20):
            g.replay()
        trace.zero_()
        g.replay()
        st.synchronize()
    tr = trace.cpu().numpy()
    ctas = [c for c in range(tr.shape[0]) if tr[c, 0]]
    mhz = a.mhz or max_sm_mhz()
    rows = {}
    for c in ctas:
        for k, v in phases(tr[c]).items():
            rows.setdefault(k, []).append(v)
    print(f"gemm_i4_o16 M={a.m} N={a.n} K={a.k}: {len(ctas)} CTAs, "
          f"{nsets} operand sets per graph, {torch.cuda.get_device_name(dev)}, us at {mhz} MHz")
    print(f"{'phase':54s} {'median cyc':>10s} {'max cyc':>9s} {'median us':>10s} {'max us':>8s}")
    for k, vs in rows.items():
        v = [x for x in vs if x is not None]
        if not v:
            print(f"{k:54s} {'-':>10s} {'-':>9s} {'-':>10s} {'-':>8s}")
            continue
        med, mx = float(np.median(v)), float(np.max(v))
        us = (lambda c: f"{c / mhz:.2f}") if mhz else (lambda c: "-")
        print(f"{k:54s} {med:10.0f} {mx:9.0f} {us(med):>10s} {us(mx):>8s}")
    if a.groups:
        print("per INT4 group: cycles after griddepcontrol.wait, median over the CTAs that own the group")
        print("group " + " ".join(f"{k:>15s}" for k in GROUP_KINDS))
        for g in range(TRACE_GROUPS):
            own = [c for c in ctas if tr[c, 5] and tr[c, 8 + 6 * TRACE_GROUPS + g]]
            if not own:
                break
            cols = []
            for kind in range(len(GROUP_KINDS)):
                v = [tr[c, 8 + kind * TRACE_GROUPS + g] - tr[c, 5] for c in own if tr[c, 8 + kind * TRACE_GROUPS + g]]
                cols.append(f"{np.median(v):15.0f}" if v else f"{'-':>15s}")   # the resident variant writes fewer kinds
            print(f"{g:5d} " + " ".join(cols))


if __name__ == "__main__":
    main()
