#!/usr/bin/env python
"""Token sampling: ops.sample_tokens (atom_sample_f16) against torch.argmax and a torch pipeline with the same semantics (sort,
top-k mask, softmax at T, cumulative sum, top-p mask, inverse CDF in index order at the same uniforms), beside the FP16 lm_head
GEMM that produces the logits (hidden 4096).  Needs a GPU; there is no CPU path.

    python tools/sample_bench.py [--batch 1 16 32 64] [--vocab 32000 128256] [--out result.json]
    python tools/sample_bench.py --features [--batch 1 32 256] [--vocab 32000 128256]

--features times the plain call (T = 0.8, top-p 0.9) against the same call with each option of atom_sample_ex_f16 added, one
at a time and all together: +penalties (every row with a slot of a table holding prompt bits and counts), +min-p 0.05,
+logprobs with n = 0 and n = 20, and all of them; same method, all variants alternated in one run.

Method (that of tools/decode_attn_bench.py): for every shape each variant is captured into one CUDA graph holding one call per
logits set; the sets are distinct buffers that together cover at least 256 MB where that takes at most 256 sets (the H100's L2
holds 50 MB; the smallest shapes stay below that and are reported with their footprint).  Every shape is warmed up, then the
variants' graphs are replayed alternately and timed with CUDA events; the figure is the median replay divided by the calls it
holds.  Bytes are 2 * B * V (the logits read once); the share of peak is against the H100 SXM data sheet's 3.35 TB/s, a
data-sheet figure, not a measured one.  The card's name and power limit are read in the same run and printed beside the numbers.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from atom_b200 import ops  # noqa: E402

DATASHEET_HBM_BYTES_PER_S = 3.35e12
L2_SWEEP_BYTES = 256 << 20
SETTINGS = {"greedy": (0.0, 0, 1.0), "top-k 50": (0.8, 50, 1.0), "top-p 0.9": (0.8, 0, 0.9), "both": (0.8, 50, 0.9)}


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                                   str(torch.cuda.current_device())], text=True).strip().splitlines()[0]
    return [s.strip() for s in out.split(",")]


def torch_sample(l, T, k, p, u):
    """The sampler's semantics in torch ops: argmax at T = 0; else top-k on the sorted logits, softmax at T, the shortest prefix
    of mass >= p, and the first index (ascending) whose cumulative weight exceeds u * Z."""
    if T == 0:
        return torch.argmax(l, dim=-1)
    sv, si = torch.sort(l.float(), dim=-1, descending=True, stable=True)
    if k:
        sv[:, k:] = -math.inf
    probs = torch.softmax(sv / T, dim=-1)
    if p < 1:
        probs = probs.masked_fill(torch.cumsum(probs, -1) - probs >= p, 0.0)
    w = torch.zeros_like(probs).scatter_(1, si, probs)
    cdf = torch.cumsum(w, -1)
    return torch.searchsorted(cdf, (u * cdf[:, -1:]).contiguous(), right=True).squeeze(1)


def capture(fn, sets):
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for s in sets[:2]:
            fn(s)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for s in sets:
                fn(s)
    torch.cuda.current_stream().wait_stream(st)
    return g


def timed(g):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); g.replay(); b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3


FEATURES = {"plain": {}, "+penalties": {"pen": True}, "+min-p": {"min_p": 0.05}, "+logprobs n=0": {"logprobs": 0},
            "+logprobs n=20": {"logprobs": 20}, "all": {"pen": True, "min_p": 0.05, "logprobs": 20}}


def features(args, dev, name, limit):
    gen = torch.Generator(device=dev).manual_seed(1)
    rows = []
    for V in args.vocab:
        for B in args.batch:
            nbytes = 2 * B * V
            nsets = max(4, min(256, -(-L2_SWEEP_BYTES // nbytes)))
            sets = [(torch.randn((B, V), device=dev, generator=gen) * 4).half() for _ in range(nsets)]
            prm = [torch.full((B,), 0.8, dtype=torch.float32, device=dev), torch.zeros(B, dtype=torch.int32, device=dev),
                   torch.full((B,), 0.9, dtype=torch.float32, device=dev),
                   torch.stack([torch.zeros(B, dtype=torch.int64, device=dev), torch.arange(B, device=dev)], 1),
                   torch.arange(B, dtype=torch.int64, device=dev)]
            table = ops.penalty_table(B, V, dev)
            table[:, :V] = torch.where(torch.rand((B, V), device=dev, generator=gen) < 0.02, -0x8000, 0).short()
            table[:, :V] += torch.where(torch.rand((B, V), device=dev, generator=gen) < 0.01, 3, 0).short()
            full = lambda x: torch.full((B,), x, dtype=torch.float32, device=dev)     # noqa: E731
            pen = dict(repetition_penalty=full(1.2), frequency_penalty=full(0.3), presence_penalty=full(0.4), penalty_table=table,
                       slots=torch.arange(B, dtype=torch.int32, device=dev))

            def call(f):
                kw = dict(pen) if f.get("pen") else {}
                if "min_p" in f:
                    kw["min_p"] = full(f["min_p"])
                if "logprobs" in f:
                    kw["logprobs"] = f["logprobs"]
                return lambda l: ops.sample_tokens(l, *prm, **kw)
            variants = {t: capture(call(f), sets) for t, f in FEATURES.items()}
            for g in variants.values():
                for _ in range(3):
                    g.replay()
            torch.cuda.synchronize()
            ts = {t: [] for t in variants}
            for _ in range(args.reps):
                for t, g in variants.items():
                    ts[t].append(timed(g) / nsets)
            med = {t: statistics.median(v) for t, v in ts.items()}
            r = {"B": B, "V": V, "sets": nsets, **{f"{t}_us": round(m, 2) for t, m in med.items()}, "card": name, "power_limit": limit}
            rows.append(r)
            print(f"B={B:3d} V={V:6d} " + "  ".join(f"{t} {m:7.2f}" for t, m in med.items()) + " us", flush=True)
            del sets, table
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 16, 32, 64])
    ap.add_argument("--vocab", type=int, nargs="+", default=[32000, 128256])
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    ap.add_argument("--features", action="store_true", help="time each option of atom_sample_ex_f16 against the plain call")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, limit = card()
    print(f"card: {name}, power limit {limit}; share of peak against the data sheet's 3.35 TB/s")
    if args.features:
        rows = features(args, dev, name, limit)
        if args.out:
            with open(args.out, "w") as f:
                json.dump(rows, f, indent=1)
        print(json.dumps({"rows": len(rows), "card": name, "power_limit": limit}))
        return
    gen = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for V in args.vocab:
        wt = (torch.randn((V, args.hidden), device=dev, generator=gen) * 0.02).half()
        for B in args.batch:
            nbytes = 2 * B * V
            nsets = max(4, min(256, -(-L2_SWEEP_BYTES // nbytes)))
            sets = [(torch.randn((B, V), device=dev, generator=gen) * 4).half() for _ in range(nsets)]
            u = torch.rand((B, 1), device=dev, dtype=torch.float64, generator=gen).float()
            x = (torch.randn((B, args.hidden), device=dev, generator=gen)).half()
            head = capture(lambda _: torch.nn.functional.linear(x, wt), [None] * 4)
            for tag, (T, k, p) in SETTINGS.items():
                prm = [torch.full((B,), T, dtype=torch.float32, device=dev), torch.full((B,), k, dtype=torch.int32, device=dev),
                       torch.full((B,), p, dtype=torch.float32, device=dev),
                       torch.stack([torch.zeros(B, dtype=torch.int64, device=dev), torch.arange(B, device=dev)], 1),
                       torch.arange(B, dtype=torch.int64, device=dev)]
                variants = {"sample": (capture(lambda l: ops.sample_tokens(l, *prm), sets), nsets),
                            "argmax": (capture(lambda l: torch.argmax(l, dim=-1), sets), nsets),
                            "torch": (capture(lambda l: torch_sample(l, T, k, p, u), sets), nsets),
                            "lm_head": (head, 4)}
                for g, _ in variants.values():
                    for _ in range(3):
                        g.replay()
                torch.cuda.synchronize()
                ts = {t: [] for t in variants}
                for _ in range(args.reps):
                    for t, (g, n) in variants.items():
                        ts[t].append(timed(g) / n)
                med = {t: statistics.median(v) for t, v in ts.items()}
                r = {"B": B, "V": V, "setting": tag, "sets": nsets, "sets_MB": round(nsets * nbytes / 2 ** 20, 1),
                     **{f"{t}_us": round(m, 2) for t, m in med.items()},
                     "sample_share_of_peak": round(nbytes / DATASHEET_HBM_BYTES_PER_S * 1e6 / med["sample"], 3),
                     "sample_over_lm_head": round(med["sample"] / med["lm_head"], 4), "card": name, "power_limit": limit}
                rows.append(r)
                print(f"B={B:3d} V={V:6d} {tag:10s} sample {med['sample']:8.2f} us  argmax {med['argmax']:8.2f} us  torch "
                      f"{med['torch']:8.2f} us  | lm_head {med['lm_head']:8.2f} us  ({100 * r['sample_over_lm_head']:.1f} %)  "
                      f"sets {nsets} x {nbytes / 2 ** 20:.2f} MB", flush=True)
            del sets
        del wt
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)
    print(json.dumps({"rows": len(rows), "card": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
