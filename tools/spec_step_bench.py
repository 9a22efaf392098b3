#!/usr/bin/env python
"""Per-step cost of speculative decoding's own launches on the device: the draft sampler (ops.sample_tokens with drafts) against
the plain sampler over the same B * S rows, and ops.spec_commit_propose over B token histories of a given length.  CUDA events
around replays of a graph of the launches, so the ops' host-side work is not timed; prints one JSON line per point.  Needs a GPU.

    python tools/spec_step_bench.py --vocab 128256 --batch 1 8 32 --tokens 1 5 8
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from atom_b200 import ops  # noqa: E402


def _time(fn, iters, per_graph=20):
    """Device time of one fn() in microseconds: `per_graph` calls captured in one CUDA graph, replayed (host overheads of the
    Python op wrappers are not timed)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(per_graph):
                fn()
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = max(1, iters // per_graph)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * per_graph)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocab", type=int, nargs="+", default=[32000, 128256])
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--tokens", type=int, nargs="+", default=[1, 5, 8], help="rows per sequence (S)")
    ap.add_argument("--history", type=int, default=1024, help="tokens in each history slot")
    ap.add_argument("--iters", type=int, default=400)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    print(json.dumps({"device": torch.cuda.get_device_name(dev)}))
    for V in args.vocab:
        for B in args.batch:
            for S in args.tokens:
                R = B * S
                x = (torch.randn((R, V), device=dev) * 2.5).half()
                keys = torch.tensor([[1, i] for i in range(R)], dtype=torch.int64, device=dev)
                ctr = torch.arange(R, dtype=torch.int64, device=dev)
                d = torch.from_numpy(rng.integers(-1, V, R).astype(np.int32)).to(dev)
                for T in (0.0, 0.8):
                    t = torch.full((R,), T, device=dev)
                    k = torch.zeros(R, dtype=torch.int32, device=dev)
                    p = torch.ones(R, device=dev)
                    plain = _time(lambda: ops.sample_tokens(x, t, k, p, keys, ctr), args.iters)
                    draft = _time(lambda: ops.sample_tokens(x, t, k, p, keys, ctr, drafts=d), args.iters)
                    print(json.dumps({"op": "sample", "vocab": V, "batch": B, "S": S, "T": T, "plain_us": round(plain, 2),
                                      "draft_us": round(draft, 2)}))
    for B in args.batch:
        for K in (4, 7):
            S = K + 1
            hist, lens = ops.spec_history(B, args.history + 64, dev)
            hist[:, :args.history] = torch.from_numpy(rng.integers(0, 50, (B, args.history)).astype(np.int32)).to(dev)
            tok = torch.from_numpy(rng.integers(0, 50, B * S).astype(np.int32)).to(dev)
            cand = torch.full((B * S,), -1, dtype=torch.int32, device=dev)
            rows = torch.arange(0, B * S + 1, S, dtype=torch.int32, device=dev)
            slots = torch.arange(B, dtype=torch.int32, device=dev)
            out = torch.empty((B, 2 * K + 3), dtype=torch.int32, device=dev)

            def step():
                lens.fill_(args.history)
                ops.spec_commit_propose(tok, cand, rows, slots, hist, lens, out, K, 1, 3)
            fill = _time(lambda: lens.fill_(args.history), args.iters)
            print(json.dumps({"op": "commit_propose", "batch": B, "num_draft": K, "history": args.history,
                              "us": round(_time(step, args.iters) - fill, 2)}))


if __name__ == "__main__":
    main()
