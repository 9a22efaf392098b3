#!/usr/bin/env python
"""Prefill attention over a cached prefix (chunked prefill): one chunk of `chunk` new tokens attending to `ctx` cached tokens read
from the INT4 pages (prefill_attn_kernel<true>, plus the dequantisation of the chunk's own K/V), against the one-shot prefill of
all ctx + chunk tokens (prefill_attn_kernel<false>) that a scheduler without chunking would run instead.  Needs a GPU; there is no
CPU path.

    python tools/prefill_ctx_bench.py [--heads 32:8 64:8 32:32] [--ctx 0 4096 16384 32768] [--chunk 256 512 2048] [--page 32]
                                      [--theta 1e4] [--out result.json]

Method: one sequence per shape.  Each variant's C-ABI call (both of its launches) is captured into one CUDA graph, repeated
enough times to hold about a millisecond of work; every shape is warmed up (eager call, then two replays), then the graphs are
replayed alternately 11 times and timed with CUDA events, and the figure is the median replay divided by the calls it holds.
FLOPs are the algorithm's: 4 * chunk * (ctx + chunk / 2) * 128 * Hq (QK^T and PV over the causal half of the chunk and all of the
context); the one-shot variant is the same formula with ctx = 0 and chunk = ctx + chunk.  The share of peak is taken against the
H100 SXM data sheet's 989 TFLOP/s dense FP16 -- a data-sheet figure, not a measured one.  The card's name and power limit are
read in the same run and printed beside the numbers.
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
from atom_b200 import _lib, ops  # noqa: E402

DATASHEET_FP16_FLOPS = 989e12            # NVIDIA H100 SXM data sheet, dense FP16 / BF16 tensor core


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                                   str(torch.cuda.current_device())], text=True).strip().splitlines()[0]
    name, limit = [s.strip() for s in out.split(",")]
    return name, limit


def flops(ctx, chunk, hq):
    return 4.0 * chunk * (ctx + chunk / 2) * 128 * hq


def _inputs(t, hq, hkv, dev, gen):
    q = (torch.randn((t, hq * 128), device=dev, generator=gen) * 0.5).half()
    k4 = torch.randint(0, 256, (t, hkv * 64), dtype=torch.uint8, device=dev, generator=gen)
    v4 = torch.randint(0, 256, (t, hkv * 64), dtype=torch.uint8, device=dev, generator=gen)
    par = lambda: torch.stack([torch.empty((t, hkv), device=dev).uniform_(0.1, 1, generator=gen)] * 2, -1).mul_(
        torch.tensor([1.0, 7.5], device=dev)).half().reshape(t, hkv * 2).contiguous()
    return q, k4, par(), v4, par()


def chunk_call(ctx, chunk, hq, hkv, page, theta, dev, gen):
    """A closure running the chunk's prefill over a `ctx`-token cached prefix, and the tensors it keeps alive."""
    seq = ctx + chunk
    pages = (seq + page - 1) // page
    data = torch.randint(0, 256, (pages, 1, 2, hkv, page, 64), dtype=torch.uint8, device=dev, generator=gen)
    param = torch.empty((pages, 1, 2, hkv, page, 2), dtype=torch.float16, device=dev)
    param[..., 0].uniform_(0.1, 1.0, generator=gen)
    param[..., 1].copy_(param[..., 0] * 7.5)
    table = torch.tensor([0, pages, (seq - 1) % page + 1], dtype=torch.int32, device=dev)
    indices = torch.randperm(pages, device=dev, generator=gen).to(torch.int32)
    q, k4, kp, v4, vp = _inputs(chunk, hq, hkv, dev, gen)
    ip = torch.tensor([0, chunk], dtype=torch.int32, device=dev)
    pos = torch.arange(ctx, seq, dtype=torch.int32, device=dev)
    rope = ops.rope_table(seq, dev, theta)
    kf = torch.empty((chunk, hkv * 128), dtype=torch.float16, device=dev)
    vf, out = torch.empty_like(kf), torch.empty_like(q)
    keep = (data, param, table, indices, q, k4, kp, v4, vp, ip, pos, rope, kf, vf, out)
    lib = _lib.lib()

    def run():
        st = torch.cuda.current_stream().cuda_stream
        if ctx == 0:
            _lib.check(lib.atom_prefill_attention_gqa_i4(q.data_ptr(), k4.data_ptr(), kp.data_ptr(), v4.data_ptr(), vp.data_ptr(),
                                                         ip.data_ptr(), pos.data_ptr(), rope.data_ptr(), kf.data_ptr(), vf.data_ptr(),
                                                         out.data_ptr(), chunk, 1, chunk, hq, hkv, st), "prefill")
        else:
            _lib.check(lib.atom_prefill_attention_ctx_gqa_i4(
                q.data_ptr(), k4.data_ptr(), kp.data_ptr(), v4.data_ptr(), vp.data_ptr(), ip.data_ptr(), pos.data_ptr(), rope.data_ptr(),
                kf.data_ptr(), vf.data_ptr(), out.data_ptr(), chunk, 1, chunk, hq, hkv, data.data_ptr(), param.data_ptr(),
                table[:2].data_ptr(), indices.data_ptr(), table[2:].data_ptr(), 1, 0, page, st), "prefill ctx")
    return run, keep


def graph_of(run, reps):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(reps):
                run()
    torch.cuda.current_stream().wait_stream(s)
    return g


def time_graphs(graphs, replays=11):
    for g, _ in graphs:
        g.replay(); g.replay()
    torch.cuda.synchronize()
    times = [[] for _ in graphs]
    for _ in range(replays):
        for i, (g, reps) in enumerate(graphs):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); g.replay(); b.record()
            b.synchronize()
            times[i].append(a.elapsed_time(b) * 1e-3 / reps)
    return [statistics.median(t) for t in times]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--heads", nargs="+", default=["32:8", "64:8", "32:32"], help="Hq:Hkv pairs")
    ap.add_argument("--ctx", nargs="+", type=int, default=[0, 4096, 16384, 32768])
    ap.add_argument("--chunk", nargs="+", type=int, default=[256, 512, 2048])
    ap.add_argument("--page", type=int, default=32)
    ap.add_argument("--theta", type=float, default=1e4)
    ap.add_argument("--out", default=None, help="write the rows as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prefill_ctx_bench: needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, limit = card()
    print(f"# {name}, power limit {limit}; page {args.page}, RoPE base {args.theta:g}; peak = data sheet 989 TFLOP/s FP16")
    print(f"{'Hq:Hkv':>7} {'ctx':>6} {'chunk':>6} {'chunk us':>10} {'TFLOP/s':>8} {'% peak':>7} {'one-shot us':>12} {'TFLOP/s':>8} "
          f"{'% peak':>7}")
    gen = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for hs in args.heads:
        hq, hkv = (int(x) for x in hs.split(":"))
        for ctx in args.ctx:
            for chunk in args.chunk:
                fc, fo = flops(ctx, chunk, hq), flops(0, ctx + chunk, hq)
                run_c, keep_c = chunk_call(ctx, chunk, hq, hkv, args.page, args.theta, dev, gen)
                run_o, keep_o = chunk_call(0, ctx + chunk, hq, hkv, args.page, args.theta, dev, gen)
                reps = lambda f: max(1, min(200, math.ceil(1e-3 / (f / 3e14 + 5e-6))))
                graphs = [(graph_of(run_c, reps(fc)), reps(fc)), (graph_of(run_o, reps(fo)), reps(fo))]
                tc, to = time_graphs(graphs)
                row = dict(hq=hq, hkv=hkv, ctx=ctx, chunk=chunk, page=args.page, chunk_s=tc, chunk_flops=fc, one_shot_s=to,
                           one_shot_flops=fo, chunk_tflops=fc / tc / 1e12, one_shot_tflops=fo / to / 1e12,
                           chunk_peak_share=fc / tc / DATASHEET_FP16_FLOPS, one_shot_peak_share=fo / to / DATASHEET_FP16_FLOPS)
                rows.append(row)
                print(f"{hs:>7} {ctx:>6} {chunk:>6} {tc * 1e6:>10.1f} {row['chunk_tflops']:>8.1f} {100 * row['chunk_peak_share']:>6.1f}% "
                      f"{to * 1e6:>12.1f} {row['one_shot_tflops']:>8.1f} {100 * row['one_shot_peak_share']:>6.1f}%", flush=True)
                del graphs, keep_c, keep_o, run_c, run_o
                torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit": limit, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
