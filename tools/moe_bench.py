#!/usr/bin/env python
"""Device time of one Mixtral-8x7B sparse MoE block (hidden 4096, ffn 14336, 8 experts, top-2): the grouped path (route, plan,
gather, grouped gate/up+act, grouped down, combine) against a per-expert loop of the existing operators (index_select,
rmsnorm_fp16_i4, fused gate/up+act -- or gate, up, activate above 64 rows --, down, index_add_).  Needs a GPU.

    python tools/moe_bench.py [--tokens 1 8 32 64 512 2048] [--reps 50] [--out result.json]

Method: the loop needs every expert's token count on the host, so its routing is taken before capture (the grouped path routes
on the device).  Each variant is captured into a CUDA graph, warmed up, and the two graphs are replayed alternately, timed with
CUDA events; the figure is the median replay.  Bytes are those of the experts the routing touches (INT4 + INT8 weights and
their scales); their share is taken against the H100 SXM data sheet's 3.35 TB/s of HBM3 (decode sizes) and the share of the
FLOPs (2 * T * k * 3 * H * I) against its 1979 dense INT8 TOP/s (prefill sizes) -- data-sheet figures, not measured ones.
The card's name and power limit are read in the same run and printed beside the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from atom_b200 import ops  # noqa: E402
from atom_b200.llama import LlamaRMSNormInt4  # noqa: E402
from atom_b200.mixtral import MixtralConfig, SparseMoeInt4  # noqa: E402

DATASHEET_HBM_BYTES_PER_S = 3.35e12       # H100 SXM, HBM3
DATASHEET_INT8_OPS_PER_S = 1979e12        # H100 SXM, dense INT8 tensor core


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                                   str(torch.cuda.current_device())], text=True).strip().splitlines()[0]
    return [s.strip() for s in out.split(",")]


def expert_bytes(moe):
    per = 0
    for name in ("w13_int4", "w13_int8", "w13_scale", "w13_keeper_scale", "w2_int4", "w2_int8", "w2_scale", "w2_keeper_scale"):
        t = getattr(moe, name)
        per += t[0].numel() * t.element_size()
    return per


def loop_block(moe, hs, routing):
    """The per-expert loop over existing operators for a routing known on the host: [(expert, tok, slot, w)]."""
    n = moe.norm
    i = moe.intermediate_size
    out = torch.zeros_like(hs)
    for e, tok, slot, w in routing:
        x = ops.rmsnorm_fp16_i4(hs.index_select(0, tok), n.weight, n.reorder_index, n.variance_epsilon)
        w13 = moe._loop_ops[e]
        if tok.numel() <= 64:
            act = ops.dense_layer_gemm_i4_gateup_act(x[1], moe.w13_int4[e], x[3], moe.w13_scale[e], x[0], moe.w13_int8[e], x[2],
                                                     moe.w13_keeper_scale[e])
        else:
            gate = ops.dense_layer_gemm_i4_fp16(x[1], moe.w13_int4[e, :i], x[3], w13[0], x[0], moe.w13_int8[e, :i], x[2],
                                                moe.w13_keeper_scale[e, :i])
            up = ops.dense_layer_gemm_i4_fp16(x[1], moe.w13_int4[e, i:], x[3], w13[1], x[0], moe.w13_int8[e, i:], x[2],
                                              moe.w13_keeper_scale[e, i:])
            act = ops.activate_fp16_i4(gate, up)
        y = ops.dense_layer_gemm_i4_fp16(act[1], moe.w2_int4[e], act[3], moe.w2_scale[e], act[0], moe.w2_int8[e], act[2],
                                         moe.w2_keeper_scale[e])
        out.index_add_(0, tok, (y * w[:, None]).half())
    return out


def graph_of(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    return g


def time_pair(graphs, reps):
    times = [[] for _ in graphs]
    for g in graphs:
        for _ in range(5):
            g.replay()
    torch.cuda.synchronize()
    for _ in range(reps):
        for j, g in enumerate(graphs):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            g.replay()
            b.record()
            b.synchronize()
            times[j].append(a.elapsed_time(b) * 1e3)
    return [statistics.median(t) for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, nargs="+", default=[1, 8, 32, 64, 512, 2048])
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    cfg = MixtralConfig()
    h, inter, k = cfg.hidden_size, cfg.intermediate_size, cfg.num_experts_per_tok
    norm = LlamaRMSNormInt4(h, eps=cfg.rms_norm_eps).to(dev)
    moe = SparseMoeInt4(cfg, norm).to(dev).init_random(0)
    g = moe.w13_int4.shape[2] * 2 // 128
    moe._loop_ops = [(moe.w13_scale[e][:, :inter].contiguous(), moe.w13_scale[e][:, inter:].contiguous()) for e in range(cfg.num_local_experts)]
    per_expert = expert_bytes(moe)
    name, limit = card()
    print(f"# {name}, power limit {limit}; Mixtral-8x7B MoE block, hidden {h}, ffn {inter}, {cfg.num_local_experts} experts, top-{k}")
    print(f"{'T':>5} {'experts':>7} {'grouped us':>10} {'loop us':>9} {'speedup':>7} {'MB':>7} {'grouped share':>13}")
    rows = []
    gen = torch.Generator(device=dev).manual_seed(1)
    for t in a.tokens:
        hs = (torch.randn(t, h, device=dev, generator=gen) * 2).half()
        x = ops.rmsnorm_fp16_i4(hs, norm.weight, norm.reorder_index, norm.variance_epsilon)
        ids, w = moe.route(hs)
        routing = []
        for e in range(cfg.num_local_experts):
            tok, slot = torch.where(ids == e)
            if tok.numel():
                routing.append((e, tok, slot, w[tok, slot]))
        touched = len(routing)
        gg = graph_of(lambda: moe(hs, x))
        gl = graph_of(lambda: loop_block(moe, hs, routing))
        tg, tl = time_pair([gg, gl], a.reps)
        nbytes = touched * per_expert
        if t <= 64:
            share = f"{nbytes / (tg * 1e-6) / DATASHEET_HBM_BYTES_PER_S:.2f} of HBM"
        else:
            share = f"{2 * t * k * 3 * h * inter / (tg * 1e-6) / DATASHEET_INT8_OPS_PER_S:.2f} of INT8"
        print(f"{t:>5} {touched:>7} {tg:>10.1f} {tl:>9.1f} {tl / tg:>6.2f}x {nbytes / 1e6:>7.0f} {share:>13}")
        rows.append(dict(tokens=t, experts_touched=touched, grouped_us=tg, loop_us=tl, expert_bytes=nbytes, share=share))
        del gg, gl
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=name, power_limit=limit, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
