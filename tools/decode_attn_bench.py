#!/usr/bin/env python
"""Decode attention over the INT4 paged KV cache: the grouped-query kernel against the multi-head kernel on a head-repeated
pool (what serving a GQA model without a GQA kernel would cost).  Needs a GPU; there is no CPU path.

    python tools/decode_attn_bench.py [--batch 32] [--kv 1024 4096] [--heads 64:8 32:8 8:1] [--page 32] [--out result.json]

Method: for every shape both variants are captured into one CUDA graph each, holding one launch per page-table set; the sets
live in distinct regions of a pool and together exceed the L2 cache several times, so every launch streams its pages from HBM.
Every shape is warmed up (eager launch, then graph replays), then the two graphs are replayed alternately and timed with CUDA
events; the figure is the median replay divided by the launches it holds.  Bytes are the algorithm's: 136 bytes per cached
token and KV head (64 B K + 64 B V + 2 x 4 B parameters) plus q and o.  The share of peak is taken against the H100 SXM data
sheet's 3.35 TB/s of HBM3 bandwidth -- a data-sheet figure, not a measured one.  The card's name and power limit are read in
the same run and printed beside the numbers.
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

DATASHEET_HBM_BYTES_PER_S = 3.35e12      # NVIDIA H100 SXM data sheet, HBM3
L2_SWEEP_BYTES = 256 << 20               # bytes all page-table sets of one variant cover together (H100 L2: 50 MB)


class _KV:
    def __init__(self, data, param, indptr, indices, last):
        self.data, self.param, self.indptr, self.indicies, self.last_page_offset = data, param, indptr, indices, last


def algorithmic_bytes(batch, kv_len, hq, hkv):
    """136 * sum(len) * Hkv + 4 * B * Hq * 128 (q read + o written, fp16)."""
    return 136 * batch * kv_len * hkv + 4 * batch * hq * 128


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                                   str(torch.cuda.current_device())], text=True).strip().splitlines()[0]
    name, limit = [s.strip() for s in out.split(",")]
    return name, limit


def build_sets(batch, kv_len, hkv, page, nsets, dev, gen):
    pps = (kv_len + page - 1) // page
    pages = nsets * batch * pps
    data = torch.randint(0, 256, (pages, 1, 2, hkv, page, 64), dtype=torch.uint8, device=dev, generator=gen)
    param = torch.empty((pages, 1, 2, hkv, page, 2), dtype=torch.float16, device=dev)
    param[..., 0].uniform_(0.01, 0.05, generator=gen)
    param[..., 1].uniform_(0.0, 0.4, generator=gen)
    perm = torch.randperm(pages, device=dev, generator=gen).to(torch.int32)
    indptr = torch.arange(0, (batch + 1) * pps, pps, dtype=torch.int32, device=dev)
    last = torch.full((batch,), (kv_len - 1) % page + 1, dtype=torch.int32, device=dev)
    tables = [(indptr, perm[s * batch * pps:(s + 1) * batch * pps].contiguous(), last) for s in range(nsets)]
    return data, param, tables


def capture(q, kvs, cycles):
    def run():
        out = None
        for _ in range(cycles):
            for kv in kvs:
                out = ops.batch_decode_i4(q, kv, 0)
        return out
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        first = ops.batch_decode_i4(q, kvs[0], 0).clone()          # warm-up of this shape: module load, smem attribute
        run()
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            run()
    torch.cuda.current_stream().wait_stream(st)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    return g, first


def timed(g):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); g.replay(); b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--kv", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--heads", nargs="+", default=["64:8", "32:8", "8:1"], help="query heads : KV heads")
    ap.add_argument("--page", type=int, default=32)
    ap.add_argument("--reps", type=int, default=15, help="alternating timed replays per variant")
    ap.add_argument("--out", default=None, help="also write the records to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_attn_bench: needs a CUDA device (the INT4 kernels have no CPU path)")
    dev = torch.device("cuda:0")
    name, limit = card()
    print(f"card: {name}, power limit {limit}; share of peak is against the data sheet's {DATASHEET_HBM_BYTES_PER_S / 1e12:.2f} TB/s (HBM3)")
    gen = torch.Generator(device=dev).manual_seed(0)
    records = []
    for hh in args.heads:
        hq, hkv = (int(x) for x in hh.split(":"))
        for kv_len in args.kv:
            B, P, G = args.batch, args.page, hq // hkv
            q = torch.randn((B, hq, 128), device=dev, dtype=torch.float16, generator=gen)
            rec = {"batch": B, "kv_len": kv_len, "q_heads": hq, "kv_heads": hkv, "page": P, "card": name, "power_limit": limit}
            # the two variants sweep the same number of bytes, so the repeated pool needs fewer sets
            n_gqa = min(64, max(2, math.ceil(L2_SWEEP_BYTES / (136 * B * kv_len * hkv))))
            n_mha = min(64, max(2, math.ceil(L2_SWEEP_BYTES / (136 * B * kv_len * hq))))
            data, param, tables = build_sets(B, kv_len, hkv, P, n_gqa, dev, gen)
            gqa_kvs = [_KV(data, param, *t) for t in tables]
            used = n_mha * B * ((kv_len + P - 1) // P)            # the repeated pool: the first n_mha sets' worth of pages
            rdata = data[:used].repeat_interleave(G, dim=3).contiguous()
            rparam = param[:used].repeat_interleave(G, dim=3).contiguous()
            pps = (kv_len + P - 1) // P
            rperm = torch.randperm(used, device=dev, generator=gen).to(torch.int32)
            mha_kvs = [_KV(rdata, rparam, tables[0][0], rperm[s * B * pps:(s + 1) * B * pps].contiguous(), tables[0][2]) for s in range(n_mha)]
            cyc_g, cyc_m = max(1, 64 // n_gqa), max(1, 64 // n_mha)
            g_gqa, o_gqa = capture(q, gqa_kvs, cyc_g)
            g_mha, o_mha = capture(q, mha_kvs, cyc_m)
            # same cache content for the two variants' first launches only if the page tables match: check on a shared table
            same = _KV(rdata, rparam, tables[0][0], tables[0][1] % used, tables[0][2])
            ref = ops.batch_decode_i4(q, same, 0)
            got = ops.batch_decode_i4(q, _KV(data, param, tables[0][0], tables[0][1] % used, tables[0][2]), 0)
            rec["max_abs_diff_gqa_vs_mha"] = float((got.float() - ref.float()).abs().max())
            t_g, t_m = [], []
            for _ in range(args.reps):
                t_g.append(timed(g_gqa) / (cyc_g * n_gqa))
                t_m.append(timed(g_mha) / (cyc_m * n_mha))
            for tag, ts, heads in (("gqa", t_g, hkv), ("mha_repeated", t_m, hq)):
                med = statistics.median(ts)
                by = algorithmic_bytes(B, kv_len, hq, heads)
                rec[tag] = {"us_per_launch": med * 1e6, "us_min": min(ts) * 1e6, "us_max": max(ts) * 1e6, "bytes": by,
                            "TB_per_s": by / med / 1e12, "share_of_datasheet_hbm": by / med / DATASHEET_HBM_BYTES_PER_S,
                            "ctas": B * heads, "launches_per_replay": (cyc_g * n_gqa) if tag == "gqa" else (cyc_m * n_mha)}
            rec["speedup_gqa_over_mha_repeated"] = rec["mha_repeated"]["us_per_launch"] / rec["gqa"]["us_per_launch"]
            records.append(rec)
            print(json.dumps(rec))
            del data, param, rdata, rparam, g_gqa, g_mha
            torch.cuda.empty_cache()
    print(f"\n{'Hq:Hkv':>7} {'kv':>5} | {'GQA us':>8} {'MB':>7} {'TB/s':>5} {'share':>6} | {'MHA-rep us':>10} {'MB':>7} {'TB/s':>5} {'share':>6} | speed-up")
    for r in records:
        a, b = r["gqa"], r["mha_repeated"]
        print(f"{r['q_heads']:>4}:{r['kv_heads']:<2} {r['kv_len']:>5} | {a['us_per_launch']:8.1f} {a['bytes'] / 1e6:7.1f} {a['TB_per_s']:5.2f} "
              f"{a['share_of_datasheet_hbm']:6.1%} | {b['us_per_launch']:10.1f} {b['bytes'] / 1e6:7.1f} {b['TB_per_s']:5.2f} "
              f"{b['share_of_datasheet_hbm']:6.1%} | {r['speedup_gqa_over_mha_repeated']:.2f}x")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
