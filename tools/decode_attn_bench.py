#!/usr/bin/env python
"""Decode attention over the INT4 paged KV cache: the grouped-query kernel at each requested split-KV setting against the
multi-head kernel on a head-repeated pool (what serving a GQA model without a GQA kernel would cost).  Needs a GPU; there is no
CPU path.

    python tools/decode_attn_bench.py [--batch 32] [--kv 1024 4096] [--heads 64:8 32:8 8:1] [--page 32] [--theta 1e4]
                                      [--kv-split 0] [--no-mha] [--out result.json]

--batch takes several sizes (1 and 4 included); --kv-split takes several settings of the `kv_split` argument (0 = the automatic
rule, 1 = never split, 2 / 4 / 8 = forced), each a variant of its own, e.g. `--kv-split 1 0` for unsplit against automatic.
Method: for every shape each variant is captured into one CUDA graph, holding one launch per page-table set; the sets
live in distinct regions of a pool and together exceed the L2 cache several times, so every launch streams its pages from HBM.
Every shape is warmed up (eager launch, then graph replays), then the variants' graphs are replayed alternately and timed with CUDA
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


def capture(q, kvs, cycles, theta, kv_split=0):
    def run():
        out = None
        for _ in range(cycles):
            for kv in kvs:
                out = ops.batch_decode_i4(q, kv, 0, rope_theta=theta, kv_split=kv_split)
        return out
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        # warm-up of this shape: module load, smem attribute, cluster occupancy check
        first = ops.batch_decode_i4(q, kvs[0], 0, rope_theta=theta, kv_split=kv_split).clone()
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
    ap.add_argument("--batch", type=int, nargs="+", default=[32])
    ap.add_argument("--kv", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--heads", nargs="+", default=["64:8", "32:8", "8:1"], help="query heads : KV heads")
    ap.add_argument("--page", type=int, default=32)
    ap.add_argument("--theta", type=float, default=1e4, help="RoPE base passed to every call")
    ap.add_argument("--kv-split", type=int, nargs="+", default=[0], help="kv_split settings of the grouped-query variants")
    ap.add_argument("--no-mha", action="store_true", help="skip the multi-head kernel on the head-repeated pool")
    ap.add_argument("--reps", type=int, default=15, help="alternating timed replays per variant")
    ap.add_argument("--out", default=None, help="also write the records to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_attn_bench: needs a CUDA device (the INT4 kernels have no CPU path)")
    dev = torch.device("cuda:0")
    name, limit = card()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    print(f"card: {name}, power limit {limit}, {sms} SMs; share of peak is against the data sheet's "
          f"{DATASHEET_HBM_BYTES_PER_S / 1e12:.2f} TB/s (HBM3)")
    gen = torch.Generator(device=dev).manual_seed(0)
    records = []
    for hh in args.heads:
        hq, hkv = (int(x) for x in hh.split(":"))
        for B in args.batch:
            for kv_len in args.kv:
                P, G = args.page, hq // hkv
                q = torch.randn((B, hq, 128), device=dev, dtype=torch.float16, generator=gen)
                rec = {"batch": B, "kv_len": kv_len, "q_heads": hq, "kv_heads": hkv, "page": P, "rope_theta": args.theta,
                       "auto_kv_split": ops.decode_kv_split(B, hkv, G, dev), "card": name, "power_limit": limit}
                # the variants sweep the same number of bytes, so the repeated pool needs fewer sets
                n_gqa = min(64, max(2, math.ceil(L2_SWEEP_BYTES / (136 * B * kv_len * hkv))))
                n_mha = min(64, max(2, math.ceil(L2_SWEEP_BYTES / (136 * B * kv_len * hq))))
                data, param, tables = build_sets(B, kv_len, hkv, P, n_gqa, dev, gen)
                gqa_kvs = [_KV(data, param, *t) for t in tables]
                cyc_g, cyc_m = max(1, 64 // n_gqa), max(1, 64 // n_mha)
                variants = {}                        # tag -> (graph, first output, launches per replay, KV heads streamed)
                for sp in args.kv_split:
                    g, first = capture(q, gqa_kvs, cyc_g, args.theta, sp)
                    variants[f"gqa_split{sp}"] = (g, first, cyc_g * n_gqa, hkv)
                rdata = rparam = None
                if not args.no_mha:
                    used = n_mha * B * ((kv_len + P - 1) // P)        # the repeated pool: the first n_mha sets' worth of pages
                    rdata = data[:used].repeat_interleave(G, dim=3).contiguous()
                    rparam = param[:used].repeat_interleave(G, dim=3).contiguous()
                    pps = (kv_len + P - 1) // P
                    rperm = torch.randperm(used, device=dev, generator=gen).to(torch.int32)
                    mha_kvs = [_KV(rdata, rparam, tables[0][0], rperm[s * B * pps:(s + 1) * B * pps].contiguous(), tables[0][2])
                               for s in range(n_mha)]
                    g, first = capture(q, mha_kvs, cyc_m, args.theta)
                    variants["mha_repeated"] = (g, first, cyc_m * n_mha, hq)
                    # same cache content for both kernels only if the page tables match: check on a shared table
                    same = _KV(rdata, rparam, tables[0][0], tables[0][1] % used, tables[0][2])
                    ref = ops.batch_decode_i4(q, same, 0, rope_theta=args.theta)
                    got = ops.batch_decode_i4(q, _KV(data, param, tables[0][0], tables[0][1] % used, tables[0][2]), 0,
                                              rope_theta=args.theta)
                    rec["max_abs_diff_gqa_vs_mha"] = float((got.float() - ref.float()).abs().max())
                firsts = [v[1] for k, v in variants.items() if k.startswith("gqa")]
                rec["max_abs_diff_between_splits"] = max(float((f.float() - firsts[0].float()).abs().max()) for f in firsts)
                times = {k: [] for k in variants}
                for _ in range(args.reps):
                    for k, (g, _, launches, _) in variants.items():
                        times[k].append(timed(g) / launches)
                for k, (_, _, launches, heads) in variants.items():
                    ts = times[k]
                    med = statistics.median(ts)
                    by = algorithmic_bytes(B, kv_len, hq, heads)
                    rec[k] = {"us_per_launch": med * 1e6, "us_min": min(ts) * 1e6, "us_max": max(ts) * 1e6, "bytes": by,
                              "TB_per_s": by / med / 1e12, "share_of_datasheet_hbm": by / med / DATASHEET_HBM_BYTES_PER_S,
                              "ctas": B * heads, "launches_per_replay": launches}
                records.append(rec)
                print(json.dumps(rec))
                del data, param, rdata, rparam, variants, firsts
                torch.cuda.empty_cache()
    tags = [f"gqa_split{sp}" for sp in args.kv_split] + ([] if args.no_mha else ["mha_repeated"])
    print(f"\n{'Hq:Hkv':>7} {'B':>3} {'kv':>6} {'C':>2} | " + " | ".join(f"{t:>14} us  share" for t in tags))
    for r in records:
        print(f"{r['q_heads']:>4}:{r['kv_heads']:<2} {r['batch']:>3} {r['kv_len']:>6} {r['auto_kv_split']:>2} | "
              + " | ".join(f"{r[t]['us_per_launch']:17.1f} {r[t]['share_of_datasheet_hbm']:6.1%}" for t in tags))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
