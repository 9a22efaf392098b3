#!/usr/bin/env python
"""Shared-prefix decode: the cascade (ops.batch_decode_i4 on a batch with prefix groups) against unshared decode (the same
forked page tables read by the decode kernel, automatic split-KV) and against the automatic choice, whose pick
(ops.decode_cascade) should be the faster variant on each side of its threshold.  Needs a GPU; there is no CPU path.

    python tools/shared_prefix_bench.py [--page 32] [--quick] [--out result.json]

Workloads (`CASES`): heads 32:8, 64:8, 8:1 and 32:32; groups of 2 to 32 members; shared prefixes of 512 to 32k tokens; private
suffixes of 16 to 1k tokens; mixed batches of groups and lone sequences.  Method as tools/decode_attn_bench.py: every variant of a
shape is captured into one CUDA graph holding one launch per page-table set; the sets live in distinct regions of a pool and
together exceed the L2 cache several times, so every launch streams its pages from HBM.  Each shape is warmed up (eager launch,
then graph replays), the variants' graphs are replayed alternately and timed with CUDA events, and the figure is the median
replay divided by the launches it holds.  The card's name and power limit are read in the same run and printed beside the
numbers.
"""
import argparse
import json
import math
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from atom_b200 import ops  # noqa: E402
from decode_attn_bench import L2_SWEEP_BYTES, card, timed  # noqa: E402

# (heads, [(members, shared prefix tokens, private suffix tokens) per group], (lone rows, their length))
CASES = [
    ("32:8", [(32, 512, 128)], (0, 0)),
    ("32:8", [(32, 2048, 128)], (0, 0)),
    ("32:8", [(32, 8192, 128)], (0, 0)),
    ("32:8", [(32, 32768, 128)], (0, 0)),
    ("32:8", [(2, 2048, 256)] * 16, (0, 0)),
    ("32:8", [(4, 2048, 256)] * 8, (0, 0)),
    ("32:8", [(8, 2048, 256)] * 4, (0, 0)),
    ("32:8", [(16, 2048, 256)] * 2, (0, 0)),
    ("32:8", [(16, 4096, 16)], (0, 0)),
    ("32:8", [(16, 4096, 1024)], (0, 0)),
    ("32:8", [(2, 512, 64)], (0, 0)),
    ("32:8", [(2, 4096, 64)], (0, 0)),
    ("32:8", [(2, 8192, 64)], (0, 0)),
    ("32:8", [(4, 512, 512)], (2, 512)),
    ("32:8", [(4, 2048, 64)] * 4, (16, 2048)),
    ("32:8", [(8, 1024, 128)] * 2, (16, 4096)),
    ("64:8", [(32, 4096, 128)], (0, 0)),
    ("64:8", [(2, 512, 512)] * 16, (0, 0)),
    ("64:8", [(8, 8192, 256)] * 4, (0, 0)),
    ("8:1", [(32, 8192, 128)], (0, 0)),
    ("8:1", [(4, 2048, 64)] * 2, (8, 1024)),
    ("32:32", [(8, 2048, 128)], (0, 0)),
    ("32:32", [(2, 512, 1024)] * 4, (0, 0)),
    ("32:32", [(32, 4096, 64)], (0, 0)),
]


class _KV:
    def __init__(self, data, param, t, groups=None):
        self.data, self.param = data, param
        self.indptr, self.last_page_offset, self.indicies = t["indptr"], t["last"], t["indices"]
        if groups is not None:
            self.groups = groups
            self.group_indptr, self.group_members, self.shared_pages = t["gindptr"], t["gmembers"], t["shared"]


def layout(groups, lone, P):
    """Rows (group members first, then lone rows) and the pages each needs, with prefix pages shared inside a group."""
    rows, gl, r = [], [], 0
    for m, pre, suf in groups:
        gl.append((list(range(r, r + m)), pre // P))
        rows += [(pre, suf)] * m
        r += m
    rows += [(0, lone[1])] * lone[0]
    pages = sum(pre // P + m * -(-suf // P) for m, pre, suf in groups) + lone[0] * -(-lone[1] // P)
    return rows, gl, pages


def tables(groups, lone, P, ids, dev):
    """One page-table set on the pages `ids` (host ints), in the layout BatchedKvCacheInt4 builds."""
    it = iter(ids)
    indptr, indices, last, members, shared = [0], [], [], [], []
    for m, pre, suf in groups:
        common = [next(it) for _ in range(pre // P)]
        for _ in range(m):
            own = [next(it) for _ in range(-(-suf // P))]
            indices += common + own
            indptr.append(len(indices))
            last.append((pre + suf - 1) % P + 1)
            members.append(len(indptr) - 2)
            shared.append(pre // P)
    for _ in range(lone[0]):
        indices += [next(it) for _ in range(-(-lone[1] // P))]
        indptr.append(len(indices))
        last.append((lone[1] - 1) % P + 1)
        shared.append(0)
    gind = np.cumsum([0] + [m for m, _, _ in groups])
    T = lambda a: torch.tensor(np.asarray(a, dtype=np.int32), device=dev)
    return dict(indptr=T(indptr), indices=T(indices), last=T(last), gindptr=T(gind), gmembers=T(members), shared=T(shared))


def capture(fn, kvs, cycles):
    def run():
        out = None
        for _ in range(cycles):
            for kv in kvs:
                out = fn(kv)
        return out
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        first = fn(kvs[0]).clone()
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--page", type=int, default=32)
    ap.add_argument("--theta", type=float, default=5e5)
    ap.add_argument("--reps", type=int, default=15, help="alternating timed replays per variant")
    ap.add_argument("--quick", action="store_true", help="every third case only")
    ap.add_argument("--out", default=None, help="also write the records to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("shared_prefix_bench: needs a CUDA device (the INT4 kernels have no CPU path)")
    dev = torch.device("cuda:0")
    name, limit = card()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    print(f"card: {name}, power limit {limit}, {sms} SMs")
    gen = torch.Generator(device=dev).manual_seed(0)
    rng = np.random.default_rng(0)
    P = args.page
    records = []
    for heads, groups, lone in (CASES[::3] if args.quick else CASES):
        hq, hkv = (int(x) for x in heads.split(":"))
        rows, gl, pps = layout(groups, lone, P)
        B = len(rows)
        streamed = 136 * P * hkv * pps                           # bytes the cascade streams per launch (once per shared page)
        nsets = min(64, max(2, math.ceil(L2_SWEEP_BYTES / streamed)))
        data = torch.randint(0, 256, (nsets * pps, 1, 2, hkv, P, 64), dtype=torch.uint8, device=dev, generator=gen)
        param = torch.empty((nsets * pps, 1, 2, hkv, P, 2), dtype=torch.float16, device=dev)
        param[..., 0].uniform_(0.01, 0.05, generator=gen)
        param[..., 1].uniform_(0.0, 0.4, generator=gen)
        perm = rng.permutation(nsets * pps)
        sets = [tables(groups, lone, P, perm[s * pps:(s + 1) * pps].tolist(), dev) for s in range(nsets)]
        q = torch.randn((B, hq, 128), device=dev, dtype=torch.float16, generator=gen)
        shared_kvs = [_KV(data, param, t, gl) for t in sets]
        plain_kvs = [_KV(data, param, t) for t in sets]
        cyc = max(1, 64 // nsets)
        cascade = lambda kv: ops._batch_decode_shared(torch.empty_like(q), q, kv, kv.groups, 1, hkv, P, 0, args.theta, sms)
        variants = {
            "cascade": capture(cascade, shared_kvs, cyc),
            "unshared": capture(lambda kv: ops.batch_decode_i4(q, kv, 0, rope_theta=args.theta), plain_kvs, cyc),
            "auto": capture(lambda kv: ops.batch_decode_i4(q, kv, 0, rope_theta=args.theta), shared_kvs, cyc),
        }
        pick = ops.decode_cascade(gl, B, P, hkv, hq // hkv, sms)
        rec = {"heads": heads, "groups": [list(g) for g in groups], "lone": list(lone), "batch": B, "page": P,
               "rule_picks_cascade": pick, "card": name, "power_limit": limit,
               "max_abs_diff_cascade_vs_unshared": float((variants["cascade"][1].float() - variants["unshared"][1].float()).abs().max()),
               "auto_is_pick_bitwise": bool(torch.equal(variants["auto"][1], variants["cascade" if pick else "unshared"][1]))}
        times = {k: [] for k in variants}
        for _ in range(args.reps):
            for k, (g, _) in variants.items():
                times[k].append(timed(g) / (cyc * nsets))
        for k in variants:
            rec[k + "_us"] = statistics.median(times[k]) * 1e6
        rec["speedup"] = rec["unshared_us"] / rec["cascade_us"]
        rec["pick_is_faster"] = (rec["cascade_us"] < rec["unshared_us"]) == pick
        records.append(rec)
        print(json.dumps(rec), flush=True)
        del data, param, sets, shared_kvs, plain_kvs, variants
        torch.cuda.empty_cache()
    print(f"\n{'heads':>6} {'B':>3} {'groups (members x prefix + suffix)':>40} {'lone':>9} | {'cascade':>8} {'unshared':>8} "
          f"{'auto':>8} us | speed-up  pick")
    for r in records:
        gs = ", ".join(f"{m}x{p}+{s}" for m, p, s in r["groups"][:2]) + (f" (x{len(r['groups'])})" if len(r["groups"]) > 2 else "")
        lone = f"{r['lone'][0]}x{r['lone'][1]}" if r["lone"][0] else "-"
        print(f"{r['heads']:>6} {r['batch']:>3} {gs:>40} {lone:>9} | {r['cascade_us']:8.1f} {r['unshared_us']:8.1f} {r['auto_us']:8.1f}"
              f"    | {r['speedup']:7.2f}x  {'cascade' if r['rule_picks_cascade'] else 'unshared'}"
              f"{'' if r['pick_is_faster'] else '  (slower pick)'}")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
