#!/usr/bin/env python
"""Speculative decoding, the verify attention: ops.batch_verify_i4 (S query tokens per sequence over the INT4 pages, one launch
for all S x G query rows of a KV head) against the alternatives on the same cache:
  * decode_1: one batch_decode_i4 launch (S = 1: the step a non-speculative decoder runs);
  * decode_S: S successive batch_decode_i4 launches (verifying S tokens one decode at a time);
  * prefill_ctx: prefill_attention_i4(kv=) over the same tails (its dequantisation launch and prefill_attn_kernel<true>).
Needs a GPU; there is no CPU path.

    python tools/spec_bench.py [--heads 32:32 32:8 64:8 8:1] [--batch 1 8 32] [--kv 1024 4096 32768] [--S 2 4 8] [--out r.json]
    python tools/spec_bench.py --step [--layers 8] [--ctx 1024] [--batch 1 8 32] [--S 2 4 8]   (the verify step's cost ratio r(S))

Method as tools/decode_attn_bench.py: every variant of a shape is captured into one CUDA graph holding one call per page-table
set; the sets live in distinct regions of a pool and together cover at least 256 MB, beyond the 50 MB L2, so every call streams
its pages from HBM.  Each shape is warmed up (eager call, then graph replays), the variants' graphs are replayed alternately and
timed with CUDA events, and the figure is the median replay divided by the calls it holds.  The card's name and power limit are
read in the same run and printed beside the numbers.
"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from atom_b200 import _lib, ops  # noqa: E402
from decode_attn_bench import L2_SWEEP_BYTES, _KV, build_sets, card, timed  # noqa: E402


def capture(fn, kvs, cycles):
    def run():
        for _ in range(cycles):
            for kv in kvs:
                fn(kv)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        run()
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            run()
    torch.cuda.current_stream().wait_stream(st)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    return g


def prefill_ctx_call(B, S, kv_len, hq, hkv, page, theta, dev, gen):
    """prefill_attention_i4(kv=) of B prompts of S tokens that are the tails of the B sequences, through the C ABI (the operator
    builds its position vector on the host, which a graph cannot capture)."""
    t = B * S
    k4 = torch.randint(0, 256, (t, hkv * 64), dtype=torch.uint8, device=dev, generator=gen)
    v4 = torch.randint(0, 256, (t, hkv * 64), dtype=torch.uint8, device=dev, generator=gen)
    par = torch.stack([torch.full((t, hkv), 0.03, device=dev), torch.full((t, hkv), 0.2, device=dev)], -1).half().reshape(t, hkv * 2)
    ip = torch.arange(0, t + 1, S, dtype=torch.int32, device=dev)
    pos = torch.arange(kv_len - S, kv_len, dtype=torch.int32, device=dev).repeat(B)
    rope = ops.rope_table(kv_len, dev, theta)
    kf = torch.empty((t, hkv * 128), dtype=torch.float16, device=dev)
    vf = torch.empty_like(kf)
    lib = _lib.lib()

    def fn(q, out, kv):
        _lib.check(lib.atom_prefill_attention_ctx_gqa_i4(
            q.data_ptr(), k4.data_ptr(), par.data_ptr(), v4.data_ptr(), par.data_ptr(), ip.data_ptr(), pos.data_ptr(), rope.data_ptr(),
            kf.data_ptr(), vf.data_ptr(), out.data_ptr(), t, B, S, hq, hkv, kv.data.data_ptr(), kv.param.data_ptr(),
            kv.indptr.data_ptr(), kv.indicies.data_ptr(), kv.last_page_offset.data_ptr(), 1, 0, page,
            torch.cuda.current_stream().cuda_stream), "prefill ctx")
    return fn, (k4, v4, par, ip, pos, rope, kf, vf)


def attention(args, dev, gen, name, limit):
    records = []
    for heads in args.heads:
        hq, hkv = (int(x) for x in heads.split(":"))
        for B in args.batch:
            for kv_len in args.kv:
                streamed = 136 * B * kv_len * hkv
                nsets = min(64, max(2, math.ceil(L2_SWEEP_BYTES / streamed)))
                cyc = max(1, 64 // nsets)
                data, param, tabs = build_sets(B, kv_len, hkv, args.page, nsets, dev, gen)
                kvs = [_KV(data, param, *t) for t in tabs]
                q1 = torch.randn((B, hq, 128), device=dev, dtype=torch.float16, generator=gen)
                g1 = capture(lambda kv: ops.batch_decode_i4(q1, kv, 0, rope_theta=args.theta), kvs, cyc)
                for S in args.S:
                    qs = torch.randn((B * S, hq, 128), device=dev, dtype=torch.float16, generator=gen)
                    os_ = torch.empty((B * S, hq * 128), device=dev, dtype=torch.float16)
                    pf, keep = prefill_ctx_call(B, S, kv_len, hq, hkv, args.page, args.theta, dev, gen)

                    def dec_s(kv):
                        for _ in range(S):
                            ops.batch_decode_i4(q1, kv, 0, rope_theta=args.theta)
                    graphs = {
                        "decode_1": g1,
                        "decode_S": capture(dec_s, kvs, cyc),
                        "verify": capture(lambda kv: ops.batch_verify_i4(qs, kv, 0, S, rope_theta=args.theta, max_len=kv_len), kvs, cyc),
                        "prefill_ctx": capture(lambda kv: pf(qs.view(B * S, hq * 128), os_, kv), kvs, cyc),
                    }
                    times = {k: [] for k in graphs}
                    for _ in range(args.reps):
                        for k, g in graphs.items():
                            times[k].append(timed(g) / (cyc * nsets))
                    rec = {"heads": heads, "batch": B, "kv": kv_len, "S": S, "page": args.page, "card": name, "power_limit": limit,
                           "verify_chunks": ops.verify_chunks(B, hkv, dev)}
                    for k in graphs:
                        rec[k + "_us"] = statistics.median(times[k]) * 1e6
                    rec["meets_bar"] = rec["verify_us"] < rec["decode_S_us"] and rec["verify_us"] < rec["prefill_ctx_us"]
                    records.append(rec)
                    print(json.dumps(rec), flush=True)
                    del graphs, keep
                del data, param, tabs, kvs, g1
                torch.cuda.empty_cache()
    print(f"\n{'heads':>6} {'B':>3} {'kv':>6} {'S':>2} | {'decode_1':>9} {'decode_S':>9} {'prefill':>9} {'verify':>9} us | "
          f"verify/decode_1")
    for r in records:
        print(f"{r['heads']:>6} {r['batch']:>3} {r['kv']:>6} {r['S']:>2} | {r['decode_1_us']:9.1f} {r['decode_S_us']:9.1f} "
              f"{r['prefill_ctx_us']:9.1f} {r['verify_us']:9.1f}    | {r['verify_us'] / r['decode_1_us']:6.2f}"
              f"{'' if r['meets_bar'] else '  (misses)'}")
    return records


def step_ratio(args, dev, name, limit):
    """r(S) = t(decode-only step carrying S tokens per sequence) / t(plain decode step), for a llama3-8b-shaped model of
    args.layers layers (hidden 4096, MLP 14336, 32:8 heads, base 5e5, vocab 128256, lm_head over every row) at contexts of
    args.ctx tokens.  Each step is captured into a CUDA graph; the graphs of one batch size are replayed alternately."""
    from atom_b200.cat_tensor import BatchLenInfo
    from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
    from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(hidden_size=4096, intermediate_size=14336, num_attention_heads=32, num_key_value_heads=8,
                      num_hidden_layers=args.layers, vocab_size=128256, rope_theta=5e5)
    torch.manual_seed(0)
    torch.set_default_dtype(torch.float16)
    try:
        with dev:
            model = LlamaForCausalLM(cfg)
    finally:
        torch.set_default_dtype(torch.float32)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    for layer in model.model.layers:
        layer.fuse()
    model.eval()
    P, smax = 32, max(args.S)
    records = []
    for B in args.batch:
        pool = KvPoolInt4(args.layers, 8, 128, B * (-(-(args.ctx + smax) // P)) + 4, P, dev)
        pool.buf.random_(0, 256)
        pool.param[..., 0].uniform_(0.01, 0.05)
        pool.param[..., 1].uniform_(0.0, 0.4)
        graphs = {}
        for S in [1] + list(args.S):
            seqs = [KvCacheInt4(pool, args.ctx + S) for _ in range(B)]
            kv = BatchedKvCacheInt4(seqs)
            blen = BatchLenInfo([], B, dev, decode_len=S)
            ids = torch.randint(0, 128256, (B * S,), device=dev)
            keep = (seqs, kv, blen, ids)
            run = lambda kv=kv, blen=blen, ids=ids: model(ids, blen, None, kv)
            st = torch.cuda.Stream()
            st.wait_stream(torch.cuda.current_stream())
            with torch.inference_mode(), torch.cuda.stream(st):
                run(); run()
                st.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=st):
                    run()
            torch.cuda.current_stream().wait_stream(st)
            for _ in range(3):
                g.replay()
            torch.cuda.synchronize()
            graphs[S] = (g, keep)
            for c in seqs:
                c.release()
        times = {S: [] for S in graphs}
        for _ in range(args.reps):
            for S, (g, _) in graphs.items():
                times[S].append(timed(g))
        t1 = statistics.median(times[1])
        for S in graphs:
            t = statistics.median(times[S])
            rec = {"step": "decode-only", "layers": args.layers, "batch": B, "ctx": args.ctx, "S": S, "step_us": t * 1e6,
                   "r": t / t1, "card": name, "power_limit": limit}
            records.append(rec)
            print(json.dumps(rec), flush=True)
        del graphs, pool
        torch.cuda.empty_cache()
    return records


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", nargs="+", default=["32:32", "32:8", "64:8", "8:1"])
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--kv", type=int, nargs="+", default=[1024, 4096, 32768])
    ap.add_argument("--S", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--page", type=int, default=32)
    ap.add_argument("--theta", type=float, default=1e4)
    ap.add_argument("--reps", type=int, default=9, help="alternating timed replays per variant")
    ap.add_argument("--step", action="store_true", help="measure r(S) of a multi-layer model step instead of the attention")
    ap.add_argument("--layers", type=int, default=8, help="--step: decoder layers")
    ap.add_argument("--ctx", type=int, default=1024, help="--step: tokens cached per sequence")
    ap.add_argument("--out", default=None, help="also write the records to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spec_bench: needs a CUDA device (the INT4 kernels have no CPU path)")
    dev = torch.device("cuda:0")
    name, limit = card()
    print(f"card: {name}, power limit {limit}, {torch.cuda.get_device_properties(dev).multi_processor_count} SMs")
    gen = torch.Generator(device=dev).manual_seed(0)
    records = step_ratio(args, dev, name, limit) if args.step else attention(args, dev, gen, name, limit)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
