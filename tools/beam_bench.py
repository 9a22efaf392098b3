"""Device time per call of the beam step and the batched page copy, from CUDA-graph replays (DESIGN section 6).

beam_select at R = 1, 8, 32 and 64 rows (one request per W rows), W = 1, 4 and 8, V = 32000 and 128256, against the greedy
sample_tokens call on the same rows, a torch pipeline (log_softmax + topk + the merge's topk over each request's candidates) and
the lm_head GEMM of that shape (torch.matmul, [R, 4096] x [4096, V] in FP16).  copy_kv_pages: the bytes moved per second for the
copies of a llama3-8b-shaped step (32 layers, 8 KV heads, pages of 32 tokens).  Prints one JSON line."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from atom_b200 import ops
from atom_b200.kvcache import KvPoolInt4

DEV = torch.device("cuda:0")


def graph_us(fn, reps=200):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(10):
            fn()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * 10)


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": q.stdout.strip(), "beam_select": [], "copy_kv_pages": []}
    g = torch.Generator(device=DEV).manual_seed(0)
    for V in (32000, 128256):
        w_head = (torch.randn((4096, V), device=DEV, generator=g) * 0.02).half()
        for R in (1, 8, 32, 64):
            x = (torch.randn((R, 4096), device=DEV, generator=g)).half()
            logits = (torch.randn((R, V), device=DEV, generator=g) * 3).half()
            t0 = torch.zeros(R, dtype=torch.float32, device=DEV)
            k0 = torch.zeros(R, dtype=torch.int32, device=DEV)
            p1 = torch.ones(R, dtype=torch.float32, device=DEV)
            keys = torch.zeros((R, 2), dtype=torch.int64, device=DEV)
            ctr = torch.zeros(R, dtype=torch.int64, device=DEV)
            greedy = graph_us(lambda: ops.sample_tokens(logits, t0, k0, p1, keys, ctr))
            # the sampler's row passes one by one, at T = 0: the load and maximum (greedy), + the exact Z1 (logprobs=0),
            # + the radix select at K = n and its compaction (logprobs=n): the beam row's passes, like for like
            with_z1 = graph_us(lambda: ops.sample_tokens(logits, t0, k0, p1, keys, ctr, logprobs=0))
            head = graph_us(lambda: torch.matmul(x, w_head))
            for W in (1, 4, 8):
                if R < W:
                    continue
                B = -(-R // W)
                rip = torch.tensor([min(R, i * W) for i in range(B + 1)], dtype=torch.int32, device=DEV)
                sums = -torch.rand(R, device=DEV, generator=g) * 10
                bout = ops.beam_out(B, W, DEV)
                ws = torch.empty(R * 192, dtype=torch.uint8, device=DEV)
                beam = graph_us(lambda: ops.beam_select(logits, rip, sums, W, (2,), out=bout, workspace=ws))
                with_topn = graph_us(lambda: ops.sample_tokens(logits, t0, k0, p1, keys, ctr, logprobs=W))
                # no rows: the merge launch alone
                none = torch.zeros(B + 1, dtype=torch.int32, device=DEV)
                merge = graph_us(lambda: ops.beam_select(logits[:0], none, sums[:0], W, (2,), out=bout, workspace=ws))

                def torch_pipeline():
                    lp = torch.log_softmax(logits.float(), dim=-1) + sums[:, None]
                    v, i = torch.topk(lp, W, dim=-1)
                    return torch.topk(v.view(B, -1), W, dim=-1)
                tp = graph_us(torch_pipeline)
                out["beam_select"].append({"V": V, "R": R, "W": W, "beam_select_us": round(beam, 2), "greedy_sample_us": round(greedy, 2),
                                           "torch_pipeline_us": round(tp, 2), "lm_head_us": round(head, 2),
                                           "sample_load_z1_us": round(with_z1, 2), "sample_load_z1_topn_us": round(with_topn, 2),
                                           "merge_only_us": round(merge, 2),
                                           "beam_over_lm_head": round(beam / head, 4)})
        del w_head
    pool = KvPoolInt4(32, 8, 128, 256, 32, DEV)
    for n in (8, 24, 48):
        src = torch.arange(n, dtype=torch.int32, device=DEV)
        dst = src + 128
        slots = torch.full((n,), 16, dtype=torch.int32, device=DEV)
        us = graph_us(lambda: ops.copy_kv_pages(pool, src, dst, slots))
        nbytes = 2 * n * 16 * 32 * 2 * 8 * 68              # read + write of 16 slots per (layer, K|V, head) block
        out["copy_kv_pages"].append({"pairs": n, "slots": 16, "us": round(us, 2), "GB_per_s": round(nbytes / us / 1e3, 1)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
