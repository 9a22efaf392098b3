#!/usr/bin/env python
"""CLI of the continuous-batching harness: the reference's `python -m benchmarks.bench_textgen --system punica`
(e2e/punica-atom/benchmarks/bench_textgen.py:488-528) on the H100 kernels.  Same flags, same request set, same report
lines, plus one JSON line.  Random INT4 weights of the named architecture (the reference's e2e run does the same,
e2e/README.md), synthetic token ids.  Needs a GPU; there is no CPU path.

    python tools/bench_textgen.py --model 7b --batch-size 16 --num-batches 2 --maxlen 512
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from atom_b200 import textgen as tg  # noqa: E402
from atom_b200.kvcache import KvPoolInt4  # noqa: E402
from atom_b200.llama import LinearInt4, LlamaConfig, LlamaForCausalLM  # noqa: E402


def build_model(mc: tg.ModelConfig, layers: int):
    device = torch.device(mc.device)
    default = torch.get_default_dtype()
    torch.set_default_dtype(getattr(torch, mc.dtype))
    try:
        with device:
            model = LlamaForCausalLM(LlamaConfig(hidden_size=mc.hidden_size, num_attention_heads=mc.num_heads,
                                                 intermediate_size=mc.intermediate_size, num_hidden_layers=layers,
                                                 num_key_value_heads=mc.num_kv_heads, rope_theta=mc.rope_theta))
    finally:
        torch.set_default_dtype(default)
    model = model.to(device)
    for i, m in enumerate(mod for mod in model.modules() if isinstance(mod, LinearInt4)):
        m.init_random(i)
    return model.eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=tg.MODEL_CFGS.keys(), default="7b")
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--num-batches", type=int, default=10)
    ap.add_argument("--maxlen", type=int, default=2048)
    ap.add_argument("--dtype", choices=["float16"], default="float16")
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--layers", type=int, default=0, help="override the number of decoder layers (0 = the model's)")
    ap.add_argument("--block-len", type=int, default=32)
    ap.add_argument("--no-cuda-graphs", action="store_true", help="run decode-only steps eagerly too (the reference's way)")
    ap.add_argument("--prefill-chunk", type=int, default=None,
                    help="chunked prefill: at most this many prompt tokens per step (default: whole prompts)")
    ap.add_argument("--shared-prefix", type=int, default=0, metavar="N",
                    help="precede every prompt with one common N-token system prompt, prefilled once and shared by forking")
    ap.add_argument("--temperature", type=float, default=None,
                    help="sample at this temperature on the device (ops.sample_tokens); default: greedy (argmax)")
    ap.add_argument("--top-k", type=int, default=0, help="with sampling: keep the k largest logits (0 = off)")
    ap.add_argument("--top-p", type=float, default=1.0, help="with sampling: keep the smallest set of mass >= p (1 = off)")
    ap.add_argument("--seed", type=int, default=0, help="with sampling: request r draws from the Philox key (seed, r)")
    ap.add_argument("--min-p", type=float, default=0.0, help="with sampling: drop tokens below m times the top one's weight (0 = off)")
    ap.add_argument("--repetition-penalty", type=float, default=1.0, help="with sampling: on prompt and generated tokens (1 = off)")
    ap.add_argument("--frequency-penalty", type=float, default=0.0, help="with sampling: times a token's count (0 = off)")
    ap.add_argument("--presence-penalty", type=float, default=0.0, help="with sampling: on generated tokens (0 = off)")
    ap.add_argument("--logprobs", type=int, default=None, metavar="N",
                    help="with sampling: each token's log-probability and the top N (0 to 20)")
    ap.add_argument("--stop-token", type=int, action="append", default=[], metavar="ID",
                    help="a request that emits this id finishes on it (repeatable)")
    ap.add_argument("--speculate", type=int, default=0, metavar="K",
                    help="speculative decoding with up to K prompt-lookup drafts per sequence and step (0 = off; 1 to 7)")
    ap.add_argument("--ngram-max", type=int, default=3, help="with --speculate: the longest n-gram the proposer matches")
    ap.add_argument("--ngram-min", type=int, default=1, help="with --speculate: the shortest n-gram the proposer matches")
    ap.add_argument("--beam-width", type=int, default=0, metavar="W",
                    help="beam search with W beams per request (0 = off; 1 to 8); --batch-size then counts beams")
    ap.add_argument("--length-penalty", type=float, default=0.0, help="with --beam-width: hypotheses score sum / len^A")
    ap.add_argument("--warmup-batches", type=int, default=1,
                    help="untimed request batches served first (first-use costs: lazy kernel loading, attribute calls, graph "
                         "capture); 0 = time the cold process like the reference's script")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_textgen: needs a CUDA device (the INT4 kernels have no CPU path)")
    mc = tg.MODEL_CFGS[args.model]
    mc.dtype, mc.device = args.dtype, args.device
    layers = args.layers or mc.num_layers
    device = torch.device(args.device)
    torch.manual_seed(tg.SEED)
    model = build_model(mc, layers)
    rs = tg.generate_request_set(args.batch_size * args.num_batches, args.maxlen)
    if args.temperature is None and (args.top_k or args.top_p != 1.0):
        ap.error("--top-k / --top-p need --temperature")
    extra = dict(min_p=args.min_p, repetition_penalty=args.repetition_penalty, frequency_penalty=args.frequency_penalty,
                 presence_penalty=args.presence_penalty, logprobs=args.logprobs)
    if args.temperature is None and tg.SamplingParams(1.0, **extra).extended:
        ap.error("--min-p, the penalties and --logprobs need --temperature")
    sampling = None if args.temperature is None else tg.SamplingParams(args.temperature, args.top_k, args.top_p, args.seed, **extra)
    spec = tg.SpeculativeParams(args.speculate, args.ngram_max, args.ngram_min) if args.speculate else None
    cfg = tg.TextGenConfig(args.batch_size, prefill_chunk=args.prefill_chunk, shared_prefix=args.shared_prefix, sampling=sampling,
                           stop_token_ids=tuple(args.stop_token), speculate=spec,
                           beam=tg.BeamSearchParams(args.beam_width, args.length_penalty) if args.beam_width else None)
    # speculating, a sequence grows by up to K + 1 tokens past its length within a step: those pages too, per sequence
    spec_pages = -(-(args.speculate + 1) // args.block_len) if spec else 0
    shared_pages = -(-args.shared_prefix // args.block_len)           # the system prompt's pages, held once
    pool = KvPoolInt4(layers, mc.kv_heads, mc.hidden_size // mc.num_heads,     # the cache holds KV heads (grouped-query: fewer)
                      tg.pool_capacity(args.batch_size, args.maxlen, args.block_len) + shared_pages + args.batch_size * (shared_pages > 0)
                      + args.batch_size * spec_pages,
                      args.block_len, device)
    runner = None if args.no_cuda_graphs else tg.DecodeGraphRunner(
        model, pool, device, max_pages_per_seq=(args.maxlen + args.block_len - 1) // args.block_len + 1 + shared_pages + spec_pages,
        sampling=sampling, speculate=spec, beam=cfg.beam, stop_token_ids=cfg.stop_token_ids)
    if args.warmup_batches > 0:
        wrs = tg.generate_request_set(args.batch_size * args.warmup_batches, args.maxlen)
        tg.run_textgen(model, wrs, cfg, pool, device, sync=torch.cuda.synchronize, decode_runner=runner)
        torch.cuda.synchronize()
        rs = tg.generate_request_set(args.batch_size * args.num_batches, args.maxlen)     # the generator is seeded: same set as without warm-up
    res = tg.run_textgen(model, rs, cfg, pool, device, sync=torch.cuda.synchronize, decode_runner=runner)
    rep = tg.report(rs, cfg, res)
    rep["warmup_batches"] = args.warmup_batches
    e, et, d = rep["encode_latency_ms_per_request"], rep["encode_latency_ms_per_token"], rep["decode_latency_ms_per_token"]
    print("num_requests:", rep["num_requests"])
    print("batch_size:", rep["batch_size"])
    print("encode_latency:", f"{e[0]:.3f}ms ± {e[1]:.3f}ms per request;", f"{et[0]:.3f}ms ± {et[1]:.3f}ms per token")
    print("decode_latency:", f"{d[0]:.3f}ms ± {d[1]:.3f}ms per token")
    print("total prompt tokens:", rep["total_prompt_tokens"])
    print("total new tokens:", rep["total_new_tokens"])
    print("duration:", f"{rep['duration_s']:.3f}s")
    print("throughput ((prompt+new)/duration):", f"{rep['throughput_tokens_per_s']:.3f} token/s")
    print("peak KV pages in use:", rep["peak_kv_pages_in_use"], f"of {pool.capacity}")
    if cfg.beam is not None:
        b = rep["beam"]
        print("beam:", f"width {b['width']}, length penalty {b['length_penalty']}, {b['page_copies']} page copies "
              f"({b['page_copies_per_step']:.2f} per step, {b['bytes_copied'] / 1e6:.1f} MB), {b['stop_finished_requests']} requests "
              "ended on a stop id")
    if spec is not None:
        s = rep["speculative"]
        print("speculative:", f"{s['verify_steps']} verify steps, {s['accepted_tokens']} of {s['drafted_tokens']} drafts accepted "
              f"({s['acceptance_rate']:.3f}), {s['tokens_per_sequence_per_verify_step']:.3f} tokens per sequence per verify step")
    rep.update({"model": args.model, "layers": layers, "maxlen": args.maxlen, "kv_pool_pages": pool.buf.size(0),
                "kv_pool_GB": round((pool.buf.numel() + 2 * pool.param.numel()) / 1e9, 2)})
    print(json.dumps(rep))


if __name__ == "__main__":
    main()
