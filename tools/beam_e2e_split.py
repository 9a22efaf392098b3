"""Where greedy and width-1 beam serving differ in time (DESIGN section 6): llama3-8b, 32 rows, maxlen 512, runs alternated in
one process (greedy, W = 1, greedy, W = 1), each after an untimed warm-up on the same runner.  Per run: the wall time, the host
seconds spent in the scheduler's admit and commit (commit / commit_beam) and in the runner's call (run / run_beam, which
includes the graph replay and the read-back), and the device time of one replay of the run's widest decode graph (CUDA events,
50 replays).  Prints one JSON line per run."""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # bench_textgen (it puts the repository on the path)
from bench_textgen import build_model  # noqa: E402
from atom_b200 import textgen as tg  # noqa: E402
from atom_b200.kvcache import KvPoolInt4  # noqa: E402

HOST = {}


def _timed(cls, name):
    f = getattr(cls, name)

    def wrapper(*a, **k):
        t = time.perf_counter()
        try:
            return f(*a, **k)
        finally:
            HOST[name] = HOST.get(name, 0.0) + time.perf_counter() - t
    setattr(cls, name, wrapper)


def _replay_us(graph, reps=50):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    graph.replay()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def main():
    if not torch.cuda.is_available():
        raise SystemExit("beam_e2e_split: needs a CUDA device")
    for cls, name in ((tg.TextGenScheduler, "admit"), (tg.TextGenScheduler, "commit"), (tg.TextGenScheduler, "commit_beam"),
                      (tg.DecodeGraphRunner, "run"), (tg.DecodeGraphRunner, "run_beam")):
        _timed(cls, name)
    mc = tg.MODEL_CFGS["llama3-8b"]
    dev = torch.device(mc.device)
    torch.manual_seed(tg.SEED)
    model = build_model(mc, mc.num_layers)
    for w in (0, 1, 0, 1):
        beam = tg.BeamSearchParams(w) if w else None
        cfg = tg.TextGenConfig(32, beam=beam)
        pool = KvPoolInt4(mc.num_layers, mc.kv_heads, 128, tg.pool_capacity(32, 512, 32), 32, dev)
        runner = tg.DecodeGraphRunner(model, pool, dev, max_pages_per_seq=512 // 32 + 1, beam=beam)
        tg.run_textgen(model, tg.generate_request_set(32, 512), cfg, pool, dev, sync=torch.cuda.synchronize, decode_runner=runner)
        HOST.clear()
        res = tg.run_textgen(model, tg.generate_request_set(32, 512), cfg, pool, dev, sync=torch.cuda.synchronize,
                             decode_runner=runner)
        keys = [k for k, e in runner._entries.items() if e["graph"] is not None]
        widest = max(keys, key=lambda k: k[1] if w else k[0])          # (b, groups), or ("beam", b, groups)
        print(json.dumps({"W": w, "duration_s": round(res.duration, 4), "steps": res.steps, "graphed_steps": res.graphed_steps,
                          "host_s": {k: round(v, 4) for k, v in HOST.items()}, "graph": str(widest),
                          "graph_replay_us": round(_replay_us(runner._entries[widest]["graph"]), 1)}), flush=True)


if __name__ == "__main__":
    main()
