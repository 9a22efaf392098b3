"""Decode-step timing of one W4A4 Llama decoder layer (BASELINE configs #3 / #4), one CUDA graph per step.
python tools/layer_bench.py [--hidden 4096 --inter 11008 --heads 32 --batch 16 --kvlen 2048 --layers 32]
Prints JSON: us per layer-step, tokens/s extrapolated to `layers` layers."""
import argparse, json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from atom_b200.cat_tensor import BatchLenInfo
from atom_b200.kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4
from atom_b200.llama import LlamaConfig, LlamaDecoderLayer

ap = argparse.ArgumentParser()
ap.add_argument("--hidden", type=int, default=4096); ap.add_argument("--inter", type=int, default=11008)
ap.add_argument("--heads", type=int, default=32); ap.add_argument("--batch", type=int, default=16)
ap.add_argument("--kvlen", type=int, default=2048); ap.add_argument("--layers", type=int, default=32)
ap.add_argument("--page", type=int, default=32); ap.add_argument("--copies", type=int, default=3)
a = ap.parse_args()
dev = torch.device("cuda:0")
cfg = LlamaConfig(hidden_size=a.hidden, intermediate_size=a.inter, num_attention_heads=a.heads, num_hidden_layers=1)
# several independent layer instances + KV pools so that consecutive steps do not find their weights / KV in L2
layers = [LlamaDecoderLayer(cfg, 0).to(dev).init_random(i) for i in range(a.copies)]
pages = a.batch * ((a.kvlen + a.page) // a.page + 1)
kvs = []
for i in range(a.copies):
    pool = KvPoolInt4(1, a.heads, 128, capacity=pages, block_len=a.page, device=dev)
    pool.buf.random_(0, 256); pool.param[..., 0].uniform_(0.01, 0.05); pool.param[..., 1].uniform_(0.0, 0.4)
    caches = [KvCacheInt4(pool, a.kvlen) for _ in range(a.batch)]
    for c in caches:
        c.acquire_one()
    kvs.append(BatchedKvCacheInt4(caches))
blen = BatchLenInfo([], a.batch, dev)
x = torch.randn(a.batch, a.hidden, device=dev, dtype=torch.float16)
st = torch.cuda.Stream()
with torch.cuda.stream(st):
    for l, kv in zip(layers, kvs):
        l(x, blen, None, kv)
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        for l, kv in zip(layers, kvs):
            y = l(x, blen, None, kv)
    for _ in range(3):
        g.replay()
    st.synchronize()
    ts = []
    for _ in range(20):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st); g.replay(); e1.record(st); e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / a.copies)
ts.sort()
us = ts[len(ts) // 2]
w_bytes = (4 * a.hidden * a.hidden + 3 * a.hidden * a.inter) / 2 * 1.0625
kv_bytes = a.batch * a.heads * (a.kvlen + 1) * 136
print(json.dumps({"layer_decode_step": {"hidden": a.hidden, "inter": a.inter, "heads": a.heads, "batch": a.batch, "kv_len": a.kvlen},
                  "us_per_layer": round(us, 2), "tokens_per_s_at_layers": {str(a.layers): round(a.batch / (us * a.layers * 1e-6), 1)},
                  "hbm_bytes_per_layer": int(w_bytes + kv_bytes), "hbm_GBps": round((w_bytes + kv_bytes) / us * 1e-3, 1),
                  "frac_of_h100_datasheet_hbm_3350": round((w_bytes + kv_bytes) / us * 1e-3 / 3350.0, 3)}))
