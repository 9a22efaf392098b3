"""Continuous-batching text-generation harness -- the serving loop of
/root/reference/e2e/punica-atom/benchmarks/bench_textgen.py:21-200 (`generate_request_set`, `textgen_punica`): first come
first served, greedy, a step's batch = the prompts of newly admitted requests (prefill) followed by one token per running
request (decode), INT4 paged KV cache, per-request encode / decode latencies.

The reference writes the loop inline around the model call; here the scheduler is its own object so that the host logic
(admission, page accounting, completion, latency bookkeeping) is testable without a GPU: `TextGenScheduler.next_batch()`
produces exactly what `LlamaForCausalLM.forward(input_ids, blen, prefill_kv, decode_kv)` takes, `.commit(next_tokens,
t1, t2)` consumes the argmax of the step.  `run_textgen()` is the driver (`tools/bench_textgen.py` is its CLI).

Same workload: the request set (prompt ~ lognorm(0.8, -1, 18) clipped to [1, maxlen-2], total ~ U[0, maxlen), PCG64 seed
0xabcdabcd987) is reproduced bit for bit (tests/golden/ref_py_request_set.npz).  Differences, all deliberate:
  * the KV pool has one slot per layer (the reference allocates a single layer "to hack the memory usage", :96, and every
    layer overwrites it); 180 GB of HBM hold the real thing: 7B, batch 32, 2048 tokens = 17 GB of INT4 KV;
  * token ids are drawn on the host once per request with a seeded generator (reference: unseeded torch.randint per step);
  * admission checks the pool for free pages instead of assuming capacity.
"""
import dataclasses
import time
from typing import Callable, List, Optional

import numpy as np
import torch

from .cat_tensor import BatchLenInfo
from .kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4

SEED = 0xABCDABCD987


@dataclasses.dataclass
class RequestSet:
    prompt_lens: np.ndarray
    output_lens: np.ndarray

    def __len__(self):
        return len(self.prompt_lens)


def generate_request_set(num_requests: int, maxlen: int) -> RequestSet:
    """bench_textgen.py:31-47.  scipy draws one variate per call from the shared PCG64 stream, prompt first, then total."""
    import scipy.stats
    rng = np.random.Generator(np.random.PCG64(seed=SEED))
    prompt_dist = scipy.stats.lognorm(0.8, -1.0, 18.0)
    total_dist = scipy.stats.randint(0, maxlen)
    prompts, outputs = [], []
    for _ in range(num_requests):
        p = min(max(1, prompt_dist.rvs(random_state=rng)), maxlen - 2)
        t = max(p + 2, total_dist.rvs(random_state=rng))
        prompts.append(p)
        outputs.append(t - p)
    return RequestSet(np.array(prompts, dtype=np.int32), np.array(outputs, dtype=np.int32))


@dataclasses.dataclass
class ModelConfig:
    num_layers: int
    num_heads: int
    hidden_size: int
    intermediate_size: int
    dtype: str = "float16"
    device: str = "cuda:0"
    num_kv_heads: Optional[int] = None     # None = multi-head attention; the KV pool has this many heads
    rope_theta: float = 10000.0

    @property
    def kv_heads(self) -> int:
        return self.num_kv_heads or self.num_heads


MODEL_CFGS = {
    "7b": ModelConfig(num_layers=32, num_heads=32, hidden_size=4096, intermediate_size=11008),
    "13b": ModelConfig(num_layers=40, num_heads=40, hidden_size=5120, intermediate_size=13824),
    "70b": ModelConfig(num_layers=80, num_heads=64, hidden_size=8192, intermediate_size=28672, num_kv_heads=8),
    "llama3-8b": ModelConfig(num_layers=32, num_heads=32, hidden_size=4096, intermediate_size=14336, num_kv_heads=8, rope_theta=5e5),
}


@dataclasses.dataclass
class TextGenConfig:
    batch_size: int


@dataclasses.dataclass
class TextGenBenchResult:
    encode_latency: np.ndarray
    decode_latency: np.ndarray
    duration: float
    steps: int = 0
    tokens: Optional[List[List[int]]] = None
    graphed_steps: int = 0


@dataclasses.dataclass
class RequestContext:
    req_idx: int
    kvcache: KvCacheInt4
    output: List[int]
    encode_latency: float = 0.0
    decode_start_at: float = 0.0
    decode_latency: float = 0.0


@dataclasses.dataclass
class StepBatch:
    input_ids: List[int]
    blen: BatchLenInfo
    prefill_kv: Optional[BatchedKvCacheInt4]
    decode_kv: Optional[BatchedKvCacheInt4]
    num_new: int


class TextGenScheduler:
    """FCFS continuous batching over a KvPoolInt4 (bench_textgen.py:111-191 as a state machine)."""

    def __init__(self, rs: RequestSet, batch_size: int, pool: KvPoolInt4, device, vocab_size: int = 32000):
        self.rs, self.batch_size, self.pool, self.device = rs, batch_size, pool, device
        self.vocab_size = vocab_size
        self.next_req_idx = 0
        self.workset: List[RequestContext] = []
        self.done: List[RequestContext] = []
        self._new: list = []
        self._admitted = False
        self._blen = None
        self._rng = np.random.Generator(np.random.PCG64(seed=SEED))

    @property
    def finished(self) -> bool:
        return len(self.done) == len(self.rs)

    def _pages_needed(self, prompt_len: int) -> int:
        # the prompt's pages plus one spare: the first generated token may open a new page
        return (prompt_len + self.pool.block_len - 1) // self.pool.block_len + 1

    def admit(self) -> int:
        """Admit waiting requests (FCFS) while the batch has room and the pool has pages; returns how many are new this step."""
        assert not self.finished and not self._admitted, "commit() the previous step first"
        # running requests may each need a fresh page this step; keep those in reserve before admitting anyone
        reserve = len(self.workset)
        while len(self.workset) + len(self._new) < self.batch_size and self.next_req_idx < len(self.rs):
            plen = int(self.rs.prompt_lens[self.next_req_idx])
            if self.pool.num_free_blocks - reserve < self._pages_needed(plen):
                if not self.workset and not self._new:
                    raise RuntimeError(f"KV pool too small for request {self.next_req_idx} (prompt {plen} tokens)")
                break
            idx = self.next_req_idx
            self.next_req_idx += 1
            prompt = self._rng.integers(0, self.vocab_size, plen).tolist()
            self._new.append((idx, prompt, KvCacheInt4(self.pool, plen)))
            reserve += 1
        self._admitted = True
        return len(self._new)

    def next_batch(self) -> StepBatch:
        """The step's model inputs: prompts of the new requests, then the last token of every running request."""
        if not self._admitted:
            self.admit()
        input_ids: List[int] = []
        for _, prompt, _ in self._new:
            input_ids.extend(prompt)
        input_ids.extend(int(r.output[-1]) for r in self.workset)
        self._blen = BatchLenInfo([len(p) for _, p, _ in self._new], len(self.workset), self.device)
        prefill_kv = BatchedKvCacheInt4([kv for _, _, kv in self._new]) if self._new else None
        decode_kv = BatchedKvCacheInt4([r.kvcache for r in self.workset]) if self.workset else None
        return StepBatch(input_ids, self._blen, prefill_kv, decode_kv, len(self._new))

    def last_token_rows(self) -> List[int]:
        """Rows of the step's hidden states whose logits are needed: the last token of every prompt, then all decode rows."""
        blen = self._blen
        rows = [] if blen.indptr is None else (blen.indptr[1:] - 1).tolist()
        return rows + list(range(blen.doff, blen.doff + blen.decode))

    def commit(self, next_tokens, t1: float, t2: float) -> int:
        """next_tokens: one id per row of last_token_rows().  Returns the number of tokens this step processed."""
        n_new = len(self._new)
        assert len(next_tokens) == n_new + len(self.workset)
        processed = sum(len(p) for _, p, _ in self._new) + len(self.workset)
        new_workset: List[RequestContext] = []
        for b, (req_idx, _, kv) in enumerate(self._new):
            req = RequestContext(req_idx, kv, [int(next_tokens[b])], encode_latency=t2 - t1, decode_start_at=t1)
            self._finish_or_continue(req, t2, new_workset)
        for b, req in enumerate(self.workset):
            req.output.append(int(next_tokens[n_new + b]))
            self._finish_or_continue(req, t2, new_workset)
        self.workset, self._new, self._admitted = new_workset, [], False
        return processed

    def _finish_or_continue(self, req, t2, new_workset):
        if len(req.output) >= int(self.rs.output_lens[req.req_idx]):
            req.decode_latency = t2 - req.decode_start_at
            req.kvcache.release()
            self.done.append(req)
        else:
            req.kvcache.acquire_one()
            new_workset.append(req)

    def result(self, duration: float, steps: int, keep_tokens: bool = False) -> TextGenBenchResult:
        done = sorted(self.done, key=lambda r: r.req_idx)
        return TextGenBenchResult(np.array([r.encode_latency for r in done]), np.array([r.decode_latency for r in done]),
                                  duration, steps, [r.output for r in done] if keep_tokens else None)


class _StaticKv:
    """The attributes the KV ops read (kvcache.BatchedKvCacheInt4), backed by fixed device buffers."""

    def __init__(self, pool, indptr, indicies, last_page_offset):
        self.data, self.param = pool.buf, pool.param
        self.indptr, self.indicies, self.last_page_offset = indptr, indicies, last_page_offset

    @property
    def page_size(self):
        return self.data.size(-2)


class DecodeGraphRunner:
    """Decode-only steps replayed from CUDA graphs, one graph per batch size.

    In steady state almost every step of the serving loop is decode-only (outputs are ~50x longer than prompts in the
    reference's request set) and a 32-layer step is ~500 kernel launches: launch-bound from Python.  All per-step state of
    such a step is a handful of integers -- the input token of each sequence and the page table -- so they live in ONE
    fixed int32 device buffer  [ids(B) | indptr(B+1) | last_page_offset(B) | indicies(B * max_pages)]  that is refreshed
    with a single pinned H2D copy, after which the captured step (embedding, all layers: fused norm+quantise, INT4 GEMMs,
    KV append, INT4 decode attention, lm_head, argmax) is replayed.  The kernels read the page table from device memory and
    their grids depend only on B, so the graph stays valid as sequences grow and change pages.

    capture=False runs the same buffers through the model eagerly (the CPU tests use it; it is also the warm-up path)."""

    def __init__(self, model: Callable, pool: KvPoolInt4, device, max_pages_per_seq: int, capture: bool = True):
        self.model, self.pool, self.device = model, pool, torch.device(device)
        self.max_pages, self.capture = max_pages_per_seq, capture
        self._entries = {}

    def _layout(self, b):
        o_ids, o_indptr, o_last, o_ind = 0, b, 2 * b + 1, 3 * b + 1
        return o_ids, o_indptr, o_last, o_ind, 3 * b + 1 + b * self.max_pages

    def _entry(self, b):
        e = self._entries.get(b)
        if e is None:
            o_ids, o_indptr, o_last, o_ind, total = self._layout(b)
            host = torch.zeros(total, dtype=torch.int32)
            if self.device.type == "cuda":
                host = host.pin_memory()
            dev = torch.zeros(total, dtype=torch.int32, device=self.device)
            kv = _StaticKv(self.pool, dev[o_indptr:o_indptr + b + 1], dev[o_ind:o_ind + b * self.max_pages], dev[o_last:o_last + b])
            e = {"host": host, "dev": dev, "ids": dev[o_ids:o_ids + b], "kv": kv, "blen": BatchLenInfo([], b, self.device),
                 "graph": None, "out": None}
            self._entries[b] = e
        return e

    def _step(self, e):
        logits, _ = self.model(e["ids"], e["blen"], None, e["kv"])
        return torch.argmax(logits, dim=-1)

    def run(self, last_tokens: List[int], kvs: List[KvCacheInt4]) -> np.ndarray:
        b = len(kvs)
        e = self._entry(b)
        o_ids, o_indptr, o_last, o_ind, _ = self._layout(b)
        h = e["host"].numpy()
        h[o_ids:o_ids + b] = last_tokens
        n = 0
        h[o_indptr] = 0
        for i, c in enumerate(kvs):
            pages = c.indicies
            if len(pages) > self.max_pages:
                raise RuntimeError(f"sequence holds {len(pages)} pages, runner was sized for {self.max_pages}")
            h[o_ind + n:o_ind + n + len(pages)] = pages
            n += len(pages)
            h[o_indptr + i + 1] = n
            h[o_last + i] = (c.seqlen - 1) % self.pool.block_len + 1
        e["dev"].copy_(e["host"], non_blocking=True)
        if not self.capture:
            return self._step(e).cpu().numpy()
        if e["graph"] is None:
            side = torch.cuda.Stream(self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):
                self._step(e)                       # warm-up on real data (lazy initialisations must not be captured)
                side.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=side):
                    e["out"] = self._step(e)
            torch.cuda.current_stream(self.device).wait_stream(side)
            e["graph"] = g
        e["graph"].replay()
        return e["out"].cpu().numpy()               # synchronises: the caller needs the tokens to go on


def _vocab_size(model) -> int:
    """Prompt ids must index the model's own embedding table (the reference hard-codes 32000, bench_textgen.py:119)."""
    head = getattr(model, "lm_head", None)
    if head is not None and hasattr(head, "out_features"):
        return int(head.out_features)
    cfg = getattr(model, "config", None) or getattr(getattr(model, "model", None), "config", None)
    return int(getattr(cfg, "vocab_size", 32000))


def pool_capacity(batch_size: int, maxlen: int, block_len: int) -> int:
    """Pages for `batch_size` sequences of up to `maxlen` tokens (+1 spare page each), bench_textgen.py:99."""
    return batch_size * ((maxlen + block_len - 1) // block_len + 1)


@torch.inference_mode()
def run_textgen(model: Callable, rs: RequestSet, cfg: TextGenConfig, pool: KvPoolInt4, device, sync: Callable = None,
                keep_tokens: bool = False, progress: Callable = None, decode_runner: DecodeGraphRunner = None) -> TextGenBenchResult:
    """Drive `model(input_ids, blen, prefill_kv, decode_kv) -> (logits, hidden)` through the whole request set.
    Latencies are wall-clock around the step *including* the device->host read of the next tokens (which synchronises),
    as in the reference.  With a `decode_runner`, steps that admit no new request are replayed from its CUDA graphs."""
    sched = TextGenScheduler(rs, cfg.batch_size, pool, device, vocab_size=_vocab_size(model))
    steps = graphed = 0
    t_start = time.perf_counter()
    while not sched.finished:
        n_new = sched.admit()
        t1 = time.perf_counter()
        if decode_runner is not None and n_new == 0:
            next_tokens = decode_runner.run([int(r.output[-1]) for r in sched.workset], [r.kvcache for r in sched.workset])
            graphed += 1
        else:
            batch = sched.next_batch()
            ids = torch.tensor(batch.input_ids, dtype=torch.long, device=device)
            logits, _ = model(ids, batch.blen, batch.prefill_kv, batch.decode_kv)
            rows = torch.tensor(sched.last_token_rows(), dtype=torch.long, device=logits.device)
            next_tokens = torch.argmax(logits.index_select(0, rows), dim=-1).cpu().numpy()
        if sync is not None:
            sync()
        t2 = time.perf_counter()
        n = sched.commit(next_tokens, t1, t2)
        steps += 1
        if progress is not None:
            progress(n)
    res = sched.result(time.perf_counter() - t_start, steps, keep_tokens)
    res.graphed_steps = graphed
    return res


def report(rs: RequestSet, cfg: TextGenConfig, res: TextGenBenchResult) -> dict:
    """The figures bench_textgen.py:509-528 prints, as a dict (throughput = (prompt + new tokens) / duration)."""
    per_prompt_tok = res.encode_latency / rs.prompt_lens
    per_new_tok = res.decode_latency / rs.output_lens
    total = int(rs.prompt_lens.sum()) + int(rs.output_lens.sum())
    return {
        "num_requests": len(rs), "batch_size": cfg.batch_size, "steps": res.steps, "graphed_decode_steps": res.graphed_steps,
        "encode_latency_ms_per_request": [float(res.encode_latency.mean() * 1e3), float(res.encode_latency.std() * 1e3)],
        "encode_latency_ms_per_token": [float(per_prompt_tok.mean() * 1e3), float(per_prompt_tok.std() * 1e3)],
        "decode_latency_ms_per_token": [float(per_new_tok.mean() * 1e3), float(per_new_tok.std() * 1e3)],
        "total_prompt_tokens": int(rs.prompt_lens.sum()), "total_new_tokens": int(rs.output_lens.sum()),
        "duration_s": res.duration, "throughput_tokens_per_s": total / res.duration,
    }
