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
import heapq
import time
from typing import Callable, List, Optional, Tuple

import numpy as np
import torch

from .cat_tensor import BatchLenInfo
from .kvcache import BatchedKvCacheInt4, KvCacheInt4, KvPoolInt4, prefix_groups

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
class SamplingParams:
    """Sampled decoding (ops.sample_tokens): every request draws its tokens at this temperature (0 = greedy), top_k (0 = off)
    and top_p (1 = off).  Request r's Philox key is (seed, r) and the counter of a token is the number of tokens r generated
    before it, so its tokens depend on its own logits only -- not on batching, chunking, shared prefixes or graphs.

    min_p (0 = off), repetition_penalty (1 = off), frequency_penalty and presence_penalty (0 = off) and logprobs (None = off,
    else the top-n list's length, 0 to 20) are ops.sample_tokens' options.  With any penalty every request holds a slot of a
    device penalty table (its prompt tokens and a count of each token it generated), which the sampler reads and updates."""
    temperature: float
    top_k: int = 0
    top_p: float = 1.0
    seed: int = 0
    min_p: float = 0.0
    repetition_penalty: float = 1.0
    frequency_penalty: float = 0.0
    presence_penalty: float = 0.0
    logprobs: Optional[int] = None

    _EXTRAS = {"min_p": 0.0, "repetition_penalty": 1.0, "frequency_penalty": 0.0, "presence_penalty": 0.0, "logprobs": None}

    def __post_init__(self):
        if not (np.isfinite(self.temperature) and self.temperature >= 0):
            raise ValueError(f"temperature must be finite and >= 0, got {self.temperature}")
        if int(self.top_k) < 0 or not (0 < self.top_p <= 1) or not (0 <= int(self.seed) < 1 << 64):
            raise ValueError(f"need top_k >= 0, top_p in (0, 1] and a seed in [0, 2^64): {self}")
        if not (0 <= self.min_p <= 1) or not (np.isfinite(self.repetition_penalty) and self.repetition_penalty > 0) or \
                not np.isfinite(self.frequency_penalty) or not np.isfinite(self.presence_penalty):
            raise ValueError(f"need min_p in [0, 1], repetition_penalty finite and > 0, finite frequency and presence penalties: {self}")
        if self.logprobs is not None and not (isinstance(self.logprobs, (int, np.integer)) and 0 <= self.logprobs <= 20):
            raise ValueError(f"logprobs must be None or an integer in [0, 20], got {self.logprobs!r}")

    @property
    def penalties(self) -> bool:
        """Whether any penalty is on (the requests then hold penalty-table slots)."""
        return self.repetition_penalty != 1 or self.frequency_penalty != 0 or self.presence_penalty != 0

    @property
    def extended(self) -> bool:
        """Whether the sampler is called with options beyond temperature, top-k and top-p."""
        return self.penalties or self.min_p != 0 or self.logprobs is not None

    def options(self, n: int, table=None, slots=None) -> dict:
        """ops.sample_tokens' keyword options for n rows (host values) with the given table and row slots."""
        o = {"min_p": [self.min_p] * n}
        if self.penalties:
            o.update(repetition_penalty=[self.repetition_penalty] * n, frequency_penalty=[self.frequency_penalty] * n,
                     presence_penalty=[self.presence_penalty] * n, penalty_table=table, slots=slots)
        if self.logprobs is not None:
            o["logprobs"] = int(self.logprobs)
        return o

    def asdict(self) -> dict:
        """The settings; the options beyond temperature, top-k, top-p and seed only when they are not at their defaults."""
        d = dataclasses.asdict(self)
        return {k: v for k, v in d.items() if k not in self._EXTRAS or v != self._EXTRAS[k]}


@dataclasses.dataclass(frozen=True)
class SpeculativeParams:
    """Speculative decoding with prompt-lookup drafts (DESIGN sections 5.7 and 5.8).  After every step the device commits each
    sequence's accepted tokens to its token history (its whole context: the shared system prompt, its prompt and its generated
    tokens) and proposes up to num_draft drafts: the tokens that followed the latest earlier occurrence of the history's last
    n tokens, for the longest n in [ngram_min, ngram_max] that occurs.  The next step carries S = 1 + the longest draft of the
    batch tokens per running sequence (S = 1: a plain decode step), and the sampler accepts or replaces each draft so that
    greedy runs give the greedy tokens and sampled runs draw from exactly the sampler's distribution."""
    num_draft: int = 4
    ngram_max: int = 3
    ngram_min: int = 1

    def __post_init__(self):
        if not (1 <= int(self.num_draft) <= 7 and 1 <= int(self.ngram_min) <= int(self.ngram_max) <= 16):
            raise ValueError(f"need 1 <= num_draft <= 7 and 1 <= ngram_min <= ngram_max <= 16: {self}")


@dataclasses.dataclass(frozen=True)
class BeamSearchParams:
    """Beam search (DESIGN section 5.9): every request keeps up to `width` live beams, ranked by the FP32 sum of their tokens'
    log-probabilities (ops.beam_select), and up to `width` finished hypotheses -- a beam that chose a stop id, or a live beam
    that reached the output length -- scored sum / len^length_penalty in float64.  A request is done when it holds `width`
    finished hypotheses or its beams reach the output length; its output is the best finished hypothesis.  width = 1 gives the
    greedy tokens."""
    width: int = 4
    length_penalty: float = 0.0

    def __post_init__(self):
        if not (isinstance(self.width, (int, np.integer)) and 1 <= self.width <= 8) or not np.isfinite(self.length_penalty):
            raise ValueError(f"need 1 <= width <= 8 and a finite length_penalty: {self}")


@dataclasses.dataclass
class TextGenConfig:
    batch_size: int
    prefill_chunk: Optional[int] = None     # at most this many prompt tokens per step (chunked prefill); None = whole prompts
    shared_prefix: int = 0                  # tokens of one system prompt before every request's prompt, prefilled once and forked
    sampling: Optional[SamplingParams] = None   # None: greedy (argmax)
    stop_token_ids: Tuple[int, ...] = ()        # a request that emits one of these finishes on it (greedy or sampled)
    speculate: Optional[SpeculativeParams] = None   # None: one token per running request and step
    beam: Optional[BeamSearchParams] = None         # None: one sequence per request


@dataclasses.dataclass
class TextGenBenchResult:
    encode_latency: np.ndarray
    decode_latency: np.ndarray
    duration: float
    steps: int = 0
    tokens: Optional[List[List[int]]] = None
    graphed_steps: int = 0
    peak_pages: int = 0                     # most KV pages in use after any step's admission
    output_lens: Optional[np.ndarray] = None    # tokens each request generated (fewer than asked when it met a stop id)
    logprobs: Optional[List[List[float]]] = None    # with SamplingParams.logprobs and keep_tokens: each token's log-probability
    top_logprobs: Optional[List[List[Tuple[List[int], List[float]]]]] = None    # ... and each token's top-n (ids, logprobs)
    speculative: Optional[dict] = None      # with speculation: TextGenScheduler.spec_stats
    beam_scores: Optional[np.ndarray] = None    # with beam search: the score of each request's output
    beam: Optional[dict] = None             # with beam search: TextGenScheduler.beam_stats


@dataclasses.dataclass
class RequestContext:
    req_idx: int
    kvcache: KvCacheInt4
    output: List[int]
    encode_latency: float = 0.0
    decode_start_at: float = 0.0
    decode_latency: float = 0.0
    slot: int = -1                          # its penalty-table slot (-1: none)
    logprobs: List[float] = dataclasses.field(default_factory=list)
    top_logprobs: List[tuple] = dataclasses.field(default_factory=list)
    drafts: List[int] = dataclasses.field(default_factory=list)     # with speculation: the next step's drafts
    beam_sum: float = 0.0                   # with beam search: this beam's FP32 sum of log-probabilities
    group: Optional["_BeamGroup"] = None    # with beam search: the request this beam belongs to


@dataclasses.dataclass(eq=False)
class _BeamGroup:
    """A beam-search request: its finished hypotheses (score, arrival, tokens) and timings; its live beams are in the workset."""
    req_idx: int
    encode_latency: float
    decode_start_at: float
    finished: list = dataclasses.field(default_factory=list)
    arrivals: int = 0


@dataclasses.dataclass(eq=False)
class _Prefill:
    """A request whose prompt is not yet wholly in the cache."""
    req_idx: int
    prompt: List[int]
    kvcache: KvCacheInt4
    done: int = 0                           # prompt tokens already in the cache
    start_at: Optional[float] = None        # start of the step that carried its first chunk
    slot: int = -1                          # its penalty-table slot (-1: none)


@dataclasses.dataclass
class StepBatch:
    input_ids: List[int]
    blen: BatchLenInfo
    prefill_kv: Optional[BatchedKvCacheInt4]
    decode_kv: Optional[BatchedKvCacheInt4]
    num_new: int


class TextGenScheduler:
    """FCFS continuous batching over a KvPoolInt4 (bench_textgen.py:111-191 as a state machine).

    prefill_chunk=None: a step carries the whole prompt of every request it admits (the reference's schedule).  prefill_chunk=N
    (chunked prefill): a step carries at most N prompt tokens in all -- first the next chunks of the requests that are partly
    prefilled, FCFS, then the first chunks of newly admitted ones -- so that a long prompt no longer stalls every running
    sequence's decode for one long step.  A chunk is the tail of its sequence's cached tokens; the model's prefill attention then
    also reads the chunks before it from the cache.  A request gets its first token from the step that completes its prompt.

    shared_prefix=N (> 0): every request's prompt is preceded by one common N-token system prompt, drawn from a seeded stream of
    its own (the request set and the requests' prompts are those of N = 0).  It is prefilled once, first, as a root sequence that
    produces no token (chunked under prefill_chunk like any prompt); each request admitted after that is `root.fork()` followed
    by its own prompt as a continuation, and admission counts only the pages the fork takes.  The root is released when the last
    request finishes.  Decode batches of forked requests carry prefix groups (kvcache.BatchedKvCacheInt4).

    stop_token_ids: a request that emits one of them finishes on that token (its pages and slot are released).
    penalty_slots=True: every admitted request takes a slot of a penalty table of batch_size slots (the smallest free one), to be
    set up with its whole prompt -- the system prompt and its own -- before its first token is drawn: `slot_inits` lists the
    (slot, prompt tokens) the driver must apply after each admit().  The slot is freed when the request finishes; the system
    prompt's root sequence has none.

    num_draft=K (> 0, speculative decoding; needs slots, which then index the device token histories): a running request carries
    the drafts the device proposed for it after the previous step.  A step carries S = 1 + the longest of them rows per running
    request -- [last token, drafts, padding] -- after the prompt chunks; admit() grows each running sequence by S - 1 tokens for
    them and keeps pages in reserve for every running request to grow by K + 1 tokens.  commit_spec() takes the device's per-
    sequence result (tokens emitted, drafts), cuts the tokens at the output length and the first stop id, and truncates each
    sequence to the tokens it kept."""

    def __init__(self, rs: RequestSet, batch_size: int, pool: KvPoolInt4, device, vocab_size: int = 32000,
                 prefill_chunk: Optional[int] = None, shared_prefix: int = 0, stop_token_ids=(), penalty_slots: bool = False,
                 num_draft: int = 0, beam: Optional[BeamSearchParams] = None):
        if prefill_chunk is not None and int(prefill_chunk) < 1:
            raise ValueError("prefill_chunk must be a positive number of tokens (or None)")
        if int(shared_prefix) < 0:
            raise ValueError("shared_prefix must be a non-negative number of tokens")
        self.rs, self.batch_size, self.pool, self.device = rs, batch_size, pool, device
        self.vocab_size = vocab_size
        self.prefill_chunk = None if prefill_chunk is None else int(prefill_chunk)
        self.next_req_idx = 0
        self.workset: List[RequestContext] = []
        self.done: List[RequestContext] = []
        self._prefilling: List[_Prefill] = []     # admitted, prompt not yet wholly cached (FCFS)
        self._new: list = []                      # this step's prompt chunks: (_Prefill, first token, tokens)
        self._admitted = False
        self._blen = None
        self._rng = np.random.Generator(np.random.PCG64(seed=SEED))
        self.shared_prefix = int(shared_prefix)
        self._root: Optional[_Prefill] = None          # the system prompt's sequence (req_idx -1), prefilled before any request
        if self.shared_prefix:
            system = np.random.Generator(np.random.PCG64(seed=SEED + 1)).integers(0, vocab_size, self.shared_prefix).tolist()
            self._root = _Prefill(-1, system, KvCacheInt4(pool, 0))
            self._prefilling.append(self._root)
        self.stop_token_ids = frozenset(int(t) for t in stop_token_ids)
        self._free_slots = list(range(batch_size)) if penalty_slots else None
        self.slot_inits: List[tuple] = []
        self.num_draft = int(num_draft)
        if self.num_draft and self._free_slots is None:
            raise ValueError("speculation needs slots (penalty_slots=True): they index the token histories")
        self.S = 1                                  # rows per running request in the admitted step
        self.beam = beam
        self.copies: List[tuple] = []               # beam search: the page copies of the last commit's forks, for the next step
        self.beam_stats = {"page_copies": 0, "copied_slots": 0, "stop_finished": 0}
        self.spec_stats = {"verify_steps": 0, "drafted_tokens": 0, "accepted_tokens": 0, "emitted_tokens": 0,
                           "verify_sequence_steps": 0, "verify_emitted_tokens": 0}

    @property
    def finished(self) -> bool:
        return len(self.done) == len(self.rs)

    @property
    def prompt_tokens(self) -> int:
        """Prompt tokens the admitted step carries (0: a decode-only step)."""
        return sum(n for _, _, n in self._new)

    def _pages_needed(self, prompt_len: int) -> int:
        # the prompt's pages plus one spare: the first generated token may open a new page.  Behind a shared prefix of N tokens
        # a fork takes the pages from N // P on: a copy of the partly filled page, if any, and the pages its prompt adds
        n, bl = self.shared_prefix, self.pool.block_len
        if self.beam is not None:
            # beam search: the first step forks the prompt into up to W beams, each of which can take one page (a copy of the
            # partly filled page, or a fresh one for its next token)
            return (n + prompt_len + bl - 1) // bl - n // bl + self.beam.width
        if self.num_draft:
            # speculating, the spare is room for the first token and for its first step as a running request, which can grow
            # the sequence by K + 1 more tokens
            return -(-(n + prompt_len + 1 + self.num_draft + 1) // bl) - n // bl
        return (n + prompt_len + bl - 1) // bl - n // bl + 1

    def _outstanding(self, p: _Prefill) -> int:
        # pages a request being prefilled will still take: the rest of its prompt and the spare (the root: the rest of it)
        if p.req_idx < 0:
            return -(-len(p.prompt) // self.pool.block_len) - len(p.kvcache.indicies)
        return self._pages_needed(len(p.prompt)) - (len(p.kvcache.indicies) - self.shared_prefix // self.pool.block_len)

    def admit(self) -> int:
        """Continue the partly prefilled requests, then admit waiting ones (FCFS) while the batch has room, the step has prompt
        tokens to spare and the pool has pages; returns how many prompts (whole or chunks) the step carries."""
        assert not self.finished and not self._admitted, "commit() the previous step first"
        budget = self.prefill_chunk
        # running requests may each need a fresh page this step, and the requests being prefilled the pages of the rest of
        # their prompt: keep those in reserve before admitting anyone, so that no admitted request ever waits for a page
        reserve = len(self.workset) + sum(self._outstanding(p) for p in self._prefilling)
        if self.beam is not None:                   # ... or, with beams, a page for each of up to W beams per running request
            reserve += self.beam.width * len({id(r.group) for r in self.workset}) - len(self.workset)
        if self.num_draft:                          # ... or, speculating, pages for K + 1 more tokens
            bl = self.pool.block_len
            reserve += sum(-(-(r.kvcache.seqlen + self.num_draft + 1) // bl) - len(r.kvcache.indicies) - 1 for r in self.workset)
        for p in self._prefilling:
            if budget is not None and budget == 0:
                break
            n = len(p.prompt) - p.done if budget is None else min(len(p.prompt) - p.done, budget)
            before = len(p.kvcache.indicies)
            p.kvcache.acquire(n)                            # from the reserve
            reserve -= len(p.kvcache.indicies) - before
            self._new.append((p, p.done, n))
            budget = None if budget is None else budget - n
        root_done = self._root is None or self._root.done == len(self._root.prompt)
        while root_done and self._room() and self.next_req_idx < len(self.rs) and (budget is None or budget > 0):
            plen = int(self.rs.prompt_lens[self.next_req_idx])
            if self.pool.num_free_blocks - reserve < self._pages_needed(plen):
                if not self.workset and not self._prefilling:
                    raise RuntimeError(f"KV pool too small for request {self.next_req_idx} (prompt {plen} tokens)")
                break
            idx = self.next_req_idx
            self.next_req_idx += 1
            prompt = self._rng.integers(0, self.vocab_size, plen).tolist()
            n = plen if budget is None else min(plen, budget)
            if self._root is None:
                kv = KvCacheInt4(self.pool, n)
            else:
                kv = self._root.kvcache.fork()
                kv.acquire(n)
            p = _Prefill(idx, prompt, kv)
            if self._free_slots is not None:
                p.slot = heapq.heappop(self._free_slots)
                self.slot_inits.append((p.slot, (self._root.prompt if self._root is not None else []) + prompt))
            self._prefilling.append(p)
            self._new.append((p, 0, n))
            reserve += self._outstanding(p)
            budget = None if budget is None else budget - n
        self.S = 1 + max((len(r.drafts) for r in self.workset), default=0)
        for r in self.workset:                      # the verify rows' K/V slots (from the reserve)
            r.kvcache.acquire(self.S - 1)
        self._admitted = True
        return len(self._new)

    def _room(self) -> bool:
        """Whether the batch has room for one more request: a sequence, or with beam search W rows (sequences) from admission."""
        if self.beam is None:
            return len(self.workset) + len(self._prefilling) < self.batch_size
        groups = len({id(r.group) for r in self.workset}) + sum(p.req_idx >= 0 for p in self._prefilling)
        return (groups + 1) * self.beam.width <= self.batch_size

    def next_batch(self) -> StepBatch:
        """The step's model inputs: the prompt chunks (whole prompts without chunking), then the last token of every running
        request."""
        if not self._admitted:
            self.admit()
        input_ids: List[int] = []
        for p, s, n in self._new:
            input_ids.extend(p.prompt[s:s + n])
        input_ids.extend(self.decode_ids())
        self._blen = BatchLenInfo([n for _, _, n in self._new], len(self.workset), self.device, decode_len=self.S)
        prefill_kv = BatchedKvCacheInt4([p.kvcache for p, _, _ in self._new]) if self._new else None
        decode_kv = BatchedKvCacheInt4([r.kvcache for r in self.workset]) if self.workset else None
        return StepBatch(input_ids, self._blen, prefill_kv, decode_kv, len(self._new))

    def last_token_rows(self) -> List[int]:
        """Rows of the step's hidden states whose logits are needed: the last token of every prompt this step completes, then
        all decode rows.  A chunk in the middle of its prompt has none."""
        blen = self._blen
        rows = [] if blen.indptr is None else (blen.indptr[1:] - 1).tolist()
        chunks = getattr(self, "_new", None)        # None: a bare step description, whole prompts only
        if chunks is not None:
            rows = [r for r, (p, s, n) in zip(rows, chunks) if s + n == len(p.prompt) and p.req_idx >= 0]
        return rows + list(range(blen.doff, blen.doff + blen.decode * blen.decode_len))

    def _first(self) -> list:
        """The requests whose first token this step draws (prompts it completes, the system prompt's root excluded)."""
        return [p for p, s, n in (getattr(self, "_new", None) or []) if s + n == len(p.prompt) and p.req_idx >= 0]

    def decode_ids(self) -> List[int]:
        """Input ids of the running requests' rows: the last token, then (speculating) the drafts and padding up to S rows."""
        out: List[int] = []
        for r in self.workset:
            row = [int(r.output[-1])] + r.drafts
            out.extend(row + [row[-1]] * (self.S - len(row)))
        return out

    def candidates(self) -> List[int]:
        """Speculating: the candidate of every row of last_token_rows() (-1: none): row j of a running request proposes its
        draft j, the token its input at row j + 1 assumed."""
        out = [-1] * len(self._first())
        for r in self.workset:
            out.extend(r.drafts + [-1] * (self.S - len(r.drafts)))
        return out

    def sequence_rows(self) -> List[int]:
        """Speculating: the rows of last_token_rows() of each sequence that draws (those of sequence_slots()), as an indptr."""
        counts = [1] * len(self._first()) + [self.S] * len(self.workset)
        return np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int32).tolist()

    def sequence_slots(self) -> List[int]:
        """Speculating: the token-history slot of each sequence that draws, first tokens first, then the running requests."""
        return [p.slot for p in self._first()] + [r.slot for r in self.workset]

    def sample_slots(self) -> List[tuple]:
        """(request index, counter) of every row of last_token_rows(), in its order: the counter is the number of tokens the
        request has generated so far (0 for the row that completes its prompt)."""
        chunks = getattr(self, "_new", None) or []
        first = [(p.req_idx, 0) for p, s, n in chunks if s + n == len(p.prompt) and p.req_idx >= 0]
        return first + [(r.req_idx, len(r.output) + j) for r in self.workset for j in range(self.S)]

    def row_slots(self) -> List[int]:
        """The penalty-table slot of every row of last_token_rows(), in its order (-1: none)."""
        chunks = getattr(self, "_new", None) or []
        return [p.slot for p, s, n in chunks if s + n == len(p.prompt) and p.req_idx >= 0] + \
            [r.slot for r in self.workset for _ in range(self.S)]

    def commit(self, next_tokens, t1: float, t2: float, logprobs=None, _speculative=False) -> int:
        """next_tokens: one id per row of last_token_rows(); logprobs: None or (logprob [R], top_ids [R, n], top_logprobs [R, n])
        for the same rows.  Returns the number of tokens this step processed."""
        completes = [s + n == len(p.prompt) for p, s, n in self._new]
        n_first = sum(c for (p, _, _), c in zip(self._new, completes) if p.req_idx >= 0)
        assert len(next_tokens) == n_first + len(self.workset)
        processed = sum(n for _, _, n in self._new) + len(self.workset)
        new_workset: List[RequestContext] = []
        b = 0
        first = []
        for (p, _, n), c in zip(self._new, completes):
            p.done += n
            if p.start_at is None:
                p.start_at = t1
            if not c:
                continue
            self._prefilling.remove(p)
            if p.req_idx < 0:                               # the system prompt: cached, no token
                continue
            req = RequestContext(p.req_idx, p.kvcache, [int(next_tokens[b])], encode_latency=t2 - p.start_at, decode_start_at=p.start_at,
                                 slot=p.slot)
            self._keep_logprobs(req, logprobs, b)
            b += 1
            first.append(req)
            self._finish_or_continue(req, t2, new_workset)
        if _speculative:                            # commit_spec() goes on with the running requests
            self._first_committed, self._first_workset, self._running_committed = first, new_workset, self.workset
            self._new, self._admitted = [], False
            return processed
        for i, req in enumerate(self.workset):
            req.output.append(int(next_tokens[n_first + i]))
            self._keep_logprobs(req, logprobs, n_first + i)
            self._finish_or_continue(req, t2, new_workset)
        self.workset, self._new, self._admitted = new_workset, [], False
        return processed

    def commit_spec(self, out, t1: float, t2: float, logprobs=None) -> int:
        """Speculating: out int32 [sequences, 2K + 3], one row per sequence of sequence_slots() (ops.spec_commit_propose: tokens
        emitted, drafts proposed, the tokens, the drafts); logprobs as commit()'s, for the rows of last_token_rows().  Returns the
        number of tokens this step processed."""
        K, S = self.num_draft, self.S
        out = np.asarray(out)
        first, rows = len(self._first()), self.sequence_rows()
        seq_drafts = [[int(t) for t in o[K + 3:K + 3 + int(o[1])]] for o in out]
        tokens = [[int(t) for t in o[2:2 + int(o[0])]] for o in out]
        processed = sum(n for _, _, n in self._new) + S * len(self.workset)
        if S > 1:
            st = self.spec_stats
            st["verify_steps"] += 1
            st["verify_sequence_steps"] += len(self.workset)
        self.commit([t[0] for t in tokens[:first]] + [0] * len(self.workset), t1, t2, logprobs, _speculative=True)
        for req, d in zip(self._first_committed, seq_drafts[:first]):
            req.drafts = d
        new_workset = self._first_workset
        for i, req in enumerate(self._running_committed):
            seq, drafted = first + i, len(req.drafts)
            kept = 0
            for j, t in enumerate(tokens[seq]):
                req.output.append(t)
                self._keep_logprobs(req, logprobs, rows[seq] + j)
                kept += 1
                if len(req.output) >= int(self.rs.output_lens[req.req_idx]) or t in self.stop_token_ids:
                    break
            st = self.spec_stats
            st["emitted_tokens"] += kept
            st["accepted_tokens"] += min(kept - 1, drafted) if kept else 0
            if S > 1:
                st["drafted_tokens"] += drafted
                st["verify_emitted_tokens"] += kept
            if not self._finishes(req):
                req.kvcache.truncate(req.kvcache.seqlen - S + kept)
            req.drafts = seq_drafts[seq]
            self._finish_or_continue(req, t2, new_workset)
        self.workset = new_workset
        return processed

    # ---- beam search
    def beam_rows(self) -> List[int]:
        """Beam search: the rows of last_token_rows() of each request that takes a beam step, as an indptr: one row per prompt
        this step completes, then the live beams of each running request (contiguous in the workset)."""
        counts = [1] * len(self._first())
        prev = None
        for r in self.workset:
            if r.group is prev:
                counts[-1] += 1
            else:
                counts.append(1)
                prev = r.group
        return np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int32).tolist()

    def beam_sums(self) -> List[float]:
        """Beam search: the running sum of every row of last_token_rows() (0 for a prompt's row)."""
        return [0.0] * len(self._first()) + [r.beam_sum for r in self.workset]

    def take_copies(self) -> List[tuple]:
        """Beam search: the (src page, dst page, slots) copies the next step must run before any K/V is written."""
        out, self.copies = self.copies, []
        return out

    def _offer(self, g: _BeamGroup, tokens: List[int], s) -> None:
        # the W best by score; a new hypothesis replaces the worst (the latest among equals) only if it is strictly better
        h = (float(s) / float(len(tokens)) ** self.beam.length_penalty, g.arrivals, tokens)
        g.arrivals += 1
        if len(g.finished) < self.beam.width:
            g.finished.append(h)
            return
        worst = min(range(len(g.finished)), key=lambda k: (g.finished[k][0], -g.finished[k][1]))
        if h[0] > g.finished[worst][0]:
            g.finished[worst] = h

    def commit_beam(self, live, live_key, fin, fin_key, t1: float, t2: float) -> int:
        """Beam search: ops.beam_select's result for the requests of beam_rows() (rows index last_token_rows()).  Offers the
        finished candidates, makes the live ones the request's beams -- the first child of a parent inherits its sequence, any
        further child is a fork whose partly filled page is copied by the next step (take_copies) -- and finishes the requests
        that are done.  Returns the number of tokens this step processed."""
        W = self.beam.width
        live, fin = np.asarray(live), np.asarray(fin)
        live_key, fin_key = np.asarray(live_key, np.float32), np.asarray(fin_key, np.float32)
        processed = sum(n for _, _, n in self._new) + len(self.workset)
        parents = []                                # per request: (group, its parent beams in row order)
        for p, s, n in self._new:
            p.done += n
            if p.start_at is None:
                p.start_at = t1
            if s + n == len(p.prompt):
                self._prefilling.remove(p)
                if p.req_idx >= 0:
                    g = _BeamGroup(p.req_idx, t2 - p.start_at, p.start_at)
                    parents.append((g, [RequestContext(p.req_idx, p.kvcache, [], group=g)]))
        for r in self.workset:
            if parents and parents[-1][0] is r.group:
                parents[-1][1].append(r)
            else:
                parents.append((r.group, [r]))
        row0 = np.asarray(self.beam_rows()[:-1])
        assert len(parents) == len(row0)
        new_workset: List[RequestContext] = []
        for i, (g, beams) in enumerate(parents):
            for (row, t), k in zip(fin[i], fin_key[i]):
                if row >= 0:
                    self._offer(g, beams[row - row0[i]].output + [int(t)], k)
            children = [(row - row0[i], int(t), np.float32(k)) for (row, t), k in zip(live[i], live_key[i]) if row >= 0]
            if len(g.finished) >= W or not children or len(beams[0].output) + 1 >= int(self.rs.output_lens[g.req_idx]):
                if len(g.finished) < W:
                    for b, t, k in children:
                        self._offer(g, beams[b].output + [t], k)
                for b in beams:
                    b.kvcache.release()
                self._finish_group(g, t2)
                continue
            kept = {b for b, _, _ in children}
            for b, beam in enumerate(beams):        # pages return before any are taken
                if b not in kept:
                    beam.kvcache.release()
            inherited = set()
            for b, t, k in children:
                parent = beams[b]
                if b in inherited:
                    before = len(self.copies)
                    kv = parent.kvcache.fork(copies=self.copies)
                    for _, _, slots in self.copies[before:]:
                        self.beam_stats["page_copies"] += 1
                        self.beam_stats["copied_slots"] += slots
                else:
                    kv = parent.kvcache
                    inherited.add(b)
                child = RequestContext(g.req_idx, kv, parent.output + [t], beam_sum=k, group=g)
                new_workset.append(child)
            for child in new_workset[len(new_workset) - len(children):]:
                child.kvcache.acquire_one()
        self.workset, self._new, self._admitted = new_workset, [], False
        return processed

    def _finish_group(self, g: _BeamGroup, t2: float) -> None:
        tokens, score = [], -np.inf
        if g.finished:
            score, _, tokens = max(g.finished, key=lambda h: (h[0], -h[1]))
        if tokens and tokens[-1] in self.stop_token_ids:
            self.beam_stats["stop_finished"] += 1
        req = RequestContext(g.req_idx, None, tokens, encode_latency=g.encode_latency, decode_start_at=g.decode_start_at,
                             decode_latency=t2 - g.decode_start_at, beam_sum=score)
        self.done.append(req)
        if self._root is not None and self.finished:
            self._root.kvcache.release()

    @staticmethod
    def _keep_logprobs(req, logprobs, row):
        if logprobs is not None:
            lp, ids, lps = logprobs
            req.logprobs.append(float(lp[row]))
            req.top_logprobs.append(([int(t) for t in ids[row]], [float(x) for x in lps[row]]))

    def _finishes(self, req) -> bool:
        return len(req.output) >= int(self.rs.output_lens[req.req_idx]) or req.output[-1] in self.stop_token_ids

    def _finish_or_continue(self, req, t2, new_workset):
        if self._finishes(req):
            req.decode_latency = t2 - req.decode_start_at
            req.kvcache.release()
            if req.slot >= 0:
                heapq.heappush(self._free_slots, req.slot)
            self.done.append(req)
            if self._root is not None and self.finished:
                self._root.kvcache.release()
        else:
            req.kvcache.acquire_one()
            new_workset.append(req)

    def result(self, duration: float, steps: int, keep_tokens: bool = False) -> TextGenBenchResult:
        done = sorted(self.done, key=lambda r: r.req_idx)
        res = TextGenBenchResult(np.array([r.encode_latency for r in done]), np.array([r.decode_latency for r in done]),
                                 duration, steps, [r.output for r in done] if keep_tokens else None)
        res.output_lens = np.array([len(r.output) for r in done], dtype=np.int32)
        if self.beam is not None:
            res.beam_scores = np.array([r.beam_sum for r in done], dtype=np.float64)
            res.beam = dict(self.beam_stats)
        if keep_tokens and any(r.logprobs for r in done):
            res.logprobs = [r.logprobs for r in done]
            res.top_logprobs = [r.top_logprobs for r in done]
        return res


class _StaticKv:
    """The attributes the KV ops read (kvcache.BatchedKvCacheInt4), backed by fixed device buffers."""

    def __init__(self, pool, indptr, indicies, last_page_offset):
        self.data, self.param = pool.buf, pool.param
        self.indptr, self.indicies, self.last_page_offset = indptr, indicies, last_page_offset

    @property
    def page_size(self):
        return self.data.size(-2)


class DecodeGraphRunner:
    """Decode-only steps replayed from CUDA graphs, one graph per (batch size, number of prefix groups).

    In steady state almost every step of the serving loop is decode-only (outputs are ~50x longer than prompts in the
    reference's request set) and a 32-layer step is ~500 kernel launches: launch-bound from Python.  All per-step state of
    such a step is a handful of integers -- the input token of each sequence and the page table -- so they live in ONE
    fixed int32 device buffer  [ids(B) | indptr(B+1) | last_page_offset(B) | indicies(B * max_pages)]  that is refreshed
    with a single pinned H2D copy, after which the captured step (embedding, all layers: fused norm+quantise, INT4 GEMMs,
    KV append, INT4 decode attention, lm_head, argmax) is replayed.  The kernels read the page table from device memory and
    their grids depend only on B, so the graph stays valid as sequences grow and change pages.
    A batch of forked sequences (shared_prefix) has prefix groups (kvcache.prefix_groups); with G > 0 of them the buffer goes on
    with  [group_indptr(G+1) | group_members(B) | shared_pages(B)]  and the graph's shared-prefix decode is sized from bounds
    that hold under the key -- at most B members in a group, at most max_pages shared pages -- so it stays valid as members join
    or leave a group and as lengths grow.  Without groups the buffer is exactly the layout above.

    With `sampling` (SamplingParams) the step samples instead of taking the argmax, and the buffer goes on, from the next even
    offset (8-byte aligned: the buffer's base is), with  [keys(2B x u64) | counters(B x u64) | top_k(B) | T(B) | top_p(B)],
    T and top_p as FP32 bit patterns -- still one H2D copy.  `sample_op` (ops.sample_tokens' signature) is the sampler the
    step calls; host-only tests substitute a reference.  Without sampling the buffer is exactly the layout above.
    When the SamplingParams have penalties, min-p or logprobs (`extended`), it goes on with  [slots(B) | min_p(B) | rep(B) |
    freq(B) | pres(B)]  (FP32 bit patterns), the step also passes `penalty_table` (set by run_textgen) and, with logprobs, returns
    (tokens, logprob, top_ids, top_logprobs).  Otherwise the buffer and the step are exactly the above.

    With `speculate` (SpeculativeParams) every step -- graphs keyed on (B, prefix groups, S) -- carries S rows per sequence and
    ends with the draft sampler (`draft_sample_op`, ops.sample_tokens with drafts; at T = 0 when greedy) and the commit and
    proposal (`propose_op`, ops.spec_commit_propose) on the token histories set by use_history().  Its buffer is
    [ids(BS) | indptr(B+1) | last_page_offset(B) | indicies(B * max_pages) | groups (S = 1 only) | candidates(BS) |
    row_indptr(B+1) | history slots(B) | keys(2BS x u64) | counters(BS x u64) | top_k(BS) | T(BS) | top_p(BS) | min_p(BS)], one
    H2D copy; a verify step (S > 1) passes BatchLenInfo(decode_len=S, max_len=max_pages * page size) and no groups.  The step
    returns the proposer's output [B, 2K + 3] (and, with logprobs, the sampler's per-row log-probabilities).

    With `beam` (BeamSearchParams) the graphs are keyed on (B rows, prefix groups) and the buffer goes on after the page table
    and groups with  [copy src(B) | copy dst(B) | copy slots(B) | row_indptr(B+1) | sums(B, FP32 bits)], one H2D copy; the
    step is `copy_op` (ops.copy_kv_pages: the page copies of the previous commit's forks, padded with src = -1), the model, then
    `beam_select_op` (ops.beam_select at the runner's width and stop ids) into one packed buffer, read back with one D2H copy.

    capture=False runs the same buffers through the model eagerly (the CPU tests use it; it is also the warm-up path)."""

    def __init__(self, model: Callable, pool: KvPoolInt4, device, max_pages_per_seq: int, capture: bool = True,
                 sampling: Optional[SamplingParams] = None, sample_op: Callable = None,
                 speculate: Optional[SpeculativeParams] = None, propose_op: Callable = None, draft_sample_op: Callable = None,
                 beam: Optional[BeamSearchParams] = None, stop_token_ids=(), beam_select_op: Callable = None,
                 copy_op: Callable = None):
        self.model, self.pool, self.device = model, pool, torch.device(device)
        self.max_pages, self.capture = max_pages_per_seq, capture
        self.sampling = sampling
        if sample_op is None and sampling is not None:
            from . import ops
            sample_op = ops.sample_tokens
        self.sample_op = sample_op
        self.penalty_table = None
        self._entries = {}
        self.speculate = speculate
        self.history = None
        if speculate is not None:
            if sampling is not None and sampling.penalties:
                raise ValueError("speculative decoding cannot be combined with penalties")
            if propose_op is None or draft_sample_op is None:
                from . import ops
            self.propose_op = propose_op or ops.spec_commit_propose
            self.draft_sample_op = draft_sample_op or ops.sample_tokens
        self.beam, self.stop_token_ids = beam, tuple(int(t) for t in stop_token_ids)
        if beam is not None:
            if beam_select_op is None or copy_op is None:
                from . import ops
            self.beam_select_op = beam_select_op or ops.beam_select
            self.copy_op = copy_op or ops.copy_kv_pages

    def use_history(self, history):
        """The (token histories, lengths) the speculative step commits to and proposes from; graphs captured with others are
        dropped."""
        if self.history is None or history[0] is not self.history[0] or history[1] is not self.history[1]:
            self.history = history
            self._entries = {}

    def use_table(self, table):
        """The penalty table the sampling step reads and updates; graphs captured with another one are dropped."""
        if table is not self.penalty_table:
            self.penalty_table = table
            self._entries = {}

    def _layout(self, b, ng=0):
        o_ids, o_indptr, o_last, o_ind = 0, b, 2 * b + 1, 3 * b + 1
        o_grp = 3 * b + 1 + b * self.max_pages
        return o_ids, o_indptr, o_last, o_ind, o_grp, o_grp + (ng + 1 + 2 * b if ng else 0)

    def _sampling_layout(self, b, ng=0):
        """int32 offsets of keys, counters, top_k, T, top_p and the buffer's total size, when sampling."""
        o_key = (self._layout(b, ng)[-1] + 1) // 2 * 2
        o_ctr = o_key + 4 * b
        o_k = o_ctr + 2 * b
        return o_key, o_ctr, o_k, o_k + b, o_k + 2 * b, o_k + 3 * b

    def _ext_layout(self, b, ng=0):
        """int32 offsets of slots, min_p, rep, freq, pres and the buffer's total size, with extended sampling."""
        o = self._sampling_layout(b, ng)[-1]
        return tuple(o + i * b for i in range(6))

    def _entry(self, b, ng):
        e = self._entries.get((b, ng))
        if e is None:
            o_ids, o_indptr, o_last, o_ind, o_grp, total = self._layout(b, ng)
            if self.sampling is not None:
                total = self._sampling_layout(b, ng)[-1]
                if self.sampling.extended:
                    total = self._ext_layout(b, ng)[-1]
            host = torch.zeros(total, dtype=torch.int32)
            if self.device.type == "cuda":
                host = host.pin_memory()
            dev = torch.zeros(total, dtype=torch.int32, device=self.device)
            kv = _StaticKv(self.pool, dev[o_indptr:o_indptr + b + 1], dev[o_ind:o_ind + b * self.max_pages], dev[o_last:o_last + b])
            if ng:
                kv.group_indptr = dev[o_grp:o_grp + ng + 1]
                kv.group_members = dev[o_grp + ng + 1:o_grp + ng + 1 + b]
                kv.shared_pages = dev[o_grp + ng + 1 + b:o_grp + ng + 1 + 2 * b]
                kv.group_bounds = (b, self.max_pages)
            e = {"host": host, "dev": dev, "ids": dev[o_ids:o_ids + b], "kv": kv, "blen": BatchLenInfo([], b, self.device),
                 "graph": None, "out": None}
            if self.sampling is not None:
                o_key, o_ctr, o_k, o_t, o_p, _ = self._sampling_layout(b, ng)
                e["sample"] = (dev[o_t:o_t + b].view(torch.float32), dev[o_k:o_k + b], dev[o_p:o_p + b].view(torch.float32),
                               dev[o_key:o_ctr].view(torch.int64).view(b, 2), dev[o_ctr:o_k].view(torch.int64))
                if self.sampling.extended:
                    sp = self.sampling
                    o_sl, o_m, o_r, o_f, o_q, _ = self._ext_layout(b, ng)
                    f32 = lambda o: dev[o:o + b].view(torch.float32)      # noqa: E731
                    ext = {"min_p": f32(o_m)} if sp.min_p != 0 else {}
                    if sp.penalties:
                        ext.update(repetition_penalty=f32(o_r), frequency_penalty=f32(o_f), presence_penalty=f32(o_q),
                                   penalty_table=self.penalty_table, slots=dev[o_sl:o_sl + b])
                    if sp.logprobs is not None:
                        ext["logprobs"] = int(sp.logprobs)
                    e["ext"] = ext
            self._entries[(b, ng)] = e
        return e

    def _step(self, e):
        logits, _ = self.model(e["ids"], e["blen"], None, e["kv"])
        if self.sampling is not None:
            return self.sample_op(logits, *e["sample"], **e.get("ext", {}))
        return torch.argmax(logits, dim=-1)

    def run(self, last_tokens: List[int], kvs: List[KvCacheInt4], slots: Optional[List[tuple]] = None,
            row_slots: Optional[List[int]] = None):
        """slots: (request index, counter) per sequence, needed with sampling (TextGenScheduler.sample_slots); row_slots: the
        penalty-table slot per sequence, needed with penalties (TextGenScheduler.row_slots).  Returns the tokens, or with
        logprobs (tokens, logprob, top_ids, top_logprobs), as numpy arrays."""
        b = len(kvs)
        groups = prefix_groups(kvs)
        ng = len(groups)
        e = self._entry(b, ng)
        o_ids, o_indptr, o_last, o_ind, o_grp, _ = self._layout(b, ng)
        h = e["host"].numpy()
        h[o_ids:o_ids + b] = last_tokens
        self._fill_pages(h, kvs, o_indptr, o_last, o_ind)
        self._fill_groups(h, e, groups, b, o_grp)
        if self.sampling is not None:
            o_key, o_ctr, o_k, o_t, o_p, _ = self._sampling_layout(b, ng)
            sp = self.sampling
            self._fill_draw(h, sp, slots, o_key, o_ctr, o_k, o_t, o_p, b)
            if sp.extended:
                o_sl, o_m, o_r, o_f, o_q, _ = self._ext_layout(b, ng)
                h[o_sl:o_m] = row_slots if sp.penalties else -1
                for o, v in ((o_m, sp.min_p), (o_r, sp.repetition_penalty), (o_f, sp.frequency_penalty), (o_q, sp.presence_penalty)):
                    h[o:o + b] = np.float32(v).view(np.int32)
        return self._launch(e, self._step)

    def _fill_pages(self, h, kvs, o_indptr, o_last, o_ind):
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

    @staticmethod
    def _fill_groups(h, e, groups, b, o_grp):
        ng = len(groups)
        if ng:
            members = [r for rows, _ in groups for r in rows]
            h[o_grp:o_grp + ng + 1] = np.cumsum([0] + [len(rows) for rows, _ in groups])
            h[o_grp + ng + 1:o_grp + ng + 1 + b] = members + [0] * (b - len(members))
            shared = h[o_grp + ng + 1 + b:o_grp + ng + 1 + 2 * b]
            shared[:] = 0
            for rows, n in groups:
                shared[rows] = n
            e["kv"].groups = groups              # the host view: it decides, when the step is captured, which decode runs

    @staticmethod
    def _fill_draw(h, sp, slots, o_key, o_ctr, o_k, o_t, o_p, n):
        words = np.array([w for r, _ in slots for w in (int(sp.seed), r)], dtype=np.uint64)
        h[o_key:o_ctr] = words.view(np.int32)
        h[o_ctr:o_k] = np.array([c for _, c in slots], dtype=np.uint64).view(np.int32)
        h[o_k:o_t] = int(sp.top_k)
        h[o_t:o_p] = np.float32(sp.temperature).view(np.int32)
        h[o_p:o_p + n] = np.float32(sp.top_p).view(np.int32)

    def _launch(self, e, step):
        e["dev"].copy_(e["host"], non_blocking=True)
        if not self.capture:
            return _to_numpy(step(e))
        if e["graph"] is None:
            side = torch.cuda.Stream(self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):
                table = self.penalty_table if self.sampling is not None and self.sampling.penalties else None
                state = ([table] if table is not None else []) + (list(self.history) if self.speculate is not None else [])
                saved = [t.clone() for t in state]
                step(e)                             # warm-up on real data (lazy initialisations must not be captured)
                for t, v in zip(state, saved):
                    t.copy_(v)                      # the warm-up's draw was recorded: the replay below is the step's draw
                side.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=side):
                    e["out"] = step(e)
            torch.cuda.current_stream(self.device).wait_stream(side)
            e["graph"] = g
        e["graph"].replay()
        return _to_numpy(e["out"])                  # synchronises: the caller needs the tokens to go on

    # ---- speculative steps
    def _spec_layout(self, b, ng, S):
        """int32 offsets: ids, indptr, last, indicies, groups, candidates, row_indptr, history slots, keys, counters, top_k, T,
        top_p, min_p and the total."""
        R = b * S
        o_ind = R + 2 * b + 1
        o_grp = o_ind + b * self.max_pages
        o_cand = o_grp + (ng + 1 + 2 * b if ng else 0)
        o_rip = o_cand + R
        o_hs = o_rip + b + 1
        o_key = (o_hs + b + 1) // 2 * 2
        o_ctr = o_key + 4 * R
        o_k = o_ctr + 2 * R
        return {"ids": 0, "indptr": R, "last": R + b + 1, "ind": o_ind, "grp": o_grp, "cand": o_cand, "rip": o_rip, "hs": o_hs,
                "key": o_key, "ctr": o_ctr, "k": o_k, "t": o_k + R, "p": o_k + 2 * R, "m": o_k + 3 * R, "total": o_k + 4 * R}

    def _spec_entry(self, b, ng, S):
        e = self._entries.get((b, ng, S))
        if e is None:
            o, R = self._spec_layout(b, ng, S), b * S
            host = torch.zeros(o["total"], dtype=torch.int32)
            if self.device.type == "cuda":
                host = host.pin_memory()
            dev = torch.zeros(o["total"], dtype=torch.int32, device=self.device)
            kv = _StaticKv(self.pool, dev[o["indptr"]:o["indptr"] + b + 1], dev[o["ind"]:o["ind"] + b * self.max_pages],
                           dev[o["last"]:o["last"] + b])
            g = o["grp"]
            if ng:
                kv.group_indptr = dev[g:g + ng + 1]
                kv.group_members = dev[g + ng + 1:g + ng + 1 + b]
                kv.shared_pages = dev[g + ng + 1 + b:g + ng + 1 + 2 * b]
                kv.group_bounds = (b, self.max_pages)
            blen = BatchLenInfo([], b, self.device) if S == 1 else \
                BatchLenInfo([], b, self.device, decode_len=S, max_len=self.max_pages * self.pool.block_len)
            f32 = lambda x: dev[o[x]:o[x] + R].view(torch.float32)      # noqa: E731
            sp = self.sampling
            ext = {}
            if sp is not None and sp.min_p != 0:
                ext["min_p"] = f32("m")
            if sp is not None and sp.logprobs is not None:
                ext["logprobs"] = int(sp.logprobs)
            K = self.speculate.num_draft
            e = {"host": host, "dev": dev, "ids": dev[:R], "kv": kv, "blen": blen, "graph": None, "out": None, "ext": ext,
                 "sample": (f32("t"), dev[o["k"]:o["k"] + R], f32("p"), dev[o["key"]:o["ctr"]].view(torch.int64).view(R, 2),
                            dev[o["ctr"]:o["k"]].view(torch.int64)),
                 "cands": dev[o["cand"]:o["cand"] + R], "rip": dev[o["rip"]:o["rip"] + b + 1], "hs": dev[o["hs"]:o["hs"] + b],
                 "spec_out": torch.zeros((b, 2 * K + 3), dtype=torch.int32, device=self.device)}
            self._entries[(b, ng, S)] = e
        return e

    def _spec_step(self, e):
        logits, _ = self.model(e["ids"], e["blen"], None, e["kv"])
        out = self.draft_sample_op(logits, *e["sample"], drafts=e["cands"], **e["ext"])
        tokens = out[0] if isinstance(out, tuple) else out
        sp = self.speculate
        self.propose_op(tokens, e["cands"], e["rip"], e["hs"], self.history[0], self.history[1], e["spec_out"], sp.num_draft,
                        sp.ngram_min, sp.ngram_max)
        return (e["spec_out"],) + tuple(out[1:]) if isinstance(out, tuple) else e["spec_out"]

    def run_spec(self, S: int, ids: List[int], cands: List[int], kvs: List[KvCacheInt4], slots: List[tuple], hist_slots: List[int]):
        """A speculative step of S rows per sequence (TextGenScheduler: S, decode_ids, candidates, sample_slots, sequence_slots;
        the sequences' pages already hold the S rows).  Returns the proposer's output [B, 2K + 3] (with logprobs, and then the
        sampler's logprob, top_ids, top_logprobs per row), as numpy arrays."""
        b = len(kvs)
        groups = prefix_groups(kvs) if S == 1 else []
        ng = len(groups)
        e = self._spec_entry(b, ng, S)
        o, R = self._spec_layout(b, ng, S), b * S
        h = e["host"].numpy()
        h[:R] = ids
        self._fill_pages(h, kvs, o["indptr"], o["last"], o["ind"])
        self._fill_groups(h, e, groups, b, o["grp"])
        h[o["cand"]:o["cand"] + R] = cands
        h[o["rip"]:o["rip"] + b + 1] = np.arange(0, R + 1, S)
        h[o["hs"]:o["hs"] + b] = hist_slots
        sp = self.sampling if self.sampling is not None else SamplingParams(0.0)
        self._fill_draw(h, sp, slots, o["key"], o["ctr"], o["k"], o["t"], o["p"], R)
        h[o["m"]:o["m"] + R] = np.float32(sp.min_p).view(np.int32)
        return self._launch(e, self._spec_step)


    # ---- beam steps
    def _beam_layout(self, b, ng):
        o = self._layout(b, ng)[-1]
        return {"src": o, "dst": o + b, "slots": o + 2 * b, "rip": o + 3 * b, "sums": o + 4 * b + 1, "total": o + 5 * b + 1}

    def _beam_entry(self, b, ng):
        e = self._entries.get(("beam", b, ng))
        if e is None:
            o_ids, o_indptr, o_last, o_ind, o_grp, _ = self._layout(b, ng)
            o = self._beam_layout(b, ng)
            host = torch.zeros(o["total"], dtype=torch.int32)
            if self.device.type == "cuda":
                host = host.pin_memory()
            dev = torch.zeros(o["total"], dtype=torch.int32, device=self.device)
            kv = _StaticKv(self.pool, dev[o_indptr:o_indptr + b + 1], dev[o_ind:o_ind + b * self.max_pages], dev[o_last:o_last + b])
            if ng:
                kv.group_indptr = dev[o_grp:o_grp + ng + 1]
                kv.group_members = dev[o_grp + ng + 1:o_grp + ng + 1 + b]
                kv.shared_pages = dev[o_grp + ng + 1 + b:o_grp + ng + 1 + 2 * b]
                kv.group_bounds = (b, self.max_pages)
            W = self.beam.width
            e = {"host": host, "dev": dev, "ids": dev[o_ids:o_ids + b], "kv": kv, "blen": BatchLenInfo([], b, self.device),
                 "graph": None, "out": None, "copy": tuple(dev[o[k]:o[k] + b] for k in ("src", "dst", "slots")),
                 "rip": dev[o["rip"]:o["rip"] + b + 1], "sums": dev[o["sums"]:o["sums"] + b].view(torch.float32),
                 "bout": torch.zeros(6 * b * W, dtype=torch.int32, device=self.device),
                 "ws": torch.zeros(b * 16 * 12, dtype=torch.uint8, device=self.device)}
            self._entries[("beam", b, ng)] = e
        return e

    def _beam_step(self, e):
        self.copy_op(self.pool, *e["copy"])
        logits, _ = self.model(e["ids"], e["blen"], None, e["kv"])
        self.beam_select_op(logits, e["rip"], e["sums"], self.beam.width, self.stop_token_ids, out=e["bout"], workspace=e["ws"])
        return e["bout"]

    def run_beam(self, last_tokens: List[int], kvs: List[KvCacheInt4], copies: List[tuple], row_indptr: List[int],
                 sums: List[float]):
        """A beam step over B rows (TextGenScheduler: take_copies, beam_rows, beam_sums).  Returns (live, live_key, fin, fin_key)
        of the requests of row_indptr, as numpy arrays."""
        b = len(kvs)
        groups = prefix_groups(kvs)
        ng = len(groups)
        if len(copies) > b:
            raise RuntimeError(f"{len(copies)} page copies for a step of {b} rows")
        for src, dst, slots in copies:                  # the kernel skips such pairs: a scheduler fault must not pass silently
            if src == dst or not (0 <= src < self.pool.capacity and 0 <= dst < self.pool.capacity and 1 <= slots <= self.pool.block_len):
                raise RuntimeError(f"page copy ({src}, {dst}, {slots}) needs src != dst, pages in range and slots in [1, page size]")
        e = self._beam_entry(b, ng)
        o_ids, o_indptr, o_last, o_ind, o_grp, _ = self._layout(b, ng)
        o = self._beam_layout(b, ng)
        h = e["host"].numpy()
        h[o_ids:o_ids + b] = last_tokens
        self._fill_pages(h, kvs, o_indptr, o_last, o_ind)
        self._fill_groups(h, e, groups, b, o_grp)
        n = len(copies)
        for k, name in enumerate(("src", "dst", "slots")):
            h[o[name]:o[name] + b] = [c[k] for c in copies] + [-1] * (b - n)
        nreq = len(row_indptr) - 1
        h[o["rip"]:o["rip"] + b + 1] = list(row_indptr) + [row_indptr[-1]] * (b - nreq)
        h[o["sums"]:o["sums"] + b] = np.asarray(sums, np.float32).view(np.int32)
        out = self._launch(e, self._beam_step)
        from .ops import split_beam_out
        return tuple(x[:nreq] for x in split_beam_out(out, b, self.beam.width))


def _to_numpy(out):
    return tuple(x.cpu().numpy() for x in out) if isinstance(out, tuple) else out.cpu().numpy()


def _vocab_size(model) -> int:
    """Prompt ids must index the model's own embedding table (the reference hard-codes 32000, bench_textgen.py:119)."""
    head = getattr(model, "lm_head", None)
    if head is not None and hasattr(head, "out_features"):
        return int(head.out_features)
    cfg = getattr(model, "config", None) or getattr(getattr(model, "model", None), "config", None)
    return int(getattr(cfg, "vocab_size", 32000))


def pool_capacity(batch_size: int, maxlen: int, block_len: int, num_draft: int = 0) -> int:
    """Pages for `batch_size` sequences of up to `maxlen` tokens (+1 spare page each), bench_textgen.py:99.  With num_draft = K
    (speculative decoding) each sequence also gets the pages of K + 1 more tokens: a verify step grows a sequence by up to K
    tokens past its length and the commit by one more, so every request can reach its full length without waiting for a page
    in the middle of a step."""
    return batch_size * ((maxlen + block_len - 1) // block_len + 1 + (-(-(num_draft + 1) // block_len) if num_draft else 0))


@torch.inference_mode()
def run_textgen(model: Callable, rs: RequestSet, cfg: TextGenConfig, pool: KvPoolInt4, device, sync: Callable = None,
                keep_tokens: bool = False, progress: Callable = None, decode_runner: DecodeGraphRunner = None,
                sample_op: Callable = None, slot_init_op: Callable = None, propose_op: Callable = None,
                draft_sample_op: Callable = None, beam_select_op: Callable = None, copy_op: Callable = None) -> TextGenBenchResult:
    """Drive `model(input_ids, blen, prefill_kv, decode_kv) -> (logits, hidden)` through the whole request set.
    Latencies are wall-clock around the step *including* the device->host read of the next tokens (which synchronises),
    as in the reference.  With a `decode_runner`, steps that carry no prompt tokens are replayed from its CUDA graphs.
    cfg.prefill_chunk, cfg.shared_prefix: see TextGenScheduler.  cfg.sampling: the eager steps call `sample_op` (default
    ops.sample_tokens) on the rows whose logits are needed, with each row's key (seed, request) and counter; the runner, which
    must have been built with the same SamplingParams, samples in its graphs.  With penalties a penalty table of
    cfg.batch_size slots is made on `device` (ops.penalty_table) and each admitted request's slot is set up by `slot_init_op`
    (default ops.init_penalty_slot) before its first token; the runner is given the same table.  cfg.stop_token_ids: see
    TextGenScheduler.
    cfg.speculate: token histories of cfg.batch_size slots (ops.spec_history) hold each request's context, set up at admission
    (ops.spec_init_slot); every step samples with `draft_sample_op` (default ops.sample_tokens with drafts, at T = 0 when
    greedy) and then commits and proposes with `propose_op` (default ops.spec_commit_propose); the runner must have been built
    with the same SpeculativeParams and is given the same histories.  Not with penalties.
    cfg.beam: every request keeps up to W beams (TextGenScheduler.commit_beam); each step first runs the page copies of the
    previous step's forks with `copy_op` (default ops.copy_kv_pages), then the model, then `beam_select_op` (default
    ops.beam_select) on the rows of every request's beams; the runner must have been built with the same BeamSearchParams and
    stop ids.  The result's tokens are each request's best hypothesis, beam_scores their scores.  Not with sampling or
    speculation, and cfg.batch_size (rows) must hold W."""
    sp = cfg.sampling
    if sp is not None and sample_op is None:
        from . import ops
        sample_op = ops.sample_tokens
    if decode_runner is not None and decode_runner.sampling != sp:
        raise ValueError("decode_runner was built for other sampling parameters than cfg.sampling")
    spec = cfg.speculate
    if spec is not None and sp is not None and sp.penalties:
        raise ValueError("speculative decoding cannot be combined with penalties")
    if decode_runner is not None and decode_runner.speculate != spec:
        raise ValueError("decode_runner was built for other speculative parameters than cfg.speculate")
    beam = cfg.beam
    if beam is not None:
        if sp is not None or spec is not None:
            raise ValueError("beam search cannot be combined with sampling, penalties or speculative decoding")
        if cfg.batch_size < beam.width:
            raise ValueError(f"batch_size={cfg.batch_size} rows cannot hold a request of {beam.width} beams")
        if decode_runner is not None and (decode_runner.beam != beam or
                                          decode_runner.stop_token_ids != tuple(int(t) for t in cfg.stop_token_ids)):
            raise ValueError("decode_runner was built for other beam parameters or stop ids than cfg")
        if beam_select_op is None or copy_op is None:
            from . import ops
        beam_select_op = beam_select_op or ops.beam_select
        copy_op = copy_op or ops.copy_kv_pages
    elif decode_runner is not None and decode_runner.beam is not None:
        raise ValueError("decode_runner was built for beam search and cfg.beam is None")
    vocab = _vocab_size(model)
    table = None
    if sp is not None and sp.penalties:
        from . import ops
        table = ops.penalty_table(cfg.batch_size, vocab, device)
        old = None if decode_runner is None else decode_runner.penalty_table
        if old is not None and old.shape == table.shape and old.device == table.device:
            table = old                     # its graphs stay valid; every slot is set up again at admission
        if slot_init_op is None:
            slot_init_op = ops.init_penalty_slot
        if decode_runner is not None:
            decode_runner.use_table(table)
    hist = None
    if spec is not None:
        from . import ops
        propose_op = propose_op or ops.spec_commit_propose
        draft_sample_op = draft_sample_op or ops.sample_tokens
        # every token a request's history can hold: its context, its output and the drafts a last step may commit past it
        cap = cfg.shared_prefix + int(rs.prompt_lens.max()) + int(rs.output_lens.max()) + spec.num_draft + 1
        old = None if decode_runner is None else decode_runner.history
        if old is not None and old[0].size(0) == cfg.batch_size and old[0].size(1) >= cap and \
                old[0].device == torch.empty(0, device=device).device:
            hist = old                      # its graphs stay valid; every slot is set up again at admission
        else:
            hist = ops.spec_history(cfg.batch_size, cap, device)
        if decode_runner is not None:
            decode_runner.use_history(hist)
    gsp = sp if sp is not None else SamplingParams(0.0)     # speculating, greedy is the draft sampler at T = 0
    sched = TextGenScheduler(rs, cfg.batch_size, pool, device, vocab_size=vocab, prefill_chunk=cfg.prefill_chunk,
                             shared_prefix=cfg.shared_prefix, stop_token_ids=cfg.stop_token_ids,
                             penalty_slots=table is not None or spec is not None, num_draft=0 if spec is None else spec.num_draft,
                             beam=beam)
    steps = graphed = peak = 0
    t_start = time.perf_counter()
    while not sched.finished:
        sched.admit()
        for slot, prompt in sched.slot_inits:
            if table is not None:
                slot_init_op(table, slot, prompt)
            if hist is not None:
                ops.spec_init_slot(hist[0], hist[1], slot, prompt)
        sched.slot_inits.clear()
        peak = max(peak, pool.capacity - pool.num_free_blocks)
        t1 = time.perf_counter()
        logprobs = None
        if beam is not None:
            copies = sched.take_copies()
            if decode_runner is not None and sched.prompt_tokens == 0:
                next_tokens = decode_runner.run_beam([int(r.output[-1]) for r in sched.workset], [r.kvcache for r in sched.workset],
                                                     copies, sched.beam_rows(), sched.beam_sums())
                graphed += 1
            else:
                if copies:
                    copy_op(pool, *([c[k] for c in copies] for k in range(3)))
                batch = sched.next_batch()
                ids = torch.tensor(batch.input_ids, dtype=torch.long, device=device)
                logits, _ = model(ids, batch.blen, batch.prefill_kv, batch.decode_kv)
                rows = torch.tensor(sched.last_token_rows(), dtype=torch.long, device=logits.device)
                rip = torch.tensor(sched.beam_rows(), dtype=torch.int32, device=logits.device)
                next_tokens = ([], [], [], [])
                if len(rip) > 1:                    # (a step of prompt chunks alone takes no beam step)
                    sums = torch.tensor(sched.beam_sums(), dtype=torch.float32, device=logits.device)
                    next_tokens = _to_numpy(tuple(beam_select_op(logits.index_select(0, rows), rip, sums, beam.width,
                                                                 cfg.stop_token_ids)))
        elif spec is not None and decode_runner is not None and sched.prompt_tokens == 0:
            out = decode_runner.run_spec(sched.S, sched.decode_ids(), sched.candidates(), [r.kvcache for r in sched.workset],
                                         sched.sample_slots(), sched.sequence_slots())
            next_tokens, logprobs = (out[0], out[1:]) if isinstance(out, tuple) else (out, None)
            graphed += 1
        elif spec is not None:
            batch = sched.next_batch()
            ids = torch.tensor(batch.input_ids, dtype=torch.long, device=device)
            logits, _ = model(ids, batch.blen, batch.prefill_kv, batch.decode_kv)
            rows = torch.tensor(sched.last_token_rows(), dtype=torch.long, device=logits.device)
            slots = sched.sample_slots()
            n = len(slots)
            i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=logits.device)      # noqa: E731
            cands = i32(sched.candidates())
            opts = {} if gsp.min_p == 0 else {"min_p": [gsp.min_p] * n}
            if gsp.logprobs is not None:
                opts["logprobs"] = int(gsp.logprobs)
            out = draft_sample_op(logits.index_select(0, rows), [gsp.temperature] * n, [gsp.top_k] * n, [gsp.top_p] * n,
                                  [(int(gsp.seed), r) for r, _ in slots], [c for _, c in slots], drafts=cands, **opts)
            res_out = torch.empty((len(sched.sequence_slots()), 2 * spec.num_draft + 3), dtype=torch.int32, device=logits.device)
            if len(res_out):                        # (a step of prompt chunks alone draws nothing)
                propose_op(out[0] if isinstance(out, tuple) else out, cands, i32(sched.sequence_rows()), i32(sched.sequence_slots()),
                           hist[0], hist[1], res_out, spec.num_draft, spec.ngram_min, spec.ngram_max)
            next_tokens = res_out.cpu().numpy()
            if isinstance(out, tuple):
                logprobs = _to_numpy(out[1:])
        elif decode_runner is not None and sched.prompt_tokens == 0:
            next_tokens = decode_runner.run([int(r.output[-1]) for r in sched.workset], [r.kvcache for r in sched.workset],
                                            sched.sample_slots() if sp is not None else None,
                                            sched.row_slots() if table is not None else None)
            if isinstance(next_tokens, tuple):
                next_tokens, logprobs = next_tokens[0], next_tokens[1:]
            graphed += 1
        else:
            batch = sched.next_batch()
            ids = torch.tensor(batch.input_ids, dtype=torch.long, device=device)
            logits, _ = model(ids, batch.blen, batch.prefill_kv, batch.decode_kv)
            rows = torch.tensor(sched.last_token_rows(), dtype=torch.long, device=logits.device)
            if sp is None:
                next_tokens = torch.argmax(logits.index_select(0, rows), dim=-1).cpu().numpy()
            else:
                slots = sched.sample_slots()
                n = len(slots)
                args = (logits.index_select(0, rows), [sp.temperature] * n, [sp.top_k] * n, [sp.top_p] * n,
                        [(int(sp.seed), r) for r, _ in slots], [c for _, c in slots])
                if not sp.extended:
                    next_tokens = sample_op(*args).cpu().numpy()
                else:
                    out = _to_numpy(sample_op(*args, **sp.options(n, table, sched.row_slots())))
                    next_tokens, logprobs = (out[0], out[1:]) if isinstance(out, tuple) else (out, None)
        if sync is not None:
            sync()
        t2 = time.perf_counter()
        if beam is not None:
            n = sched.commit_beam(*next_tokens, t1, t2)
        elif spec is not None:
            n = sched.commit_spec(next_tokens, t1, t2, logprobs)
        else:
            n = sched.commit(next_tokens, t1, t2) if logprobs is None else sched.commit(next_tokens, t1, t2, logprobs)
        steps += 1
        if progress is not None:
            progress(n)
    res = sched.result(time.perf_counter() - t_start, steps, keep_tokens)
    res.graphed_steps = graphed
    res.peak_pages = peak
    if spec is not None:
        res.speculative = dict(sched.spec_stats)
    if beam is not None:                    # a copied slot is 64 bytes of pool.buf and 4 of pool.param per (layer, K|V, head)
        res.beam["bytes_copied"] = res.beam["copied_slots"] * pool.num_layers * 2 * pool.buf.shape[3] * 68
    return res


def report(rs: RequestSet, cfg: TextGenConfig, res: TextGenBenchResult) -> dict:
    """The figures bench_textgen.py:509-528 prints, as a dict (throughput = (prompt + new tokens) / duration; the shared system
    prompt's tokens are not counted), plus the peak of KV pages in use.  New tokens are those each request generated: the
    request set's output lengths, unless a stop id ended a request early."""
    gen = rs.output_lens if res.output_lens is None else res.output_lens
    per_prompt_tok = res.encode_latency / rs.prompt_lens
    per_new_tok = res.decode_latency / gen
    total = int(rs.prompt_lens.sum()) + int(gen.sum())
    out = {
        "num_requests": len(rs), "batch_size": cfg.batch_size, "steps": res.steps, "graphed_decode_steps": res.graphed_steps,
        "encode_latency_ms_per_request": [float(res.encode_latency.mean() * 1e3), float(res.encode_latency.std() * 1e3)],
        "encode_latency_ms_per_token": [float(per_prompt_tok.mean() * 1e3), float(per_prompt_tok.std() * 1e3)],
        "decode_latency_ms_per_token": [float(per_new_tok.mean() * 1e3), float(per_new_tok.std() * 1e3)],
        "total_prompt_tokens": int(rs.prompt_lens.sum()), "total_new_tokens": int(gen.sum()),
        "duration_s": res.duration, "throughput_tokens_per_s": total / res.duration, "peak_kv_pages_in_use": res.peak_pages,
        "shared_prefix": cfg.shared_prefix,
        "sampling": None if cfg.sampling is None else cfg.sampling.asdict(),
    }
    if cfg.stop_token_ids:
        out["stop_token_ids"] = [int(t) for t in cfg.stop_token_ids]
    if cfg.beam is not None and res.beam is not None:
        st = res.beam
        out["beam"] = {"width": cfg.beam.width, "length_penalty": cfg.beam.length_penalty, "page_copies": st["page_copies"],
                       "page_copies_per_step": st["page_copies"] / res.steps if res.steps else 0.0,
                       "bytes_copied": st["bytes_copied"], "stop_finished_requests": st["stop_finished"]}
    if cfg.speculate is not None and res.speculative is not None:
        st, sp = res.speculative, cfg.speculate
        out["speculative"] = {
            "num_draft": sp.num_draft, "ngram_min": sp.ngram_min, "ngram_max": sp.ngram_max,
            "verify_steps": st["verify_steps"], "drafted_tokens": st["drafted_tokens"], "accepted_tokens": st["accepted_tokens"],
            "acceptance_rate": st["accepted_tokens"] / st["drafted_tokens"] if st["drafted_tokens"] else 0.0,
            "emitted_tokens": st["emitted_tokens"],
            "tokens_per_sequence_per_verify_step":
                st["verify_emitted_tokens"] / st["verify_sequence_steps"] if st["verify_sequence_steps"] else 0.0,
        }
    return out
