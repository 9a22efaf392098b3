"""CPU suite: sampled decoding in the serving harness (atom_b200/textgen.py) -- each row's Philox key and counter through
prefill completion, chunked prefill, shared-prefix forks and decode steps; the sampling runner's static buffer; and the same
tokens with and without DecodeGraphRunner, with the numpy sampler of tests/sample_ref64.py standing in for the kernel."""
import numpy as np
import pytest
import torch

from atom_b200 import textgen as tg
from atom_b200.kvcache import KvCacheInt4, KvPoolInt4
from tests import sample_ref64 as R


class _FakeLM:
    """Stand-in model: logits = one_hot(7 * id + 3 mod vocab) for every row, whatever the step carries (prompt chunks,
    continuations, decode rows)."""

    def __init__(self, vocab, batch_size, block_len):
        self.vocab = vocab

    def __call__(self, ids, blen, prefill_kv, decode_kv):
        assert ids.numel() == blen.doff + blen.decode
        return torch.nn.functional.one_hot((ids.long() * 7 + 3) % self.vocab, self.vocab).float(), None


class _Recorder:
    """sample_op that records every row's (key, counter) and samples with the numpy reference."""

    def __init__(self):
        self.rows = []

    def __call__(self, logits, temperature, top_k, top_p, keys, counters):
        kw = np.asarray(keys.cpu().numpy().view(np.uint64) if hasattr(keys, "cpu") else keys, dtype=object).reshape(-1, 2)
        cw = np.asarray(counters.cpu().numpy().view(np.uint64) if hasattr(counters, "cpu") else counters).reshape(-1)
        self.rows.extend((int(k0), int(k1), int(c)) for (k0, k1), c in zip(kw, cw))
        return R.sample_tokens_np(logits, temperature, top_k, top_p, keys, counters)


def _run(cfg, rs, use_runner, sample_op, block=16, maxlen=96, vocab=97):
    pool = KvPoolInt4(1, 2, 128, tg.pool_capacity(cfg.batch_size, maxlen, block) + 8, block, torch.device("cpu"))
    runner = None
    if use_runner:
        runner = tg.DecodeGraphRunner(_FakeLM(vocab, cfg.batch_size, block), pool, "cpu",
                                      max_pages_per_seq=(maxlen + cfg.shared_prefix) // block + 2, capture=False,
                                      sampling=cfg.sampling, sample_op=sample_op)
    res = tg.run_textgen(_FakeLM(vocab, cfg.batch_size, block), rs, cfg, pool, torch.device("cpu"), keep_tokens=True,
                         decode_runner=runner, sample_op=sample_op)
    return res, pool


@pytest.mark.parametrize("chunk,shared", [(None, 0), (5, 0), (None, 20), (7, 20)])
@pytest.mark.parametrize("use_runner", [False, True])
def test_each_request_draws_with_its_own_key_and_token_counter(chunk, shared, use_runner):
    rs = tg.generate_request_set(11, 64)
    sp = tg.SamplingParams(0.8, top_k=20, top_p=0.9, seed=2 ** 63 + 5)
    rec = _Recorder()
    res, _ = _run(tg.TextGenConfig(4, prefill_chunk=chunk, shared_prefix=shared, sampling=sp), rs, use_runner, rec)
    assert [len(t) for t in res.tokens] == rs.output_lens.tolist()
    seen = {}
    for k0, k1, c in rec.rows:
        assert k0 == sp.seed
        seen.setdefault(k1, []).append(c)
    # every request: counters 0, 1, ..., output_len - 1 in that order, one per token; the system prompt draws nothing
    assert sorted(seen) == list(range(len(rs)))
    for r, cs in seen.items():
        assert cs == list(range(int(rs.output_lens[r])))


@pytest.mark.parametrize("shared", [0, 20])
def test_tokens_are_the_same_with_and_without_the_decode_runner(shared):
    rs = tg.generate_request_set(10, 80)
    cfg = tg.TextGenConfig(4, shared_prefix=shared, sampling=tg.SamplingParams(0.8, top_p=0.9, seed=9))
    a, pa = _run(cfg, rs, False, R.sample_tokens_np)
    b, pb = _run(cfg, rs, True, R.sample_tokens_np)
    assert a.tokens == b.tokens and b.graphed_steps > 0
    greedy, _ = _run(tg.TextGenConfig(4, shared_prefix=shared), rs, False, None)
    assert a.tokens != greedy.tokens                                    # the stand-in's argmax chain is not what is drawn
    top1, _ = _run(tg.TextGenConfig(4, shared_prefix=shared, sampling=tg.SamplingParams(0.8, top_k=1, seed=9)), rs, True,
                   R.sample_tokens_np)
    assert top1.tokens == greedy.tokens
    other, _ = _run(tg.TextGenConfig(4, shared_prefix=shared, sampling=tg.SamplingParams(0.8, top_p=0.9, seed=10)), rs, True,
                    R.sample_tokens_np)
    assert other.tokens != a.tokens


def test_sampling_runner_buffer_layout():
    block, maxp = 16, 4
    pool = KvPoolInt4(1, 2, 128, 16, block, torch.device("cpu"))
    sp = tg.SamplingParams(0.7, top_k=40, top_p=0.95, seed=2 ** 64 - 3)
    seen = {}

    def op(logits, *args):
        seen["args"] = args
        return torch.zeros(logits.size(0), dtype=torch.int32)

    r = tg.DecodeGraphRunner(lambda ids, blen, p, kv: (torch.zeros(ids.numel(), 5), None), pool, "cpu", max_pages_per_seq=maxp,
                             capture=False, sampling=sp, sample_op=op)
    plain = tg.DecodeGraphRunner(None, pool, "cpu", max_pages_per_seq=maxp, capture=False)
    for b in (1, 2, 3):
        kvs = [KvCacheInt4(pool, 5 + i) for i in range(b)]
        slots = [(10 + i, 3 * i) for i in range(b)]
        r.run([1] * b, kvs, slots)
        for c in kvs:
            c.release()
        e = r._entries[(b, 0)]
        o_key, o_ctr, o_k, o_t, o_p, total = r._sampling_layout(b)
        base = plain._layout(b)[-1]
        assert o_key in (base, base + 1) and o_key % 2 == 0 and e["host"].numel() == total == o_key + 9 * b
        assert e["host"].numel() > plain._layout(b)[-1]
        h = e["host"].numpy()
        assert h[o_key:o_ctr].view(np.uint64).reshape(b, 2).tolist() == [[sp.seed, 10 + i] for i in range(b)]
        assert h[o_ctr:o_k].view(np.uint64).tolist() == [3 * i for i in range(b)]
        assert h[o_k:o_t].tolist() == [40] * b
        assert h[o_t:o_p].view(np.float32).tolist() == [np.float32(0.7)] * b
        assert h[o_p:total].view(np.float32).tolist() == [np.float32(0.95)] * b
        t, k, p, keys, ctr = seen["args"]                    # the op gets views of the one device buffer
        assert keys.dtype == torch.int64 and keys.shape == (b, 2) and ctr.shape == (b,) and t.dtype == torch.float32
        dev = e["dev"]
        assert keys.data_ptr() == dev.data_ptr() + 4 * o_key and keys.data_ptr() % 8 == 0 and ctr.data_ptr() % 8 == 0
        assert keys.view(torch.uint64 if hasattr(torch, "uint64") else torch.int64).shape == (b, 2)


def test_sampling_params_are_validated():
    for bad in [dict(temperature=-1.0), dict(temperature=float("nan")), dict(temperature=1.0, top_k=-1),
                dict(temperature=1.0, top_p=0.0), dict(temperature=1.0, top_p=1.5), dict(temperature=1.0, seed=-1)]:
        with pytest.raises(ValueError):
            tg.SamplingParams(**bad)
    pool = KvPoolInt4(1, 2, 128, 16, 16, torch.device("cpu"))
    runner = tg.DecodeGraphRunner(None, pool, "cpu", max_pages_per_seq=2, capture=False)
    with pytest.raises(ValueError, match="sampling"):
        tg.run_textgen(_FakeLM(97, 2, 16), tg.generate_request_set(2, 32), tg.TextGenConfig(2, sampling=tg.SamplingParams(1.0)),
                       pool, torch.device("cpu"), decode_runner=runner, sample_op=R.sample_tokens_np)


def test_report_records_the_sampling_settings():
    rs = tg.generate_request_set(3, 32)
    sp = tg.SamplingParams(0.5, top_k=3, seed=4)
    res, _ = _run(tg.TextGenConfig(2, sampling=sp), rs, False, R.sample_tokens_np)
    rep = tg.report(rs, tg.TextGenConfig(2, sampling=sp), res)
    assert rep["sampling"] == {"temperature": 0.5, "top_k": 3, "top_p": 1.0, "seed": 4}
    assert tg.report(rs, tg.TextGenConfig(2), res)["sampling"] is None


def test_ops_sample_tokens_checks_its_inputs_on_the_host():
    from atom_b200 import ops
    l = torch.zeros(2, 8, dtype=torch.float16)
    with pytest.raises(RuntimeError, match="CUDA device"):
        ops.sample_tokens(l, [1.0, 1.0], [0, 0], [1.0, 1.0], [(0, 0), (0, 1)], [0, 0])
