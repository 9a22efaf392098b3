"""CPU suite: the split-KV rule of decode attention (atom_decode_kv_split) against a restatement of it in Python, over a grid of
batch sizes, KV heads, group sizes and SM counts that includes every threshold.  The library is loaded; no kernel is launched."""
import pytest

from atom_b200 import _lib


def rule(batch, kv_heads, sm_count):
    """1 when every SM already has a (sequence, KV head) CTA; else the smallest C in {2, 4, 8} with batch * kv_heads * C >= sm_count,
    8 at most."""
    ctas = batch * kv_heads
    if ctas >= sm_count:
        return 1
    for c in (2, 4):
        if ctas * c >= sm_count:
            return c
    return 8


def test_rule_matches_its_statement_over_a_grid_with_every_threshold():
    l = _lib.lib()
    seen = set()
    for sms in (1, 2, 7, 8, 16, 66, 114, 131, 132, 133, 264):
        sizes = sorted({1, 2, 3, 4, 5, 8, 16, 17, 32, 33, 64, 65, 131, 132, 133}
                       | {max(1, sms // c + d) for c in (1, 2, 4, 8) for d in (-1, 0, 1)})
        for b in sizes:
            for hkv in (1, 2, 8):
                for g in (1, 2, 4, 8):
                    got = l.atom_decode_kv_split(b, hkv, g, sms)
                    assert got == rule(b, hkv, sms), (b, hkv, g, sms, got)
                    seen.add(got)
    assert seen == {1, 2, 4, 8}


def test_rule_boundaries_on_a_132_sm_card():
    l = _lib.lib()
    for ctas, c in [(132, 1), (133, 1), (131, 2), (66, 2), (65, 4), (33, 4), (32, 8), (17, 8), (16, 8), (1, 8)]:
        assert l.atom_decode_kv_split(ctas, 1, 8, 132) == c, ctas
    # the harness shapes: llama3-8b (8 KV heads) at batch 1 / 4 / 16 / 32, Llama-2-70B at TP-8 (one KV head per rank)
    assert [l.atom_decode_kv_split(b, 8, 4, 132) for b in (1, 4, 16, 32)] == [8, 8, 2, 1]
    assert [l.atom_decode_kv_split(b, 1, 8, 132) for b in (1, 17, 33, 66, 132)] == [8, 8, 4, 2, 1]


@pytest.mark.parametrize("args", [(0, 1, 1, 132), (1, 0, 1, 132), (1, 1, 1, 0), (1, 1, 3, 132), (-1, 1, 1, 132)])
def test_rule_rejects_invalid_sizes(args):
    l = _lib.lib()
    assert l.atom_decode_kv_split(*args) < 0
    assert b"decode_kv_split" in l.atom_last_error()
