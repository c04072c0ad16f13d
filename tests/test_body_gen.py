"""The body generators of tests/body_gen.py, which tests/test_gpu_bodies_edges.py runs on the GPU: deterministic for their
seeds, reaching the statuses they are meant to reach, placing bodies at the phases they claim, and inside the budgets the
GPU tests use.  Runs without a GPU."""
import collections

import numpy as np
import pytest

import bodies_oracle as bo
import body_gen as g
import json_model as jm

FAMILIES = ("carry_bodies", "many_starts", "window_bodies", "past_end_bodies", "key_bodies", "scalar_bodies", "abutting_scalars",
            "u_escape_bodies", "unescape_bodies", "fuzz_bodies")
TEXT_CAP_64K = 32768   # a chunk's staging at CTMR_FE_TEXT_CAP=65536
ENTRIES_CAP = 4096     # the max_batch_entries the GPU tests give


def staged(pairs):
    """staged offsets when the bodies are packed back to back from offset 0"""
    return np.cumsum([0] + [len(b) for b, _ in pairs[:-1]]).tolist()


@pytest.mark.parametrize("name", FAMILIES)
def test_each_family_is_deterministic_and_fits_the_budgets(name):
    a, b = getattr(g, name)(), getattr(g, name)()
    assert a == b and len(a) > 10
    assert all(isinstance(x, bytes) and 0 <= m <= 16 for x, m in a)
    assert max(len(x) for x, _ in a) <= (TEXT_CAP_64K if name == "fuzz_bodies" else 1 << 20)
    assert sum(m for _, m in a) <= 4 * ENTRIES_CAP


def test_deep_bodies_are_deterministic():
    with g.deep_recursion():
        assert g.deep_bodies() == g.deep_bodies()


def test_phased_puts_each_body_at_its_phase():
    items = [(b"x" * n, 0, p) for n, p in ((5, 0), (64, 63), (1, 1), (0, 2), (130, 2), (7, 62))]
    out = g.phased(items)
    offs = staged(out)
    assert [offs[2 * k + 1] % 64 for k in range(len(items))] == [p for _, _, p in items]
    for sac, _ in out[::2]:  # each sacrificial body: an open quote and a dangling backslash (or the backslash alone)
        assert sac.endswith(b"\\") and (sac == b"\\" or sac.startswith(b'"'))
        assert bo.parse_body(sac, 0)[0] == bo.BODY_BAD_JSON


def test_carries_reach_ok_and_bad_json_at_every_phase():
    out = g.carry_bodies()
    offs = staged(out)
    seen = collections.defaultdict(set)
    for k in range(1, len(out), 2):
        seen[offs[k] % 64].add(bo.parse_body(*out[k])[0])
    assert all({bo.BODY_OK, bo.BODY_BAD_JSON} <= seen[p] for p in range(64)), seen


def test_carry_runs_end_on_the_block_edges():
    """every run length of the family ends on the last two and the first two bytes of a block"""
    out = g.carry_bodies()
    offs = staged(out)
    got = collections.defaultdict(set)
    for k in range(1, len(out), 2):
        body = out[k][0]
        i = body.rfind(b"\\")
        j = i
        while j >= 0 and body[j] == 0x5C:
            j -= 1
        got[i - j].add((offs[k] + i) % 64)
    for run in range(1, 131):
        assert {62, 63, 0, 1} <= got[run], run


def test_many_starts_fill_blocks_with_body_starts():
    out = g.many_starts()
    offs = staged(out)
    per_block = collections.Counter(o // 64 for o in offs)
    assert max(per_block.values()) >= 10 and sum(v >= 10 for v in per_block.values()) >= 20
    # each block's junk body ends it exactly: the next block's first body starts on its first byte
    ends = [offs[k] + len(out[k][0]) for k in range(len(out)) if out[k][1] == 0]
    assert ends and all(e % 64 == 0 for e in ends), ends[:8]


def test_window_family_places_tokens_on_lane_edges():
    out = g.window_bodies()
    bodies = {b for b, _ in out}
    for T in g.lane_edges():
        assert any(len(b) > T and b[T] == 0x7B and b[:T].strip(g.WS) == b"" for b in bodies), T
    sts = collections.Counter(bo.parse_body(b, m)[0] for b, m in out[1::2])
    assert sts[bo.BODY_OK] > 100 and sts[bo.BODY_BAD_JSON] > 50


def test_past_end_strings_are_bad_json():
    assert all(bo.parse_body(b, m)[0] == bo.BODY_BAD_JSON for b, m in g.past_end_bodies())


def test_deep_builders_agree_with_the_oracle():
    import random
    rng = random.Random(0)
    with g.deep_recursion():
        for D in g.DEPTHS:
            for swap in (None, 1, 63, 64, 65, D):
                if swap is not None and swap > D:
                    continue
                body = g.deep_member(D, random.Random(rng.random()), swap_at=swap)
                st, ents = bo.parse_body(body, 2)
                assert (st, len(ents)) == g.deep_expected(D, swap), (D, swap)
                depth = maxd = 0
                for c in body:
                    depth += (c in b"{[") - (c in b"}]")
                    maxd = max(maxd, depth)
                assert maxd == D


def test_key_family_matches_and_misses():
    out = g.key_bodies()
    counts = collections.Counter()
    for b, m in out[1::2]:
        st, ents = bo.parse_body(b, m)
        counts[(st, len(ents), bool(ents) and ents[0][0] is not None)] += 1
    assert counts[(bo.BODY_OK, 1, True)] > 200      # matched key: the entry and its leaf_input
    assert counts[(bo.BODY_OK, 0, False)] > 20         # a miss of "entries": no entries
    assert counts[(bo.BODY_OK, 1, False)] > 20      # a miss of "leaf_input": an entry without it


def test_scalar_table_reaches_every_status_it_should():
    sts = collections.Counter(bo.parse_body(b, m)[0] for b, m in g.scalar_bodies())
    assert sts[bo.BODY_OK] > 50 and sts[bo.BODY_BAD_JSON] > 500 and sts[bo.BODY_BAD_TYPE] > 50
    for s in (b"-0", b"0e1", b"1E+2", b"1e400"):
        assert bo.parse_body(s, 0)[0] == bo.BODY_BAD_TYPE
    for s in (b"01", b"1.", b"-", b".5", b"tru", b"nulll"):
        assert bo.parse_body(s, 0)[0] == bo.BODY_BAD_JSON


def test_escaping_keeps_the_decoded_text():
    import random
    rng = random.Random(1)
    for l, x in g.real_strings():
        for s in (l, x):
            e = g.escape_b64(s, rng, 20)
            assert e != s
            st, ents = bo.parse_body(b'{"entries":[{"leaf_input":"' + e + b'"}]}', 1)
            assert st == bo.BODY_OK and ents[0][0].escaped and ents[0][0].data == s


def test_long_string_body_depends_on_its_last_run():
    b0, b1 = g.long_string_body(1 << 16, False), g.long_string_body(1 << 16, True)
    assert len(b1) == len(b0) + 1
    assert bo.parse_body(b0, 1)[0] == bo.BODY_OK and bo.parse_body(b1, 1)[0] == bo.BODY_BAD_JSON


def test_fuzz_reaches_all_five_statuses():
    sts = collections.Counter()
    sizes = []
    for seed in (9, 10):
        for b, m in g.fuzz_bodies(seed=seed, n=1000):
            sts[bo.parse_body(b, m)[0]] += 1
            sizes.append(len(b))
    n = sum(sts.values())
    assert sts[bo.BODY_OK] > n // 3 and sts[bo.BODY_BAD_JSON] > n // 10
    for s in (bo.BODY_BAD_TYPE, bo.BODY_TOO_MANY, bo.BODY_REPEATED_ENTRIES):
        assert sts[s] > n // 100, sts
    assert max(sizes) > 15000 and sum(s >= 50 for s in sizes) > n * 2 // 3


def test_json_model_on_the_carry_family():
    """the classify words of json_model against the byte scan over the carry family's staged text (what the GPU tests
    compare end to end)"""
    out = g.carry_bodies()[:600] + g.many_starts()
    text = b"".join(b for b, _ in out)
    starts = staged(out)
    e1, s1 = jm.classify(text, starts)
    e2, s2 = jm.byte_scan(text, starts)
    for k in range(len(e2)):
        valid = jm.M64 if 64 * k + 64 <= len(text) else (1 << (len(text) - 64 * k)) - 1
        assert e1[k] & valid == e2[k] and s1[k] & valid == s2[k], k
