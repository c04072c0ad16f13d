"""The GPU body scanner (csrc/ctmr_json.cu) where its bit arithmetic can go wrong, each family of tests/body_gen.py in one
call through run_pair (everything against a twin ctmr_process_raw given the oracle's spans): escape and string carries at
every block phase, the warp window's edges, nesting past the register stack, folded and escaped keys, scalars against
every delimiter, \\u escapes and the unescape of real entries, one body over many scan tiles, the chunk budgets, and a
grammar fuzz in both upload layouts, over many chunks and on a group.  Marked gpu."""
import random

import pytest

import bodies_oracle as bo
import body_gen as g
from bodies_pair import run_pair
from conftest import NOW_NS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def pair(eng, entries=1 << 14):
    """a db and its twin; entries per chunk large enough that a phase-controlled family stays in one chunk"""
    kw = dict(table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=entries)
    return eng.GpuCertDatabase(**kw), eng.GpuCertDatabase(**kw)


def run_both_layouts(db, twin, items, **kw):
    """packed, and one copy without gaps: the same staged offsets, so the same phases"""
    bodies, maxes = [b for b, _ in items], [m for _, m in items]
    run_pair(db, twin, bodies, maxes, layout="packed", **kw)
    return run_pair(db, twin, bodies, maxes, layout="one_copy", gaps=[b""] * len(bodies), **kw)


def test_escape_and_string_carries_at_every_phase(eng):
    items = g.carry_bodies() + g.many_starts()
    db, twin = pair(eng)
    with db, twin:
        r = run_both_layouts(db, twin, items)
        assert (r.body_status == bo.BODY_OK).sum() > 1000
        starts = g.many_starts(seed=12)  # the tiny bodies again, with junk gaps between them
        run_pair(db, twin, [b for b, _ in starts], [m for _, m in starts], layout="one_copy")


def test_warp_window_edges(eng):
    items = g.window_bodies()
    db, twin = pair(eng)
    with db, twin:
        r = run_both_layouts(db, twin, items)
        assert r.escaped.any() and (r.entry_status == 0).sum() >= 6
        past = g.past_end_bodies()  # the would-be closing quote in the next body, then in the junk after the body
        bodies, maxes = [b for b, _ in past], [m for _, m in past]
        run_pair(db, twin, bodies, maxes, layout="packed")
        run_pair(db, twin, bodies, maxes, layout="one_copy", gaps=[b'"'] * len(bodies))


def test_nesting_past_the_register_stack(eng):
    with g.deep_recursion():
        items = g.deep_bodies()
        db, twin = pair(eng)
        with db, twin:
            r = run_both_layouts(db, twin, items)
            assert (r.body_status == bo.BODY_OK).sum() == len(g.DEPTHS)
            for D in (65, 128, 1000, 10000):  # four deep bodies back to back: they share p.stack words at their edges
                four = [(g.deep_member(D, random.Random(D * 10 + k), swap_at=(None if k % 2 else 64)), 2)
                        for k in range(4)]
                bodies, maxes = [b for b, _ in four], [m for _, m in four]
                run_pair(db, twin, bodies, maxes, layout="packed")
                run_pair(db, twin, bodies, maxes, layout="one_copy", gaps=[b""] * 4)
                run_pair(db, twin, bodies, maxes, layout="one_copy")


def test_folded_escaped_and_near_miss_keys(eng):
    items = g.key_bodies()
    db, twin = pair(eng)
    with db, twin:
        r = run_both_layouts(db, twin, items)
        assert (r.entry_status == 0).sum() > 200


def test_scalars_against_every_delimiter(eng):
    db, twin = pair(eng)
    with db, twin:
        items = g.scalar_bodies()
        run_both_layouts(db, twin, items)
        ab = g.abutting_scalars()  # one copy of abutting bodies: the scan of the first must stop at its end
        run_pair(db, twin, [b for b, _ in ab], [m for _, m in ab], layout="one_copy", gaps=[b""] * len(ab))


def test_u_escapes_and_unescape_of_real_entries(eng):
    db, twin = pair(eng)
    with db, twin:
        run_both_layouts(db, twin, g.u_escape_bodies())
        r = run_both_layouts(db, twin, g.unescape_bodies())
        assert r.escaped.sum() > 40 and (r.entry_status == 0).sum() > 60


def test_one_body_over_many_scan_tiles(eng):
    big, bad = g.long_string_body(4 << 20, False), g.long_string_body(4 << 20, True)
    assert len(big) >= 4 << 20
    small = g.fuzz_bodies(seed=21, n=12)
    bodies = [b for b, _ in small[:4]] + [big] + [b for b, _ in small[4:8]] + [bad] + [b for b, _ in small[8:]]
    maxes = [m for _, m in small[:4]] + [1] + [m for _, m in small[4:8]] + [1] + [m for _, m in small[8:]]
    db, twin = pair(eng, entries=4096)
    with db, twin:
        r = run_pair(db, twin, bodies, maxes, layout="packed")
        assert r.body_status[4] == bo.BODY_OK and r.body_status[9] == bo.BODY_BAD_JSON
        run_pair(db, twin, bodies, maxes, layout="one_copy")


def test_budgets_and_chunking(eng, monkeypatch):
    from ct_mapreduce_b200 import capi
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", "65536")  # 32 KiB of staging per chunk
    (l0, x0), = g.real_strings()[:1]
    one = b'{"leaf_input":"' + l0 + b'","extra_data":"' + x0 + b'"}'
    head = b'{"entries":[' + one + b'],"pad":"'
    exact = head + b"p" * (32768 - len(head) - 2) + b'"}'
    assert len(exact) == 32768
    ents3 = b'{"entries":[' + b",".join([b'{"leaf_input":"QUFB"}', b"null", b"{}"]) + b"]}"
    db, twin = pair(eng, entries=64)
    with db, twin:
        run_pair(db, twin, [exact, exact, b"{}"], [1, 0, 0], layout="packed")
        run_pair(db, twin, [b"{}", exact, b"{}"], [0, 1, 0], layout="one_copy")
        with pytest.raises(capi.CtmrError) as e:
            db.store_raw_bodies(exact + b" ", [0], [32769], [1], NOW_NS)
        assert e.value.code == capi.E_BATCH_TOO_LARGE
        run_pair(db, twin, [ents3] * 4, [3, 2, 0, 4], layout="one_copy")           # == body_max, + 1, max 0, under
        run_pair(db, twin, [b"{}", b"null", b'{"entries":[]}'] * 43 + [b" "], [1] * 130, layout="one_copy")  # 64 a chunk
        run_pair(db, twin, [b"{}"] * 200, [0] * 200, layout="packed")
        run_pair(db, twin, [b""] * 100, [1] * 100, layout="packed")                 # only zero-length bodies
        run_pair(db, twin, [b""] * 5, [0] * 5, layout="one_copy")


@pytest.fixture(scope="module")
def fuzz():
    items = []
    for seed in (31, 32, 33, 34):
        items += g.fuzz_bodies(seed=seed, n=1000)
    return [b for b, _ in items], [m for _, m in items]


def test_fuzz_in_both_layouts(eng, fuzz):
    bodies, maxes = fuzz
    db, twin = pair(eng, entries=4096)
    with db, twin:
        r = run_pair(db, twin, bodies, maxes, layout="one_copy")
        assert set(r.body_status.tolist()) == {0, 1, 2, 3, 4}
        run_pair(db, twin, bodies, maxes, layout="packed")


def test_fuzz_over_many_chunks(eng, fuzz, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", "65536")
    bodies, maxes = fuzz
    db, twin = pair(eng, entries=256)
    with db, twin:
        run_pair(db, twin, bodies, maxes, layout="one_copy")


def test_fuzz_on_a_group(eng, fuzz):
    bodies, maxes = fuzz
    kw = dict(table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=1024)
    with eng.GpuCertGroup([0, 0, 0], **kw) as grp, eng.GpuCertDatabase(**kw) as twin:
        run_pair(grp, twin, bodies, maxes, layout="one_copy")
