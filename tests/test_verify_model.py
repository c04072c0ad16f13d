"""verify_model on the CPU: a built filter verifies clean, a flipped bit makes exactly the predicted records missed or
blocked at every level parity, stashes turn missed records into revoked, covered_below splits counts and list, and the
list's order."""
import random
import struct

import pytest

import cascade_model as cm
import stash_model as sm
import verify_model as vm

D0, D1 = b"\x10" * 32, b"\x20" * 32


def _universe(n, seed):
    rng = random.Random(seed)
    keys = list(dict.fromkeys((D0, D1)[i % 2] + bytes([rng.randrange(1, 128)]) + rng.randbytes(i % 20) for i in range(n)))
    return [(x, 500000 + i % 3, i) for i, x in enumerate(keys)]


def _levels(flt):
    """(header bytes, [(offset of the level's bits, level, k, m)]) of a serialized filter"""
    sl = flt[3]
    o, out = 4 + sl, []
    while o < len(flt):
        _, m, k, level = struct.unpack_from("<BIIB", flt, o)
        out.append((o + 10, level, k, m))
        o += 10 + (m + 7) // 8
    return out


def _reaches(d, x, level):
    """x is contained in every level before `level`"""
    return all(cm._contains(bits, d["salt"], lv, k, m, x) for lv, k, m, bits in d["levels"][:level - 1])


@pytest.fixture(scope="module")
def built():
    recs = _universe(1500, 3)
    R, S = recs[::5], [r for i, r in enumerate(recs) if i % 5]
    flt = cm.build([x for x, _, _ in R], [x for x, _, _ in S], b"v")
    return R, S, flt


def test_a_built_filter_verifies_clean(built):
    R, S, flt = built
    counts, lst = vm.verify(R, S, flt)
    assert counts["before"] == {"revoked": len(R), "missed": 0, "valid": len(S), "blocked": 0}
    assert counts["since"] == dict.fromkeys(vm.NAMES, 0) and lst == []
    assert len(cm.decode(flt)["levels"]) >= 4


def test_a_cleared_bit_at_every_level(built):
    """clearing a bit of level l stops every record that reaches l and hashes to it there: its answer becomes 'level l is
    even'; every other record keeps its answer"""
    R, S, flt = built
    d = cm.decode(flt)
    parities = set()
    for off, level, k, m in _levels(flt):
        target = next((x for x, _, _ in R + S if _reaches(d, x, level) and cm._contains(d["levels"][level - 1][3], d["salt"], level, k, m, x)), None)
        if target is None:
            continue
        b = cm.bit(d["salt"], 0, level, target, m)
        f2 = bytearray(flt)
        f2[off + (b >> 3)] &= ~(1 << (b & 7)) & 0xFF
        hit = lambda x: _reaches(d, x, level) and any(cm.bit(d["salt"], i, level, x, m) == b for i in range(k))  # noqa: E731
        want = sorted([(x[:32], x[32:], h, f, False) for x, h, f in R if hit(x) and level % 2 == 1] +
                      [(x[:32], x[32:], h, f, True) for x, h, f in S if hit(x) and level % 2 == 0], key=lambda e: e[:3])
        counts, lst = vm.verify(R, S, bytes(f2))
        assert lst == want and want, level
        assert counts["before"]["missed"] + counts["before"]["blocked"] == len(want)
        parities.add(level % 2)
    assert parities == {0, 1}


def test_contained_in_every_level():
    """an S record that stops at the last (odd) level, with its bits there set, is contained in all L levels: revoked"""
    for seed in range(40):
        recs = _universe(400, seed)
        R, S = recs[::4], [r for i, r in enumerate(recs) if i % 4]
        flt = cm.build([x for x, _, _ in R], [x for x, _, _ in S])
        d = cm.decode(flt)
        L = len(d["levels"])
        if L % 2 == 0:
            continue
        off, level, k, m = _levels(flt)[-1]
        x, h, f = next(r for r in S if _reaches(d, r[0], L))
        f2 = bytearray(flt)
        for i in range(k):
            b = cm.bit(d["salt"], i, L, x, m)
            f2[off + (b >> 3)] |= 1 << (b & 7)
        new = cm.decode(bytes(f2))["levels"][-1][3]
        want = sorted((y[:32], y[32:], hh, ff, True) for y, hh, ff in S
                      if _reaches(d, y, L) and cm._contains(new, d["salt"], L, k, m, y))
        counts, lst = vm.verify(R, S, bytes(f2))
        assert (x[:32], x[32:], h, f, True) in lst and lst == sorted(want, key=lambda e: e[:3])
        assert counts["before"]["blocked"] == len(want) and counts["before"]["missed"] == 0
        return
    pytest.fail("no odd-level filter among the seeds")


def test_stashes_turn_missed_into_revoked(built):
    R, S, flt = built
    extra = [r for r in _universe(1700, 3)[1500:] if not cm.query(flt, r[0])]  # revoked after the filter, and missed
    counts, lst = vm.verify(R + extra, S, flt)
    assert counts["before"]["missed"] == len(extra) and all(not e[4] for e in lst) and len(lst) == len(extra)
    stash = sm.encode((x[:32], x[32:]) for x, _, _ in extra[::2])
    counts, lst = vm.verify(R + extra, S, flt, stash)
    assert counts["before"]["missed"] == len(extra[1::2]) and counts["before"]["revoked"] == len(R) + len(extra[::2])
    assert sorted(e[3] for e in lst) == sorted(f for _, _, f in extra[1::2])
    blocked = sm.encode([(S[0][0][:32], S[0][0][32:])])                    # a stash that lists a valid record blocks it
    counts, lst = vm.verify(R, S, flt, blocked)
    assert counts["before"]["blocked"] == 1 and lst == [(S[0][0][:32], S[0][0][32:], S[0][1], S[0][2], True)]


def test_covered_below_splits_counts_and_list(built):
    R, S, flt = built
    extra = [(x, h, f + 10_000) for x, h, f in _universe(1700, 3)[1500:] if not cm.query(flt, x)]
    late = [(x, h, f + 20_000) for x, h, f in _universe(1800, 5)[:60]]
    every, lst_all = vm.verify(R + extra, S + late, flt)
    split, lst = vm.verify(R + extra, S + late, flt, covered_below=10_000)
    assert split["before"] == {"revoked": len(R), "missed": 0, "valid": len(S), "blocked": 0}
    assert sum(split["since"].values()) == len(extra) + len(late) and split["since"]["missed"] == len(extra)
    assert lst == [] and len(lst_all) == every["before"]["missed"] + every["before"]["blocked"]
    for n in vm.NAMES:
        assert every["before"][n] == split["before"][n] + split["since"][n]


def test_list_order():
    """a serial before every longer serial it prefixes, and one serial under two hours twice, by hour"""
    x = D0 + b"\x05"
    R = [(D1 + b"\x01", 9, 1), (x + b"\x00", 5, 2), (x, 7, 3), (x, 6, 4), (D0 + b"\x04\xff", 5, 5)]
    flt = cm.build([], [D0 + b"\x7f"])
    counts, lst = vm.verify(R, [], flt)
    assert counts["before"]["missed"] == 5
    assert [(e[0][:1], e[1], e[2]) for e in lst] == [(b"\x10", b"\x04\xff", 5), (b"\x10", b"\x05", 6), (b"\x10", b"\x05", 7),
                                                     (b"\x10", b"\x05\x00", 5), (b"\x20", b"\x01", 9)]
