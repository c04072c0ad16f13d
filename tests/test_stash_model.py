"""stash_model on the CPU: the layout round trips, every malformation is refused, a small stash worked out by hand, and
the two properties a stash exists for: a client that applies the filter, the earlier stashes and the new stash gets
every key of R right (the client property), and the new stash lists nothing R lacks or the client already knew
(minimality)."""
import random
import struct

import pytest

import cascade_model as cm
import stash_model as sm

D1, D2, D3 = b"\x01" * 32, b"\x02" * 32, b"\xf0" + b"\x00" * 31


def test_encode_decode_round_trip_and_concatenation():
    a = sm.encode([(D2, b"\x05"), (D1, b"\x07\x01"), (D1, b"\x07"), (D2, b"\x05"), (D1, b"\x06" * 40)])
    assert sm.decode(a) == [(D1, [b"\x06" * 40, b"\x07", b"\x07\x01"]), (D2, [b"\x05"])]
    b = sm.encode([(D1, b"\x09"), (D3, b"")])
    assert sm.decode(a + b) == sm.decode(a) + sm.decode(b)
    assert sm.listed(a + b) == {D1 + b"\x06" * 40, D1 + b"\x07", D1 + b"\x07\x01", D2 + b"\x05", D1 + b"\x09", D3}
    assert sm.encode([]) == b"" and sm.decode(b"") == []
    zero = struct.pack("<IB", 0, 32) + D3
    assert sm.decode(zero) == [(D3, [])]


def test_a_prefix_sorts_first_and_bytes_are_unsigned():
    data = sm.encode([(D1, b"\x80"), (D1, b"\x7f\xff"), (D1, b"\x7f"), (D3, b"\x01"), (D2, b"\x01")])
    assert sm.decode(data) == [(D1, [b"\x7f", b"\x7f\xff", b"\x80"]), (D2, [b"\x01"]), (D3, [b"\x01"])]


@pytest.mark.parametrize("bad", [
    b"\x01",                                                        # shorter than a unit header
    struct.pack("<IB", 1, 32) + D1,                                 # an entry missing
    struct.pack("<IB", 1, 32) + D1 + b"\x03\x01\x02",               # an entry one byte short
    struct.pack("<IB", 0, 20) + D1,                                 # a hash length that is not 32
    struct.pack("<IB", 0, 32) + D1[:31],                            # a digest one byte short
    sm.encode([(D1, b"\x01")]) + b"\x00",                           # a truncated second unit
])
def test_malformed_stashes_are_refused(bad):
    with pytest.raises(ValueError):
        sm.decode(bad)


def _level(level, k, m, bits):
    return struct.pack("<BIIB", 2, m, k, level) + bits


def test_malformed_filters_are_refused():
    good = cm.build([D1 + b"\x01"], [D1 + b"\x02"], b"s")
    sm.check_filter(good)
    one = _level(1, 1, 8, b"\x00")
    hdr = struct.pack("<HBB", 2, 0, 0)
    bad = [b"", b"\x02\x00\x00", struct.pack("<HBB", 1, 0, 0) + one, struct.pack("<HBB", 2, 1, 0) + one,
           struct.pack("<HBB", 2, 0, 33) + b"\x00" * 33 + one, hdr, hdr + one + b"\x00",
           hdr + struct.pack("<BIIB", 1, 8, 1, 1) + b"\x00", hdr + _level(1, 0, 8, b"\x00"), hdr + _level(1, 65, 8, b"\x00"),
           hdr + _level(1, 1, 7, b"\x00"), hdr + _level(2, 1, 8, b"\x00"), hdr + _level(1, 1, 9, b"\x00"),
           hdr + _level(1, 1, 9, b"\x00\x02"), hdr + one + _level(3, 1, 8, b"\x00")]
    for b in bad:
        with pytest.raises(ValueError):
            sm.check_filter(b)
    sm.check_filter(hdr + _level(1, 64, 9, b"\x00\x01"))


def test_a_small_stash_by_hand():
    # level 1 sets no bit: it contains nothing, so the filter says "not revoked" to every key
    flt = struct.pack("<HBB", 2, 0, 0) + _level(1, 1, 8, b"\x00")
    R = [D2 + b"\x01", D1 + b"\x03", D1 + b"\x02", D1 + b"\x03", D3 + b"\x09"]
    earlier = struct.pack("<IB", 1, 32) + D3 + b"\x01\x09"
    data, n = sm.stash(R, flt, earlier)
    assert data == (struct.pack("<IB", 2, 32) + D1 + b"\x01\x02\x01\x03" + struct.pack("<IB", 1, 32) + D2 + b"\x01\x01")
    assert n == {"revoked": 5, "in_filter": 0, "in_stashes": 1, "serials": 3, "stash_issuers": 2}
    # every bit set with L = 1: every key is in every level, and L is odd, so the filter says "revoked" to all
    full = struct.pack("<HBB", 2, 0, 0) + _level(1, 1, 8, b"\xff")
    assert sm.stash(R, full) == (b"", {"revoked": 5, "in_filter": 5, "in_stashes": 0, "serials": 0, "stash_issuers": 0})


def _keys(rng, n, digests):
    return [rng.choice(digests) + bytes(rng.randrange(256) for _ in range(rng.randrange(1, 40))) for _ in range(n)]


@pytest.mark.parametrize("seed", range(4))
def test_client_property_and_minimality(seed):
    rng = random.Random(seed)
    digs = [bytes([i]) * 32 for i in range(1, 6)]
    keys = list(dict.fromkeys(_keys(rng, 3000, digs)))
    day0_R, S = keys[:150], keys[150:2500]
    salt = rng.randbytes(rng.choice([0, 1, 19, 32]))
    flt = cm.build(day0_R, S, salt)
    later = keys[2500:]
    day1_R = day0_R[10:] + later[:200] + later[:30]          # some revocations dropped, a serial under two hours
    s1, n1 = sm.stash(day1_R, flt)
    day2_R = day1_R + later[200:320]
    s2, n2 = sm.stash(day2_R, flt, s1)
    for R, stashes, new, n in ((day1_R, b"", s1, n1), (day2_R, s1, s2, n2)):
        old, fresh = sm.listed(stashes), sm.listed(new)
        assert n["revoked"] == n["in_filter"] + n["in_stashes"] + sum(x in fresh for x in R)
        for x in R:  # the client property
            assert cm.query(flt, x) or x in old or x in fresh
        for x in fresh:  # minimality
            assert x in R and not cm.query(flt, x) and x not in old
    assert n2["in_stashes"] > 150 and 0 < n2["serials"] <= 120
