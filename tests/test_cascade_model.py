"""The filter cascade model (cascade_model.py) on its own: every included key queries revoked and every excluded key
valid, the edges of the build, one hash assembled by hand, and the sizing values."""
import hashlib
import math
import random
import struct

import pytest

import cascade_model as cm


def _keys(rng, n, tag):
    return [bytes([tag]) * 32 + rng.randbytes(rng.randint(1, 39)) for _ in range(n)]


def _check(R, S, salt):
    data = cm.build(R, S, salt)
    d = cm.decode(data)
    assert d["salt"] == salt
    assert all(cm.query(d, x) for x in R)
    assert not any(cm.query(d, x) for x in S)
    return d


@pytest.mark.parametrize("seed", range(6))
def test_random_sets_every_salt_length_and_duplicates(seed):
    rng = random.Random(seed)
    R = _keys(rng, rng.randint(1, 300), 1)
    S = _keys(rng, rng.randint(1, 3000), 2)
    R += R[:10]  # one serial under two hours: two key records, one key
    S += S[:25]
    for sl in (0, 1, 7, 31, 32):
        _check(R, S, rng.randbytes(sl))


def test_edges():
    rng = random.Random(9)
    R, S = _keys(rng, 50, 1), _keys(rng, 50, 2)
    for r, s in (([], S), (R, []), ([], []), (R[:1], []), ([], S[:1]), (R[:1], S[:1])):
        d = _check(r, s, b"")
        if not r or not s:
            assert len(d["levels"]) == 1
    empty = cm.decode(cm.build([], [], b"ab"))
    assert empty["levels"] == [(1, 1, 8, b"\0")]
    assert cm.build([], [], b"ab")[:6] == b"\x02\x00\x00\x02ab"


def test_small_s_forces_many_levels():
    rng = random.Random(3)
    d = _check(_keys(rng, 400, 1), _keys(rng, 400, 2), b"s")
    assert len(d["levels"]) >= 4
    for level, k, m, _ in d["levels"][1:]:
        assert k == 1


def test_one_hash_by_hand():
    salt, x = b"\x5a" * 3, b"\x11" * 32 + b"\x00\x80"
    msg = salt + b"\x05\x00\x00\x00" + b"\x02" + x
    want = int.from_bytes(hashlib.sha256(msg).digest()[:4], "little") % 1000
    assert cm.bit(salt, 5, 2, x, 1000) == want
    data = cm.build([x], [], salt)
    assert data[:7] == b"\x02\x00\x00\x03" + salt
    alg, m, k, level = struct.unpack_from("<BIIB", data, 7)
    assert (alg, m, k, level) == (2, 8, 1, 1)  # n = 1, p = 0.5: ceil(1 / log 2) = 2 bits, at least 8


def test_sizing_values():
    assert cm.sizing(0, 0.5) == (1, 8)
    assert cm.sizing(0, 0.01) == (7, 8)
    assert cm.sizing(5, 0.5) == (1, 8)
    assert cm.sizing(100, 0.5) == (1, 145)
    k, m = cm.sizing(1000, 0.01)
    assert k == 7 and m == math.ceil(-7 * 1000 / math.log(1 - 0.01 ** (1 / 7)))
    assert cm.first_rate(0, 5) == cm.first_rate(5, 0) == 0.5
    assert cm.first_rate(10, 5) == 0.5
    assert cm.first_rate(1, 1000) == 1 / (math.sqrt(2) * 1000)
    assert cm.sizing(1, cm.first_rate(1, 1000))[0] == 11


def test_refusals():
    with pytest.raises(ValueError):
        cm.build([], [], b"\0" * 33)
    with pytest.raises(ValueError):
        cm.build([b"a" * 33], [b"a" * 33])
