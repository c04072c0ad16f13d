"""The probe-rule restatement (tests/probe_model.py) on the CPU: the key makers land on the chosen home slots by the
scalar restatements of keymodel / metamodel, the linear-probing model follows the rule, and the chain check finds holes
and records past the limit."""
import numpy as np
import pytest

import keymodel as K
import metamodel as M
import probe_model as P
import xchg_model as X
from fe_model import inv_mix


def test_inv_mix_inverts_mix64():
    rng = np.random.default_rng(1)
    for z in [0, 1, P.M64] + [int.from_bytes(rng.bytes(8), "little") for _ in range(200)]:
        assert inv_mix(K.mix64(z)) == z and K.mix64(inv_mix(z)) == z


@pytest.mark.parametrize("log2", (13, 14))
@pytest.mark.parametrize("home", (0, 4096, (1 << 13) - 1 - 2000, (1 << 13) - 1))
def test_known_serials_land_on_their_home(log2, home):
    homes = [home + (i & 1) * (1 << 13) if log2 > 13 else home for i in range(64)]
    serials = P.known_serials(490000, 3, homes, log2, seed=home + log2)
    assert len(set(serials)) == 64 and all(len(s) == P.SERIAL_LEN and 0 < s[0] < 0x80 for s in serials)
    bodies = [K.key_body(490000, 3, s) for s in serials]
    mask = (1 << log2) - 1
    assert [K.home_slot(K.key_hash(b), mask) for b in bodies] == homes
    vec = K.key_hash_np(np.array(bodies, np.uint32))  # the vectorised hash agrees
    assert [int(v) for v in vec] == [K.key_hash(b) for b in bodies]
    assert {K.home_slot(K.key_hash(b), (1 << 13) - 1) for b in bodies} == {home}


def test_serial_for_hash_hits_any_hash():
    rng = np.random.default_rng(2)
    prefix = b"\x42" + bytes(range(30))
    for _ in range(50):
        h = int.from_bytes(rng.bytes(8), "little")
        assert K.key_hash(K.key_body(-7, 0, P.serial_for_hash(-7, 0, prefix, h))) == h


@pytest.mark.parametrize("owner", (None, 0, 1))
def test_pair_hours_share_a_home(owner):
    kw = (2, owner) if owner is not None else ()
    hours = P.pair_hours(5, 77, 10, 40, 490000, *kw)
    assert len(set(hours)) == 40 and min(hours) > 490000 and list(hours) == sorted(hours)
    assert all(K.mix64(K.pair_key(h, 5)) & 1023 == 77 for h in hours)
    if owner is not None:
        assert all(X.key_owner(h, 5, 2) == owner for h in hours)
    # nothing skipped: every hour in between has another home or owner
    got = set(hours)
    for h in range(490001, hours[-1]):
        if h not in got:
            assert K.mix64(K.pair_key(h, 5)) & 1023 != 77 or (owner is not None and X.key_owner(h, 5, 2) != owner)


def test_meta_targets_land_on_their_home():
    mask = (1 << 13) - 1
    for salt, home in enumerate((0, 4096, mask - 2000, mask)):
        b = M.crafted(M.leaf(salt, org=M.ORG), M.KIND_DN, 0, M.target_h1(home, mask, salt))
        assert M.home_slot(M.hash_bytes(M.name_bytes(b), M.seed_of(0, M.KIND_DN))[0], mask) == home


def test_probe_table_places_up_to_the_limit_and_finds_past_it():
    """One home: keys at distance 0 .. limit are placed, the next is refused; keys placed again go anywhere and every
    one is found."""
    limit = 12
    t = P.ProbeTable(6)
    for i in range(limit + 1):
        assert t.insert(("k", i), 60, limit) == (60 + i) & 63
    with pytest.raises(P.TableFull):
        t.insert(("k", limit + 1), 60, limit)
    assert t.insert(("k", 3), 60, limit) == 63   # a key the table holds is found, not placed again
    assert t.insert(("k", limit + 1), 60, None) == (60 + limit + 1) & 63
    assert t.insert(("k", limit + 2), 61, None) == (60 + limit + 2) & 63
    for i in range(limit + 2):
        assert t.find(("k", i), 60) == (60 + i) & 63
    assert t.find(("k", limit + 2), 61) == (60 + limit + 2) & 63
    assert t.find(("x", 0), 60) is None and t.find(("x", 0), 20) is None
    for i in range(64 - (limit + 3)):
        t.insert(("f", i), 20, None)
    with pytest.raises(P.TableFull):  # every slot taken
        t.insert(("f", 99), 20, None)
    assert t.find(("f", 99), 20) is None


def test_reinsert_order_needs_no_limit():
    """Records placed within the limit, placed again in slot order: some land further than the limit (why eviction,
    resize and checkpoint loads place records again without one), and all are found."""
    rng = np.random.default_rng(3)
    limit, worse = 12, 0
    for _ in range(300):
        t = P.ProbeTable(8)
        homes = {}
        for k in range(230):
            h = int(rng.integers(0, 256))
            try:
                t.insert(k, h, limit)
                homes[k] = h
            except P.TableFull:
                pass
        again = P.ProbeTable(8)
        for pos, k in enumerate(t.slots):
            if k is not None:
                again.insert(k, homes[k], None)
        d = [P.distance(again.find(k, h), h, 255) for k, h in homes.items()]
        worse += max(d) > limit
        assert all(again.find(k, h) is not None for k, h in homes.items())
    assert worse > 0


def _walk_ok(pos, home, occ):
    s = home
    while s != pos:
        if not occ[s]:
            return False
        s = (s + 1) % occ.size
    return True


def test_check_chains_is_the_slot_walk():
    rng = np.random.default_rng(4)
    for _ in range(200):
        n = 64
        occ = rng.random(n) < rng.choice((0.3, 0.8, 0.97, 1.0))
        at = np.nonzero(occ)[0]
        if not at.size:
            continue
        homes = (at - rng.integers(0, 20, at.size)) % n
        ok = all(_walk_ok(int(p), int(h), occ) for p, h in zip(at, homes))
        if ok:
            d = P.check_chains(at, homes, occ, None)
            assert d.tolist() == [int(x) for x in (at - homes) % n]
            if d.max() > 5:
                with pytest.raises(AssertionError, match="past the probe limit"):
                    P.check_chains(at, homes, occ, 5)
        else:
            with pytest.raises(AssertionError, match="hole"):
                P.check_chains(at, homes, occ, None)


def test_check_table_holds_keys_to_the_limit():
    """keymodel.check_table on a hand-made snapshot: a chain of limit + 2 keys passes with the limit raised and fails
    with the probe limit."""
    log2, n = 13, P.PROBE_LIMIT + 2
    mask = (1 << log2) - 1
    serials = P.known_serials(490000, 0, [mask - 2000] * n, log2, seed=9)
    table = np.zeros(mask + 1, K.KNOWN_SLOT)
    pairs = np.zeros(16, K.PAIR_SLOT)
    model = K.KeyModel()
    for i, s in enumerate(serials):
        body = K.key_body(490000, 0, s)
        pos = (mask - 2000 + i) & mask
        table[pos]["body"] = body
        table[pos]["tag"] = K.ready_tag(K.key_hash(body))
        table[pos]["inv_first"] = ~np.uint64(i)
        model.first[body] = i
    pk = K.pair_key(490000, 0)
    slot = K.mix64(pk) & 15
    pairs[slot]["key"], pairs[slot]["inv_first"], pairs[slot]["count"] = pk, ~np.uint64(0), n
    model.pair_first[(490000, 0)] = 0
    assert K.check_table((table, pairs), model, n, limit=n - 1) == n
    with pytest.raises(AssertionError, match="past the probe limit"):
        K.check_table((table, pairs), model, n)
    table[(mask - 2000 + 7) & mask] = np.zeros(1, K.KNOWN_SLOT)[0]   # a hole: the keys after it are lost
    del model.first[K.key_body(490000, 0, serials[7])]
    pairs[slot]["count"] = n - 1
    with pytest.raises(AssertionError, match="hole"):
        K.check_table((table, pairs), model, n - 1, limit=n - 1)
