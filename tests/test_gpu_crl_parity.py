"""Parity for ctmr_revoked_known's CRL parser, split and join on the GPU: the whole catalogue of tests/crl_cases.py and
its seeded mutants against crl_oracle in one chunk, in chunks of 4 KiB and on a group; serials of every length with
their near misses; crafted collisions of the (issuer, serial) set; the chunk cuts and budgets; and the cascade's
coverage over the same catalogue."""
import numpy as np
import pytest

import crl_cases as cc
import crl_oracle as co
import crl_pair_model as pm
from ct_mapreduce_b200 import capi, engine
from ct_mapreduce_b200.capi import CtmrError
from oracle import oracle

pytestmark = pytest.mark.gpu

NOW = 1767225600
HOUR = NOW // 3600
UNKNOWN = b"\xee" * 32


@pytest.fixture(scope="module")
def issuers():
    cfg = oracle.synth_cfg(64, n_issuers=16, dup_mode=1)
    return oracle.synth_issuers(cfg)


def _register(db, issuers):
    """(dense indices, digests) of the registered issuers"""
    dense = [int(d) for d in db.register_issuers(*issuers)]
    return dense, [db.issuer_digest(d) for d in dense]


def _check(res, crls, digs, sets, registered):
    """Every output of the call against crl_oracle (tests/test_gpu_crl.py's check, with serial_len saturating at 255)."""
    data, offs, _ = engine.pack_crls(crls)
    e = 0
    for k, der in enumerate(crls):
        p = co.parse_crl(der)
        j = co.join(p, digs[k], sets, registered)
        assert res.crl_status[k] == j["status"], k
        if j["status"] not in (co.CRL_OK, co.CRL_UNKNOWN_ISSUER):
            assert res.crl_entries[k] == 0
            continue
        assert res.crl_flags[k] == p["flags"] and res.this_update[k] == p["this_update"] and res.next_update[k] == p["next_update"], k
        assert (res.tbs_off[k] - offs[k], res.tbs_len[k]) == p["tbs"]
        assert (res.issuer_name_off[k] - offs[k], res.issuer_name_len[k]) == p["name"]
        assert res.crl_first[k] == e and res.crl_entries[k] == len(p["entries"]), k
        for i, pe in enumerate(p["entries"]):
            g = e + i
            assert res.serial_off[g] == offs[k] + pe["serial_pos"]
            assert res.serial_len[g] == min(len(pe["serial"]), 255)
            assert res.serial(data, g) == pe["serial"][:255]
            assert (res.revoked_at[g], res.reason[g], res.entry_status[g]) == (pe["revoked_at"], pe["reason"], pe["status"]), (k, i)
            assert (res.known[g], res.known_exp_hour[g], res.known_sets[g]) == j["answers"][i], (k, i, pe["serial"])
        e += len(p["entries"])
    assert res.n_entries == e


def _same(a, b):
    for name, _ in engine.RevokedResult._CRL + engine.RevokedResult._ENTRY:
        assert np.array_equal(getattr(a, name), getattr(b, name)), name


@pytest.fixture(scope="module")
def batch():
    """The catalogue and the mutants, each CRL with a digest: issuer 4 gets only CRLs whose hand-written status is OK
    (it stays covered), issuers 0..3 the rest, and every seventh CRL a digest nobody registered."""
    cat = cc.catalogue()
    crls = [c.der for c in cat] + cc.mutants()
    want = [c.status for c in cat] + [None] * (len(crls) - len(cat))
    who = []
    for k, st in enumerate(want):
        who.append(-1 if k % 7 == 6 else 4 if st == cc.OK and k % 2 == 0 else k % 4)
    return crls, who


def _preloads(crls, who):
    """[(hour, issuer number, serial)]: every third joinable serial of the batch under its CRL's issuer, one hour of
    five, a tenth of them under a second hour, some under an expired hour; and serials no CRL revokes"""
    out = {(HOUR + 3, w, b"\x7e\x7e" + bytes([i])) for w in range(5) for i in range(60)}
    n = 0
    for k, der in enumerate(crls):
        if who[k] < 0:
            continue
        p = co.parse_crl(der)
        if p["status"] != co.CRL_OK:
            continue
        for e in p["entries"]:
            if e["status"] != co.RV_OK:
                continue
            n += 1
            if n % 3 == 0:
                out.add((HOUR + 1 + n % 5, who[k], e["serial"]))
            if n % 30 == 0:
                out.add((HOUR + 100, who[k], e["serial"]))
            if n % 11 == 0:
                out.add((HOUR - 2, who[k], e["serial"]))
    return sorted(out)


def _fill(db, issuers, pre):
    """register the issuers, preload `pre`; returns (digests, sets as crl_oracle.join takes them)"""
    _, dig = _register(db, issuers)
    groups = {}
    for h, w, s in pre:
        groups.setdefault((h, dig[w]), []).append(s)
    for (h, d), ss in groups.items():
        db.preload_known(h, d, ss)
    return dig, {k: set(v) for k, v in groups.items()}


def _digs(dig, who):
    return [UNKNOWN if w < 0 else dig[w] for w in who]


def test_catalogue_one_chunk_small_chunks_and_a_group(issuers, batch):
    crls, who = batch
    pre = _preloads(crls, who)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 18) as db:
        dig, sets = _fill(db, issuers, pre)
        digs = _digs(dig, who)
        res = db.revoked_known(crls, digs)
        _check(res, crls, digs, sets, set(dig))
        assert res.known.sum() > 1000 and (res.known_sets > 1).any()
        st = np.bincount(res.crl_status, minlength=4)
        assert min(st) > 500, st
        small = [k for k, c in enumerate(crls) if len(c) <= 4096]
        assert len(small) > 0.9 * len(crls)
        s_crls, s_digs = [crls[k] for k in small], [digs[k] for k in small]
        one = db.revoked_known(s_crls, s_digs)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 18, max_batch_bytes=4096) as db:
        _fill(db, issuers, pre)
        got = db.revoked_known(s_crls, s_digs)
        _same(got, one)
        _check(got, s_crls, s_digs, sets, set(dig))
    with engine.GpuCertGroup([0, 0, 0], table_capacity=1 << 17) as g:
        gdig, _ = _fill(g, issuers, pre)
        assert gdig == dig
        _same(g.revoked_known(crls, digs), res)


def test_serial_len_saturates_at_255(issuers):
    lens = [39, 40, 127, 128, 255, 256, 300, 1000, 65536]
    ents = [cc.ser(cc.ent(bytes([0x11]) + bytes([n % 251]) * (n - 1)), {}) for n in lens]
    der = cc.build(repl={"rc": cc.N(0x30, *ents)})
    p = co.parse_crl(der)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        _, dig = _register(db, issuers)
        db.preload_known(HOUR + 1, dig[0], [bytes([0x11]) + bytes([39]) * 38])
        res = db.revoked_known([der], [dig[0]])
    assert res.n_entries == len(lens)
    for i, n in enumerate(lens):
        assert res.serial_off[i] == p["entries"][i]["serial_pos"] and len(p["entries"][i]["serial"]) == n
        assert res.serial_len[i] == min(n, 255)
        assert res.entry_status[i] == (co.RV_OK if n <= 39 else co.RV_SERIAL_TOO_LONG)
        assert res.known[i] == (1 if n == 39 else 0)


def test_join_edges_every_length_and_near_misses(issuers):
    table = [bytes([0x10 + n]) * n for n in range(1, 40)]
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        _, dig = _register(db, issuers)
        db.preload_known(HOUR + 10, dig[0], table)
        for h in (HOUR + 50, HOUR + 30, HOUR + 40):  # the lowest hour is not the first inserted
            db.preload_known(h, dig[0], [b"\x42\x42"])
        sets = {(HOUR + 10, dig[0]): set(table)}
        for h in (HOUR + 50, HOUR + 30, HOUR + 40):
            sets[(h, dig[0])] = {b"\x42\x42"}
        crls, digs, want = [], [], []
        for s in table:
            near = [s + b"\x00", s[:-1] + bytes([s[-1] + 1])] + ([s[:-1]] if len(s) > 1 else [])
            ents = [cc.ent(x) for x in [s] + near]
            crls.append(cc.build(repl={"rc": cc.N(0x30, *ents)}))
            digs.append(dig[0])
            want += [1] + [0] * len(near)
            crls.append(cc.build(repl={"rc": cc.N(0x30, cc.ent(s))}))  # the same serial under another issuer
            digs.append(dig[1])
            want.append(0)
        crls.append(cc.build(repl={"rc": cc.N(0x30, cc.ent(b"\x42\x42"), cc.ent(b"\x42"), cc.ent(b"\x00\x42\x42"))}))
        digs.append(dig[0])
        want += [1, 0, 0]
        res = db.revoked_known(crls, digs)
    _check(res, crls, digs, sets, set(dig))
    assert res.known.tolist() == want
    assert (res.known_exp_hour[-3], res.known_sets[-3]) == (HOUR + 30, 3)
    assert set(res.known_exp_hour[res.known == 1][:-1].tolist()) == {HOUR + 10}


def _one(db, pairs):
    """revoked_known of `pairs` [(digest, [serials]) per CRL]"""
    crls = [cc.build(repl={"rc": cc.N(0x30, *[cc.ent(s) for s in ss])}) for _, ss in pairs]
    return crls, [d for d, _ in pairs], db.revoked_known(crls, [d for d, _ in pairs])


def test_crafted_collisions(issuers):
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dense, dig = _register(db, issuers)
    I = dense[2]
    full = pm.tag_collisions(I, np.random.default_rng(2), 1 << 18, full=True)[:3]
    tags = pm.tag_collisions(I, np.random.default_rng(1), 1 << 17)[:3]
    assert full and tags
    for a, b in full + tags:
        ha, hb = (int(x) for x in pm.pair_hash(pm.pair_words([I, I], [a, b])))
        assert ha & ~3 == hb & ~3
        for table in ({a: HOUR + 7, b: HOUR + 3}, {a: HOUR + 7}, {b: HOUR + 3}):
            for layout in ([[a, b]], [[a], [b]], [[b, a]]):
                with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
                    d2, g = _register(db, issuers)
                    assert d2 == dense
                    for s, h in table.items():
                        db.preload_known(h, g[2], [s])
                    sets = {(h, g[2]): {s} for s, h in table.items()}
                    crls, digs, res = _one(db, [(g[2], ss) for ss in layout])
                _check(res, crls, digs, sets, set(g))
                order = [s for ss in layout for s in ss]
                assert res.known.tolist() == [1 if s in table else 0 for s in order]
                assert res.known_exp_hour.tolist() == [table.get(s, 0) for s in order]


def test_a_cluster_on_one_home_slot_that_wraps(issuers):
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dense, _ = _register(db, issuers)
    I = dense[3]
    slots = pm.set_slots(40)
    assert slots == 128
    cl = pm.home_cluster(I, np.random.default_rng(6), slots, slots - 3, 48)
    revoked, extra = cl[:40], cl[40:]  # extra: table keys on the same home, never revoked
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:  # a fresh ctx: its set has `slots` slots
        _, dig = _register(db, issuers)
        sets = {}
        for i, s in enumerate(revoked[::2] + extra):
            h = HOUR + 1 + i % 4
            db.preload_known(h, dig[3], [s])
            sets.setdefault((h, dig[3]), set()).add(s)
        crls, digs, res = _one(db, [(dig[3], revoked[:13]), (dig[3], revoked[13:])])
    _check(res, crls, digs, sets, set(dig))
    assert res.known.tolist() == [1 - i % 2 for i in range(40)]


def test_more_than_65536_crls_in_one_call(issuers):
    kinds = [cc._min_crl(cc.min_entry(1)), cc._min_crl(cc.min_entry(2) + cc.min_entry(3)), cc._min_crl(b"")]
    n = (1 << 16) + 300
    pick = np.arange(n) % 3
    lens = np.array([len(kinds[i]) for i in pick], np.uint64)
    offs = np.zeros(n, np.uint64)
    offs[1:] = np.cumsum(lens)[:-1]
    data = np.frombuffer(b"".join(kinds[i] for i in pick.tolist()), np.uint8)
    per = np.array([1, 2, 0])[pick]
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        _, dig = _register(db, issuers)
        db.preload_known(HOUR + 1, dig[0], [b"\x03"])
        res = db.revoked_known((data, offs, lens), [dig[0]] * n)
    assert (res.crl_status == co.CRL_OK).all()
    assert np.array_equal(res.crl_entries, per)
    first = np.zeros(n, np.uint64)
    first[1:] = np.cumsum(per)[:-1]
    assert np.array_equal(res.crl_first, first) and res.n_entries == int(per.sum())
    for k in list(range(65530, 65542)) + [0, n - 1]:
        p = co.parse_crl(kinds[pick[k]])
        for i, e in enumerate(p["entries"]):
            g = int(first[k]) + i
            assert res.serial_off[g] == offs[k] + e["serial_pos"]
            assert res.known[g] == (1 if e["serial"] == b"\x03" else 0)


def _crl_of(size: int) -> bytes:
    """a CRL of exactly `size` bytes, its signature padded"""
    content = b"".join(cc.min_entry(i) for i in range(20))
    s = size - len(cc._min_crl(content, 1)) - 4
    while len(cc._min_crl(content, s)) < size:
        s += 1
    der = cc._min_crl(content, s)
    assert len(der) == size
    return der


def test_staging_budget_edge_and_entry_cap_over_three_chunks(issuers):
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16, max_batch_bytes=4096) as db:
        _, dig = _register(db, issuers)
        res = db.revoked_known([_crl_of(4096)], [dig[0]])
        assert res.crl_status[0] == co.CRL_OK and res.n_entries == 20
        with pytest.raises(CtmrError) as ei:
            db.revoked_known([_crl_of(4097)], [dig[0]])
        assert ei.value.code == capi.E_BATCH_TOO_LARGE
        # nine CRLs of 1300 bytes: three to a chunk of 4096
        crls = [_crl_of(1300) for _ in range(9)]
        digs = [dig[k % 3] for k in range(9)]
        need = db.revoked_known(crls, digs).n_entries
        assert need == 180
        full = db.revoked_known(crls, digs, entry_cap=need)
        _check(full, crls, digs, {}, set(dig))
        with pytest.raises(CtmrError) as ei:
            db.revoked_known(crls, digs, entry_cap=need - 1)  # the overflow is in the last chunk
        assert ei.value.code == capi.E_BATCH_TOO_LARGE and ei.value.n_entries == need


def test_each_chain_alone_and_a_large_crl_among_small_ones(issuers):
    chains = [c for c in cc.catalogue() if c.name.startswith("split_chain_") or c.name.startswith("split_tail_")]
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        _, dig = _register(db, issuers)
        for c in chains:  # each CRL sets its chunk's round count
            res = db.revoked_known([c.der], [dig[0]])
            assert res.crl_status[0] == c.status, c.name
            assert res.n_entries == (len(c.entries) if c.status == co.CRL_OK else 0), c.name
        large = _crl_of(300_000)
        small = [c.der for c in chains]
        crls = small[:20] + [large] + small[20:]
        digs = [dig[0]] * len(crls)
        res = db.revoked_known(crls, digs)
        _check(res, crls, digs, {}, set(dig))


def test_cascade_over_the_catalogue(issuers, batch):
    crls, who = batch
    pre = _preloads(crls, who)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 18) as db:
        dig, _ = _fill(db, issuers, pre)
        digs = _digs(dig, who)
        known = db.revoked_known(crls, digs)
        cas = db.revoked_cascade(crls, digs, NOW, b"catalogue")
    assert np.array_equal(cas.crl_status, known.crl_status)
    # the header's R / S rule: live records of the covered issuers, R = revoked by a joinable entry of an OK CRL
    status = [co.join(co.parse_crl(c), d, {}, set(dig))["status"] for c, d in zip(crls, digs)]
    batch_issuers = {d for d in digs if d in set(dig)}
    covered = {d for d in batch_issuers if all(s == co.CRL_OK for s, dd in zip(status, digs) if dd == d)}
    revoked = {(d, e["serial"]) for c, d, s in zip(crls, digs, status) if s == co.CRL_OK
               for e in co.parse_crl(c)["entries"] if e["status"] == co.RV_OK}
    R = [(h, w, s) for h, w, s in pre if h * 3600 > NOW and dig[w] in covered and (dig[w], s) in revoked]
    S = [(h, w, s) for h, w, s in pre if h * 3600 > NOW and dig[w] in covered and (dig[w], s) not in revoked]
    assert covered == {dig[4]} and len(R) > 100
    assert (cas.issuers, cas.revoked, cas.valid) == (len(covered), len(R), len(S))
