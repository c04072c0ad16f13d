"""IssuerMetadata's string reducers slot by slot: the (issuer, kind, bytes) identities of issuer Names and CRL-DP values
(K_meta: first_issuer_dn / first_crldp) and the (issuer, hour) first-seen index (first_issuer_hour), on hand-built
certificates that reach the rare paths -- strings that differ only in their partial last word, one Name under two
issuers, one byte string as a Name and as a CRL-DP value, crafted first-hash collisions, clusters that wrap, full
tables, contention, eviction, shards.  Every output is compared with the oracle, and every table left behind is decoded
from a snapshot and checked against the models of tests/metamodel.py and tests/keymodel.py."""
import hashlib

import numpy as np
import pytest

import der_build as D
import keymodel as K
import metamodel as M
from conftest import NOW_NS, pack

pytestmark = pytest.mark.gpu

PATH_FIELDS = ("status", "exp_hour", "serial_off", "serial_len", "was_unknown", "first_issuer_hour")
META_FIELDS = ("issuer_name_off", "issuer_name_len", "crldp_off", "crldp_len", "first_issuer_dn", "first_crldp")
SPANS = ("exp_hour", "serial_off", "serial_len") + META_FIELDS[:4]  # defined where the leaf parsed
ISSUERS = (M.CA.der, M.CA_REKEYED.der)


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def compare(got, want, n=None):
    n = want.status.size if n is None else n
    parsed = want.status[:n] != 1
    for f in PATH_FIELDS + META_FIELDS:
        a, b = getattr(got, f)[:n], getattr(want, f)[:n]
        if f in SPANS:
            a, b = a[parsed], b[parsed]
        bad = np.nonzero(a != b)[0]
        assert bad.size == 0, (f, bad[:10], a[bad[:10]], b[bad[:10]])
    if got.sha256 is not None:
        assert np.array_equal(got.sha256[:n], want.sha256[:n])


def ders_of(items):
    return [x.der if isinstance(x, D.Built) else x for x in items]


class Both:
    """One GPU database (or group) and the oracle fed the same batches; the models follow the tables."""

    def __init__(self, eng, ora, group=None, **kw):
        kw.setdefault("table_capacity", 1 << 12)
        kw.setdefault("pair_capacity_log2", 10)
        kw.setdefault("meta_capacity_log2", 12)
        self.group = group
        mk = (lambda **k: eng.GpuCertGroup(group, **k)) if group else (lambda **k: eng.GpuCertDatabase(**k))
        self.db = mk(log_expired_entries=True, **kw)
        self.pair_slots, self.meta_slots = 1 << kw["pair_capacity_log2"], 1 << kw["meta_capacity_log2"]
        self.odb = ora.DB(b"", True)
        self.iblob, self.ioffs = pack(list(ISSUERS))
        self.dense = self.db.register_issuers(self.iblob, self.ioffs)
        assert self.dense.tolist() == [0, 1]
        self.keys, self.meta = K.KeyModel(), M.MetaModel()

    def store(self, items, idx=None, want_sha=True):
        ders = ders_of(items)
        blob, offs = pack(ders)
        idx = np.zeros(len(ders), np.uint32) if idx is None else np.asarray(idx, np.uint32)
        want = self.odb.process(blob, offs, self.iblob, self.ioffs, idx, NOW_NS)
        got = self.db.store_batch(blob, offs, self.iblob, self.ioffs, idx, NOW_NS, want_sha=want_sha, want_meta=True)
        compare(got, want)
        self.keys.add(blob, offs, want, self.dense[idx])
        self.meta.add(ders, want, self.dense[idx])
        return got, want

    def check(self):
        """Every slot of every table left behind; returns the decoded meta table(s)."""
        assert {k: v for k, v in self.db.issuer_counts().items() if v} == {k: v for k, v in self.odb.issuer_counts().items() if v}
        snap = self.db.snapshot()
        if self.group:
            shards = M.decode_group_snapshot(snap, self.pair_slots, self.meta_slots)
            total = sum(M.check_meta(sh["meta"], self.meta, len(shards), r) for r, sh in enumerate(shards))
            assert total == len(self.meta.first)
            return [sh["meta"].copy() for sh in shards]
        K.check_table(snap, self.keys, self.db.table_stats()[0])
        meta = M.decode_snapshot(snap)["meta"]
        assert M.check_meta(meta, self.meta) == len(self.meta.first)
        return meta.copy()

    def close(self):
        self.db.close()


def filler(n, salt, **kw):
    """n new certificates under the default Name, no CRL-DP: one string identity between them."""
    base = M.leaf(salt, **kw)
    return [M.reserial(base, salt + 1 + k) for k in range(n)]


def slots_with_h1(meta, h1):
    return np.nonzero(meta["h1"] == np.uint64(h1))[0].tolist()


# ------------------------------------------------------------------------------------------------ 1. byte edges

def test_byte_edges_of_the_identity(eng, ora):
    """Names and CRL-DP values of every length mod 8 that differ only in their last byte; an empty CRL-DP value; two
    CRL-DP extensions (the last one counts)."""
    dn, crl = M.tail_pairs(M.KIND_DN, 1000), M.tail_pairs(M.KIND_CRLDP, 2000)
    empty = M.leaf(3000, extensions=[D.Ext(D.CRLDP_OID, b"")])
    two = M.leaf(3001, extensions=[D.crl_distribution_points(M.URI + b"first"), D.crl_distribution_points(M.URI + b"second")])
    assert empty.crldp[1] == 0 and M.crldp_bytes(two).endswith(b"second")
    seq = [b for p in dn + crl for b in p] + [empty, two]
    b = Both(eng, ora)
    try:
        got, _ = b.store(seq)
        assert got.first_issuer_dn[:16].all() and got.first_crldp[16:32].all()
        assert got.crldp_len[32] == 0 and got.first_crldp[32] == 0
        assert (int(got.crldp_off[33]), int(got.crldp_len[33])) == two.crldp and got.first_crldp[33] == 1
        b.check()
        # repeats of every member, and new certificates carrying the B members' strings: nothing is first
        got, _ = b.store(seq + [M.reserial(y, 9000 + k) for k, (_, y) in enumerate(dn + crl)])
        assert not got.first_issuer_dn.any() and not got.first_crldp.any()
        b.check()
    finally:
        b.close()


# ------------------------------------------------------------------------------------------------ 2. what the identity includes

def test_identity_includes_issuer_and_kind(eng, ora):
    rk, kd = M.rekeyed_pair(4000), M.kind_pair(4100)
    b = Both(eng, ora)
    try:
        got, _ = b.store(list(rk) + list(kd), idx=[0, 1, 0, 0])
        assert got.first_issuer_dn.tolist() == [1, 1, 1, 0]    # one Name under two issuers; the kind pair shares a Name
        assert got.first_crldp.tolist() == [0, 0, 0, 1]        # the Name bytes again, as a CRL-DP value
        b.check()
        got, _ = b.store([M.reserial(x, 4200 + k) for k, x in enumerate(list(rk) + list(kd))], idx=[1, 0, 0, 0])
        assert not got.first_issuer_dn.any() and not got.first_crldp.any()
        b.check()
    finally:
        b.close()


# ------------------------------------------------------------------------------------------------ 3. crafted h1 collisions

COLLISION_EDGES = ((3, 7), (10, 40), (130, 131), (690, 710), (699, 700), (1390, 1401))


def _collision_pairs(salt, edges, mask):
    out = []
    for e in range(len(edges)):
        kind = M.KIND_DN if e % 2 == 0 else M.KIND_CRLDP
        t = M.target_h1(mask - 20 + e, mask, salt + e)
        out.append((kind, t) + M.collision_pair(kind, salt + 100 * e, 0, t))
    return out


@pytest.mark.parametrize("want_sha", (True, False), ids=("stream", "light"))
def test_h1_collisions_in_one_batch(eng, ora, want_sha):
    """Pairs with one h1 and different h2 inside a warp, across warps and across host-pipeline stages (700 entries)."""
    pairs = _collision_pairs(5000, COLLISION_EDGES, (1 << 12) - 1)
    seq = filler(1500, 1_000_000)
    for (lo, hi), (_, _, x, y) in zip(COLLISION_EDGES, pairs):
        seq[lo], seq[hi] = x, y
    repeats = [M.reserial(z, 5900 + k) for k, p in enumerate(pairs) for z in p[2:]]
    b = Both(eng, ora, max_batch_entries=700)
    try:
        got, _ = b.store(seq + repeats, want_sha=want_sha)
        for (lo, hi), (kind, _, _, _) in zip(COLLISION_EDGES, pairs):
            bits = got.first_issuer_dn if kind == M.KIND_DN else got.first_crldp
            assert bits[lo] == 1 and bits[hi] == 1, (lo, hi)
        assert not got.first_issuer_dn[len(seq):].any() and not got.first_crldp[len(seq):].any()
        meta = b.check()
        for kind, t, _, _ in pairs:  # both members in the probe chain of their shared home slot
            at = slots_with_h1(meta, t)
            assert len(at) == 2 and all((s - M.home_slot(t, meta.size - 1)) % meta.size < 64 for s in at)
    finally:
        b.close()


def test_h1_collisions_across_batches_and_restore(eng, ora):
    pairs = _collision_pairs(6000, ((0, 0),) * 4, (1 << 12) - 1)
    b = Both(eng, ora)
    try:
        got, _ = b.store([p[2] for p in pairs] + filler(40, 6500))
        assert (got.first_issuer_dn[:4] | got.first_crldp[:4]).all()
        got, _ = b.store([p[3] for p in pairs[:2]] + [M.reserial(p[2], 6600 + k) for k, p in enumerate(pairs)])
        assert (got.first_issuer_dn[:2] | got.first_crldp[:2]).all()
        assert not (got.first_issuer_dn[2:] | got.first_crldp[2:]).any()
        b.check()
        snap = b.db.snapshot().copy()
    finally:
        b.close()
    b2 = Both(eng, ora)
    try:
        b2.db.restore(snap)
        b2.odb, b2.keys, b2.meta = b.odb, b.keys, b.meta
        got, _ = b2.store([p[3] for p in pairs[2:]] + [M.reserial(p[3], 6700 + k) for k, p in enumerate(pairs[:2])])
        assert (got.first_issuer_dn[:2] | got.first_crldp[:2]).all()
        assert not (got.first_issuer_dn[2:] | got.first_crldp[2:]).any()
        meta = b2.check()
        for _, t, _, _ in pairs:
            assert len(slots_with_h1(meta, t)) == 2
    finally:
        b2.close()


# ------------------------------------------------------------------------------------------------ 4. clusters and wrap

def test_cluster_and_wrap(eng, ora):
    """A 2^10 string table: 64 identities with one home slot, and identities homed on the last four slots, whose probe
    chains wrap to slot 0."""
    mask = (1 << 10) - 1
    cluster = [M.crafted(M.leaf(7000 + k, org=b"Cluster %04d " % k + M.ORG), M.KIND_DN, 0, M.target_h1(300, mask, k))
               for k in range(64)]
    wrap = []
    for k in range(16):
        t = M.target_h1(mask - 3 + k % 4, mask, 100 + k)
        if k % 2:
            wrap.append(M.crafted(M.leaf(7100 + k, uri=M.URI + b"wrap/%04d/0123456789" % k), M.KIND_CRLDP, 0, t))
        else:
            wrap.append(M.crafted(M.leaf(7100 + k, org=b"Wrap %04d " % k + M.ORG), M.KIND_DN, 0, t))
    b = Both(eng, ora, meta_capacity_log2=10)
    try:
        seq = [x for pair in zip(cluster[:16], wrap) for x in pair] + cluster[16:]
        got, _ = b.store(seq)
        assert got.first_issuer_dn.sum() + got.first_crldp.sum() == 64 + 16 + 1  # + the wrap leaves' CRL-DP Name
        meta = b.check()
        assert meta["h1"][0] != 0 and (meta["h1"][mask - 3:] != 0).all()
        assert (meta["h1"][300:364] != 0).all()
        got, _ = b.store([M.reserial(x, 7300 + k) for k, x in enumerate(seq)])
        assert not got.first_issuer_dn.any() and not got.first_crldp.any()
        b.check()
    finally:
        b.close()


# ------------------------------------------------------------------------------------------------ 5. full tables

def test_meta_table_full(eng, ora):
    from ct_mapreduce_b200.capi import E_META_TABLE_FULL, CtmrError
    names = [M.leaf(8000 + k, cn=b"Full %04d" % k) for k in range(256)]
    b = Both(eng, ora, meta_capacity_log2=8)
    try:
        got, _ = b.store(names)
        assert got.first_issuer_dn.all()
        meta = b.check()
        assert (meta["h1"] != 0).all()
        got, _ = b.store([M.reserial(x, 8300 + k) for k, x in enumerate(names[::3])])
        assert got.was_unknown.all() and not got.first_issuer_dn.any()
        b.check()
        blob, offs = pack([M.leaf(8600, cn=b"One more").der])
        with pytest.raises(CtmrError) as e:
            b.db.store_batch(blob, offs, b.iblob, b.ioffs, np.zeros(1, np.uint32), NOW_NS, want_meta=True)
        assert e.value.code == E_META_TABLE_FULL
    finally:
        b.close()


def test_pair_table_full(eng, ora):
    from ct_mapreduce_b200.capi import E_PAIR_TABLE_FULL, CtmrError
    hour0 = D.exp_hour(D.NOT_AFTER)
    sets = [[M.leaf(8700 + 10 * h + k, not_after=(hour0 + h) * 3600 + k) for k in range(1 + h % 3)] for h in range(16)]
    b = Both(eng, ora, pair_capacity_log2=4)
    try:
        got, _ = b.store([x for s in sets for x in s])
        assert got.first_issuer_hour.sum() == 16
        b.check()
        dig = b.db.issuer_digest(0)
        for h, s in enumerate(sets):
            assert b.db.get_known_certificates(hour0 + h, dig).count() == b.odb.set_cardinality(hour0 + h, dig) == len(s)
        assert b.db.get_known_certificates(hour0 + 16, dig).count() == 0
        assert b.db.get_known_certificates(hour0, b.db.issuer_digest(1)).count() == 0
        blob, offs = pack([M.leaf(8900, not_after=(hour0 + 16) * 3600).der])
        with pytest.raises(CtmrError) as e:
            b.db.store_batch(blob, offs, b.iblob, b.ioffs, np.zeros(1, np.uint32), NOW_NS, want_meta=True)
        assert e.value.code == E_PAIR_TABLE_FULL
    finally:
        b.close()


# ------------------------------------------------------------------------------------------------ 6. lowest index wins

@pytest.mark.parametrize("stage", (0, 700), ids=("one_stage", "stages_of_700"))
def test_hot_string(eng, ora, stage):
    """One Name carried by 4096 new certificates at scattered positions of one batch, and CRL-DP values whose first
    carriers sit on the stage edges."""
    rng = np.random.default_rng(11)
    n = 8192
    hot = M.leaf(10000, org=b"Hot " + M.ORG)
    seq = filler(n, 20000)
    at = np.sort(rng.choice(n, 4096, replace=False))
    for k, i in enumerate(at):
        seq[i] = M.reserial(hot, 30000 + k)
    edge_firsts = (699, 700, 1399, 1400, 4200)
    for e, i in enumerate(edge_firsts):
        x = M.leaf(11000 + e, uri=M.URI + b"edge/%d" % e)
        for k, j in enumerate((i, i + 1, i + 350, n - 1 - e)):
            seq[j] = M.reserial(x, 40000 + 10 * e + k)
    b = Both(eng, ora, max_batch_entries=stage, table_capacity=1 << 14)
    try:
        got, _ = b.store(seq, want_sha=False)
        hot_at = [i for i in range(n) if M.name_bytes(hot) in seq[i].der[:200]]
        assert got.first_issuer_dn[hot_at].sum() == 1 and got.first_issuer_dn[hot_at[0]] == 1
        for i in edge_firsts:
            assert got.first_crldp[i] == 1
        assert got.first_crldp.sum() == len(edge_firsts)
        b.check()
    finally:
        b.close()


@pytest.mark.parametrize("want_sha", (True, False), ids=("stream", "light"))
def test_string_across_device_rounds(eng, ora, want_sha):
    """ctmr_process_device cuts n = 2^18 entries into two rounds (131072 entries each); carriers of one string straddle
    the edge, in both orders."""
    import torch
    from ct_mapreduce_b200 import capi
    n, edge = 1 << 18, 1 << 17
    ders = [b"\x30"] * n  # rejected one-byte records around the carriers
    layouts = ((edge - 1, edge, edge + 9), (edge - 40, edge + 40), (edge + 1, edge + 2, n - 2), (3, edge + 700), (edge - 700, n - 1))
    for s, pos in enumerate(layouts):
        x = M.leaf(50000 + s, org=b"Round %d " % s + M.ORG, uri=M.URI + b"round/%d" % s)
        for k, j in enumerate(pos):
            ders[j] = M.reserial(x, 50100 + 10 * s + k).der
    blob, offs = pack(ders)
    iblob, ioffs = pack(list(ISSUERS))
    idx = np.zeros(n, np.uint32)
    odb = ora.DB(b"", True)
    want = odb.process(blob, offs, iblob, ioffs, idx, NOW_NS, nthreads=8)
    dev = torch.device("cuda:0")
    dblob = torch.from_numpy(np.concatenate([blob, np.zeros(64, np.uint8)])).to(dev)
    doffs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    didx = torch.from_numpy(idx.astype(np.int32)).to(dev)
    with eng.GpuCertDatabase(table_capacity=1 << 12, log_expired_entries=True, max_issuers=16, pair_capacity_log2=10,
                             meta_capacity_log2=12) as db:
        dense = db.register_issuers(iblob, ioffs)
        t = {k: torch.zeros((n,) + sh, dtype=dt, device=dev) for k, sh, dt in (
            ("status", (), torch.uint8), ("sha", (32,), torch.uint8), ("exp_hour", (), torch.int64),
            ("soff", (), torch.int32), ("slen", (), torch.int32), ("wu", (), torch.uint8), ("fi", (), torch.uint8),
            ("noff", (), torch.int32), ("nlen", (), torch.int32), ("coff", (), torch.int32), ("clen", (), torch.int32),
            ("fdn", (), torch.uint8), ("fcrl", (), torch.uint8))}
        bt = capi.DevBatch()
        bt.blob, bt.blob_bytes, bt.offsets, bt.n = dblob.data_ptr(), int(offs[-1]), doffs.data_ptr(), n
        bt.issuer_idx, bt.issuer_map, bt.issuer_map_len = didx.data_ptr(), None, 0
        bt.first_index, bt.now_unix_ns = 0, NOW_NS
        p = lambda k: t[k].data_ptr()
        o = capi.DevOut(p("status"), p("sha") if want_sha else None, p("exp_hour"), p("soff"), p("slen"), p("wu"), p("fi"), None,
                        p("noff"), p("nlen"), p("coff"), p("clen"), p("fdn"), p("fcrl"))
        db.process_device(bt, o)
        db.check_device()
        torch.cuda.synchronize()
        h = {k: v.cpu().numpy() for k, v in t.items()}
        got = eng.BatchResult(h["status"], h["sha"] if want_sha else None, h["exp_hour"], h["soff"].astype(np.uint32),
                              h["slen"].astype(np.uint32), h["wu"], h["fi"], h["noff"].astype(np.uint32), h["nlen"].astype(np.uint32),
                              h["coff"].astype(np.uint32), h["clen"].astype(np.uint32), h["fdn"], h["fcrl"])
        compare(got, want)
        for pos in layouts:
            assert got.first_issuer_dn[list(pos)].tolist() == [1] + [0] * (len(pos) - 1), pos
            assert got.first_crldp[list(pos)].tolist() == [1] + [0] * (len(pos) - 1), pos
        keys, meta = K.KeyModel(), M.MetaModel()
        keys.add(blob, offs, want, dense[idx], first_index=0)
        meta.add(ders, want, dense[idx], first_index=0)
        snap = db.snapshot()
        K.check_table(snap, keys, db.table_stats()[0])
        assert M.check_meta(M.decode_snapshot(snap)["meta"], meta) == 2 * len(layouts)


# ------------------------------------------------------------------------------------------------ 7. pair-table chains

def _hours_homed(slots, count, mask=(1 << 10) - 1, issuer=0):
    """`count` expiry hours (after the fixed notAfter) whose (issuer, hour) pair key has its home slot in `slots`."""
    out, h = [], D.exp_hour(D.NOT_AFTER)
    while len(out) < count:
        h += 1
        if K.mix64(K.pair_key(h, issuer)) & mask in slots:
            out.append(h)
    return out


def test_pair_chain_evict_and_reset(eng, ora):
    """Several (issuer, hour) sets share a home slot near the end of a 2^10 pair table, one batch per set so that the
    chain order is the storing order.  The set with the earliest hour sits in the middle of the chain and is evicted."""
    hours = _hours_homed({1022, 1023}, 6)
    order = [hours[3], hours[4], hours[0], hours[5], hours[1], hours[2]]  # the earliest hour third
    sets = [[M.leaf(60000 + 10 * s + k, uri=M.URI + b"set/%d" % s, not_after=h * 3600 + 17 * k) for k in range(3)]
            for s, h in enumerate(order)]
    b = Both(eng, ora)
    try:
        for s in sets:
            got, _ = b.store(s)
            assert got.first_issuer_hour.tolist() == [1, 0, 0]
        _, pairs = K.decode_snapshot(b.db.snapshot())
        assert pairs["key"][1023] != 0 and pairs["key"][0] != 0  # the chain wraps to slot 0
        meta_before = b.check()
        cut = hours[0] * 3600
        assert b.db.evict_expired(cut) == b.odb.evict_expired(cut) == 3
        b.keys.evict(cut)
        dig = b.db.issuer_digest(0)
        for h in order:
            assert b.db.get_known_certificates(h, dig).count() == b.odb.set_cardinality(h, dig) == (0 if h == hours[0] else 3)
        meta_after = b.check()
        assert np.array_equal(meta_before, meta_after)  # eviction leaves the string identities alone
        got, _ = b.store(sets[2] + sets[3])
        assert got.was_unknown.tolist() == [1, 1, 1, 0, 0, 0]
        assert not got.first_issuer_hour.any() and not got.first_crldp.any()  # first seen before the eviction
        assert b.db.get_known_certificates(hours[0], dig).count() == b.odb.set_cardinality(hours[0], dig) == 3
        b.check()
        b.db.reset_device()
        z = M.decode_snapshot(b.db.snapshot())
        assert not z["meta"]["h1"].any() and not z["pairs"]["key"].any() and not z["table"]["tag"].any()
        # a reset ctx is a fresh start: compared with a fresh oracle, every set is first again
        b.odb, nxt = ora.DB(b"", True), b.keys.next_index
        b.keys, b.meta = K.KeyModel(), M.MetaModel()
        b.keys.next_index = b.meta.next_index = nxt
        got, _ = b.store(sets[0] + sets[2])
        assert got.first_issuer_hour.tolist() == [1, 0, 0, 1, 0, 0] and got.first_crldp.tolist() == [1, 0, 0, 1, 0, 0]
        b.check()
    finally:
        b.close()


# ------------------------------------------------------------------------------------------------ 8. groups

def _group_devices():
    import torch
    n = torch.cuda.device_count()
    return [pytest.param([0, 0, 0], id="three_shards_one_gpu"),
            pytest.param(list(range(n)), id="all_gpus", marks=pytest.mark.skipif(n < 2, reason="needs two GPUs"))]


@pytest.mark.parametrize("devices", _group_devices())
def test_group_shards(eng, ora, devices):
    """Identities crafted onto every owner of the group, an h1 collision on the last owner, small stages."""
    world = len(devices)
    mask = (1 << 10) - 1
    crafted = []
    for o in range(world):
        for k in range(4):
            t = M.target_h1(mask - k, mask, 10 * o + k, owner=o, world=world)
            kind = M.KIND_DN if k % 2 == 0 else M.KIND_CRLDP
            x = M.leaf(70000 + 10 * o + k, org=b"Owner %d/%d " % (o, k) + M.ORG, uri=M.URI + b"owner/%d/%d/0123456789" % (o, k))
            crafted.append(M.crafted(x, kind, 0, t))
    t = M.target_h1(5, mask, 999, owner=world - 1, world=world)
    pair = M.collision_pair(M.KIND_DN, 71000, 0, t)
    items = crafted + list(pair)
    seq = filler(7 + 23 * len(items) + 40, 72000)
    for k, x in enumerate(items):
        seq[7 + 23 * k] = x
    b = Both(eng, ora, group=devices, max_batch_entries=64, meta_capacity_log2=10)
    try:
        got, _ = b.store(seq)
        assert got.first_issuer_dn[7 + 23 * len(crafted)] == 1 and got.first_issuer_dn[7 + 23 * (len(crafted) + 1)] == 1
        shards = b.check()
        assert len(slots_with_h1(shards[world - 1], t)) == 2
        for o in range(world):
            assert (shards[o]["h1"] != 0).sum() >= 4
        got, _ = b.store([M.reserial(x, 73000 + k) for k, x in enumerate(crafted + list(pair))])
        assert not got.first_issuer_dn.any() and not got.first_crldp.any()
        b.check()
    finally:
        b.close()


# ------------------------------------------------------------------------------------------------ 9. front ends

def _chain0(dense):
    return ISSUERS[dense]


def test_front_ends_share_the_identities(eng, ora):
    """The crafted leaves of cases 1-3 through a data tile, get-entries pages and store_batch in one ctx: a string first
    seen in a tile is not first again in a page or as a leaf."""
    import tiles_oracle as to
    from ct_mapreduce_b200 import frontend as fe
    t = M.target_h1(77, (1 << 12) - 1, 5)
    rk, kd = M.rekeyed_pair(80000), M.kind_pair(80100)
    cases = [x for p in M.tail_pairs(M.KIND_DN, 80200) + M.tail_pairs(M.KIND_CRLDP, 80300) for x in p]
    cases += list(rk) + list(kd) + list(M.collision_pair(M.KIND_DN, 80400, 0, t)) + list(M.collision_pair(M.KIND_CRLDP, 80500, 0, t))
    dense = [0] * len(cases)
    dense[33] = 1
    tile_part, page_part = list(range(0, len(cases), 2)), list(range(1, len(cases), 2))
    b = Both(eng, ora)
    fps = [hashlib.sha256(d).digest() for d in ISSUERS]
    try:
        b.db.register_chain_certs(*pack(list(ISSUERS)))
        # a data tile with the even cases
        leaves = [fe.tile_leaf_x509(1_700_000_000_000 + j, cases[i].der, [fps[dense[i]]], fe.leaf_index_extension(j))
                  for j, i in enumerate(tile_part)]
        data = fe.data_tile(leaves)
        targs = (data, np.array([0], np.uint64), np.array([len(data)], np.uint32), np.array([0], np.uint64),
                 np.array([len(leaves)], np.uint16))
        r_o = to.tiles_process(ora, b.odb, *targs, dict(zip(fps, ISSUERS)), NOW_NS)
        r_g = b.db.store_tiles(*targs, NOW_NS, want_meta=True)
        assert r_g.tiles_done == 1 and (r_o.entry_status == 0).all()
        compare(r_g.path, r_o.path)
        assert r_g.path.first_issuer_dn.sum() + r_g.path.first_crldp.sum() > 0
        b.keys.add(*pack(r_o.leaves), r_o.path, np.array([dense[i] for i in tile_part]))
        b.meta.add(r_o.leaves, r_o.path, [dense[i] for i in tile_part])
        b.check()
        # get-entries pages with the odd cases, and new certificates carrying the tile's strings
        items = [(cases[i], dense[i]) for i in page_part] + [(M.reserial(cases[i], 81000 + i), dense[i]) for i in tile_part]
        text = fe.get_entries_body([(fe.merkle_tree_leaf_x509(1_700_000_100_000 + k, x.der), fe.certificate_chain([_chain0(d)]))
                                    for k, (x, d) in enumerate(items)])
        spans = fe.find_entry_spans(text)
        r_o = ora.raw_process(b.odb, text, *spans, NOW_NS)
        r_g = b.db.store_raw_entries(text, *spans, NOW_NS, want_meta=True)
        assert (r_o.entry_status == 0).all()
        assert np.array_equal(r_g.entry_status, r_o.entry_status)
        compare(r_g.path, r_o.path)
        m = len(page_part)
        assert not r_g.path.first_issuer_dn[m:].any() and not r_g.path.first_crldp[m:].any()
        b.keys.add(*pack(r_o.leaves), r_o.path, np.array([d for _, d in items]))
        b.meta.add(r_o.leaves, r_o.path, [d for _, d in items])
        b.check()
        # and as leaves: every string is known by now
        got, _ = b.store([M.reserial(x, 82000 + k) for k, x in enumerate(cases)], idx=dense)
        assert got.was_unknown.all() and not got.first_issuer_dn.any() and not got.first_crldp.any()
        b.check()
    finally:
        b.close()
