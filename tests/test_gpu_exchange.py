"""The multi-GPU key exchange entry by entry and shard by shard: K_map's route_append (both map kernels), publish_counts,
the owner passes over the inbox regions, pull_bits, the three exchange parities, plan_rounds and run_round's order.

Groups of 1, 2, 3, 5 and 8 members run on cuda:0 (ctmr_group_create accepts a repeated device; everything but the NVLink
wire is the same code), and on every GPU when there are two or more.  Leaves are built with tests/der_build.py and their
keys' owners chosen through tests/xchg_model.py, so the tests decide which lane of which warp routes to which member and
how full each inbox region is.  Every call is compared with the oracle run over the batch in entry order (entry i of a
call has global index next_index + i), and after every case each shard is decoded from the group snapshot and held
against the model: its known-certificate table and pair table slot by slot (no key or pair another member owns), its
per-issuer histogram exactly, its status counters against the members that mapped the entries (plan_rounds restated),
the cardinality of every set, and the group's sums.

The last test runs the collective ctmr_process_device in two processes on one GPU, with rounds of exactly X entries and
a refusal one entry above."""
import os

import numpy as np
import pytest

import der_build as D
import keymodel as K
import metamodel as M
import xchg_model as X
from conftest import NOW_NS, pack
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

PAIR_LOG2 = META_LOG2 = 12
OUTPUTS = ("status", "was_unknown", "first_issuer_hour")
PARSED = ("exp_hour", "serial_off", "serial_len")


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def _sizes():
    import torch
    out = [pytest.param([0] * w, id="%d_on_gpu0" % w) for w in (1, 2, 3, 5, 8)]
    n = torch.cuda.device_count()
    out.append(pytest.param(list(range(min(n, 8))), id="all_gpus", marks=pytest.mark.skipif(n < 2, reason="needs two GPUs")))
    return out


def _kernel():
    return pytest.mark.parametrize("want_sha", (True, False), ids=("stream", "light"))


class Ex:
    """A group and the oracle fed the same calls; the models follow every shard."""

    def __init__(self, eng, ora, devices, want_sha, **kw):
        kw.setdefault("table_capacity", 1 << 12)
        kw.setdefault("max_batch_entries", 96)
        self.W, self.want_sha = len(devices), want_sha
        self.E, self.B = X.stage_budget(kw["max_batch_entries"], kw.get("max_batch_bytes", 0))
        self.g = eng.GpuCertGroup(devices, issuer_cn_filter=X.CN_FILTER, max_issuers=64, pair_capacity_log2=PAIR_LOG2,
                                  meta_capacity_log2=META_LOG2, **kw)
        self.odb = ora.DB(X.CN_FILTER, False)
        self.iblob, self.ioffs = pack(X.issuers())
        dense = self.g.register_issuers(self.iblob, self.ioffs)
        assert dense[:X.N_ISSUERS].tolist() == list(range(X.N_ISSUERS)) and dense[X.BAD_ISSUER] == 0xFFFFFFFE
        self.digests = [self.g.issuer_digest(k) for k in range(X.N_ISSUERS)]
        self.keys = K.KeyModel()
        self.status = np.zeros((self.W, X.STATUS_COUNT), np.uint64)
        self.plans = []
        self.counter_shift = np.zeros(X.STATUS_COUNT, np.int64)   # oracle status counts the group does not keep

    def store(self, entries):
        """entries: [(der, issuer_idx, tag)] (tag: the key's owner, a REJECTED kind, or None).  Every output of every entry
        against the oracle; returns (got, want)."""
        ders = [e[0] for e in entries]
        idx = np.array([e[1] for e in entries], np.uint32)
        blob, offs = pack(ders)
        # the oracle keeps serials of any length; the GPU declines those longer than a key record holds
        # (CTMR_ST_SERIAL_TOO_LONG, tests/test_gpu_parity.py).  The oracle sees them without an issuer: the same outputs
        # and no state, then their status is the GPU's.
        long = np.array([e[2] == "long_serial" for e in entries], bool)
        want = self.odb.process(blob, offs, self.iblob, self.ioffs, np.where(long, X.NO_ISSUER, idx).astype(np.uint32), NOW_NS)
        assert (want.status[long] == 5).all()
        want.status[long] = 7
        self.counter_shift[5] += int(long.sum())
        self.counter_shift[7] -= int(long.sum())
        got = self.g.store_batch(blob, offs, self.iblob, self.ioffs, idx, NOW_NS, want_sha=self.want_sha)
        n = len(ders)
        for f in OUTPUTS + (("sha256",) if self.want_sha else ()):
            a, b = getattr(got, f), getattr(want, f)
            bad = np.nonzero((a != b).reshape(n, -1).any(axis=1))[0]
            assert bad.size == 0, (f, bad[:12], a[bad[:12]], b[bad[:12]])
        parsed = want.status != 1
        for f in PARSED:
            assert np.array_equal(getattr(got, f)[parsed], getattr(want, f)[parsed]), f
        # the oracle's own check of what was stored: a valid key is owned where the builders meant it to be
        for (_, i, tag), st, h in zip(entries, want.status, want.exp_hour):
            if isinstance(tag, int):
                assert st == 0 and X.key_owner(int(h), int(i), self.W) == tag
            elif tag is not None:
                assert st != 0, tag
        plan = X.plan_rounds(offs, self.W, self.E, self.B) if n else []
        self.plans.append(plan)
        if n:
            self.status += X.status_by_member(plan, want.status, self.W)
        self.keys.add(blob, offs, want, np.where(idx < X.N_ISSUERS, idx, 0))
        return got, want

    def preload(self, hour, issuer, serials):
        """The same set seeded into both: the group's preload, and leaves carrying the serials stored by the oracle."""
        self.g.preload_known(hour, self.digests[issuer], serials)
        ders = [D.cert(serial=s, not_after=hour * 3600 + j).der for j, s in enumerate(serials)]
        blob, offs = pack(ders)
        r = self.odb.process(blob, offs, self.iblob, self.ioffs, np.full(len(ders), issuer, np.uint32), NOW_NS)
        assert (r.status == 0).all()
        self.counter_shift[0] += len(ders)   # a preload maps nothing
        X.preload(self.keys, hour, issuer, serials, self.keys.next_index)

    def evict(self, now_sec):
        assert self.g.evict_expired(now_sec) == self.odb.evict_expired(now_sec)
        self.keys.evict(now_sec)

    def check(self):
        """Every shard on its own, then the group's sums and every set's cardinality."""
        W = self.W
        shards = M.decode_group_snapshot(self.g.snapshot(), 1 << PAIR_LOG2, 1 << META_LOG2)
        exp = X.shard_expectations(self.keys, W)
        for r, (sh, ex) in enumerate(zip(shards, exp)):
            K.check_table((sh["table"], sh["pairs"]), ex.model, self.g.members[r].table_stats()[0], owner=(X.key_owner, W, r))
            hist = sh["issuer_counts"]
            want = np.zeros(hist.size, np.uint64)
            for k, v in ex.hist.items():
                want[k] = v
            assert np.array_equal(hist, want), ("histogram of shard", r, np.nonzero(hist != want)[0][:8])
            assert np.array_equal(sh["status_counts"], self.status[r]), ("status counters of shard", r, sh["status_counts"], self.status[r])
            assert np.array_equal(self.g.members[r].status_counters(), self.status[r])
        oc = self.odb.issuer_counts()
        assert {k: v for k, v in self.g.issuer_counts().items() if v} == {k: v for k, v in oc.items() if v}
        counters = (self.odb.filter_counters().astype(np.int64) - self.counter_shift).astype(np.uint64)
        assert np.array_equal(self.g.status_counters(), counters)
        assert np.array_equal(self.status.sum(axis=0), counters)
        assert self.g.table_stats()[0] == len(self.keys.first)
        sets = {}
        for k in self.keys.first:
            sets[(k[0], k[1])] = sets.get((k[0], k[1]), 0) + 1
        for (h, i), c in set(sets.items()) | {(pk, 0) for pk in self.keys.pair_first if pk not in sets}:
            hour = X.signed_hour(h)
            assert self.g.get_known_certificates(hour, self.digests[i]).count() == self.odb.set_cardinality(hour, self.digests[i]) == c

    def close(self):
        self.g.close()


# ------------------------------------------------------------------------------------------------ T1 every group size

def _t1_calls(seed=11, calls=(700, 1, 900, 613)):
    """~20 issuers x a few hours, twins inside and across calls, every rejection status."""
    rng = np.random.default_rng(seed)
    hours = [X.BASE_HOUR + d for d in (0, 5, 17, 40)]
    made, out, salt = [], [], 100_000
    for n in calls:
        call = []
        for _ in range(n):
            u = rng.random()
            if made and u < 0.2:
                call.append(made[int(rng.integers(len(made)))])
            elif u < 0.3:
                salt += 1
                kind = X.REJECTED[salt % len(X.REJECTED)]
                call.append(X.leaf(salt, X.BASE_HOUR, kind) + (kind,))
            else:
                salt += 1
                e = X.leaf(salt, hours[int(rng.integers(len(hours)))], "ok", int(rng.integers(300, 1500)) if u > 0.8 else None) + (None,)
                made.append(e)
                call.append(e)
        out.append(call)
    return out


@_kernel()
@pytest.mark.parametrize("devices", _sizes())
def test_every_group_size(eng, ora, devices, want_sha):
    calls = _t1_calls()
    ex = Ex(eng, ora, devices, want_sha)
    try:
        for call in calls:
            ex.store(call)
            ex.check()
        assert (ex.status.sum(axis=0) > 0).all()                           # every status occurred
        got, want = ex.store([e for c in calls for e in c])                # a replay: everything known
        assert not got.was_unknown.any() and not got.first_issuer_hour.any()
        ex.check()
        if len(devices) > 1:
            per = [m.table_stats()[0] for m in ex.g.members]
            assert all(p > 0 for p in per)
    finally:
        ex.close()


# ------------------------------------------------------------------------------------------------ T2 warp routing patterns

def _t2_batch(W, salt):
    """One round: every member's slice is 8 warps of 32 entries (max_batch_entries 256), warp w of member m routed by
    pattern (w + m) mod 6, with chunk count 3 + w so that the stream kernel's length order keeps each group one warp."""
    out = []
    for m in range(W):
        for w in range(8):
            out += X.warp_entries(X.WARP_PATTERNS[(w + m) % len(X.WARP_PATTERNS)], W, m, salt + 1000 * (8 * m + w), w)
    return out


@_kernel()
@pytest.mark.parametrize("W", (3, 8))
def test_warp_routing_patterns(eng, ora, W, want_sha):
    ex = Ex(eng, ora, [0] * W, want_sha, max_batch_entries=256)
    try:
        a = _t2_batch(W, 1_000_000)
        got, want = ex.store(a)
        assert len(ex.plans[-1]) == 1
        for m in range(W):
            for w in range(8):
                lo = 256 * m + 32 * w
                assert X.warp_sets_are_fixed([len(e[0]) for e in a[256 * m:256 * m + 256]])
                kinds = X.warp_targets(X.WARP_PATTERNS[(w + m) % len(X.WARP_PATTERNS)], W, m)
                valid = np.array([not isinstance(t, str) for t in kinds])
                assert (got.was_unknown[lo:lo + 32] == valid).all(), (m, w)
        ex.check()
        # a second call: new keys, and twins of the first call's keys in other members' warps (all known)
        b = _t2_batch(W, 2_000_000)
        for j in range(0, len(b), 5):
            b[j] = a[(j * 7) % len(a)]
        ex.store(b)
        ex.check()
        got, _ = ex.store(a + b)
        assert not got.was_unknown.any()
        ex.check()
    finally:
        ex.close()


# ------------------------------------------------------------------------------------------------ T3 full and empty regions

@_kernel()
def test_full_and_empty_regions(eng, ora, want_sha):
    es, kinds = X.t3_corpus()
    ex = Ex(eng, ora, [0, 0, 0], want_sha, max_batch_entries=256, table_capacity=1 << 14)
    try:
        got, want = ex.store(es)
        plan = ex.plans[-1]
        owners = X.owners_of(es)
        _, full = X.inbox_counts(plan, owners, owners >= 0, 256)
        assert full == [0, 4, 8, 9] and len(plan) == 11
        ex.check()
        for n in (2, 1):   # calls with fewer entries than members
            part = [X.owned_leaf(400_000 + n + k, 3, (k + 1) % 3) + ((k + 1) % 3,) for k in range(n - 1)] + [es[7]]
            ex.store(part)
            ex.check()
        got, _ = ex.store(es[::-1])
        assert not got.was_unknown.any()
        ex.check()
    finally:
        ex.close()


# ------------------------------------------------------------------------------------------------ T4 lowest index wins

def _t4_corpus():
    """W = 3, 64 entries per member and round, 5 rounds.  Fillers are keys their own member owns; crafted entries:"""
    W, E, R = 3, 64, 5
    fill = [X.owned_leaf(500_000 + j, W, (j % (W * E)) // E) + ((j % (W * E)) // E,) for j in range(W * E * R)]
    at = lambda k, m, j: k * W * E + m * E + j
    A = X.owned_leaf(510_001, W, 2) + (2,)      # non-owner copy lower, same round
    B = X.owned_leaf(510_002, W, 2) + (2,)      # from two sources' regions
    C = X.owned_leaf(510_003, W, 1) + (1,)      # twice in one warp, adjacent inbox positions
    Dw = X.owned_leaf(510_004, W, 0) + (0,)     # on every member (lowest at its owner)
    D1 = X.owned_leaf(510_005, W, 1) + (1,)     # on every member (lowest at member 0)
    Ek = X.owned_leaf(510_006, W, 1) + (1,)     # rounds k and k + 3 (one parity)
    Fk = X.owned_leaf(510_007, W, 0) + (0,)     # rounds 1 and 4, owner's copy first
    places = {A: [at(0, 0, 3), at(0, 2, 12)], B: [at(0, 0, 10), at(0, 1, 6)], C: [at(0, 0, 20), at(0, 0, 21)],
              Dw: [at(0, 0, 40), at(0, 1, 40), at(0, 2, 40)], D1: [at(0, 0, 41), at(0, 1, 41), at(0, 2, 41)],
              Ek: [at(0, 0, 60), at(3, 2, 50)], Fk: [at(1, 0, 7), at(4, 1, 9)]}
    for e, ps in places.items():
        for p in ps:
            fill[p] = e
    # first_issuer_hour: one set of member 2 whose lowest new certificate arrives through the inbox from member 0, while
    # member 2 maps higher ones of the same set in the same round; and the same with the inbox copy from member 1
    sets = []
    for v, src in enumerate((0, 1)):
        iss = 7 + v
        h = X.hour_for(iss, W, 2, X.BASE_HOUR + 300)
        es = [X.leaf(iss + X.N_ISSUERS * (520_000 + 10 * v + k), h) + (2,) for k in range(3)]
        fill[at(2, src, 30)] = es[0]
        fill[at(2, 2, 5)], fill[at(2, 2, 6)] = es[1], es[2]
        sets.append((at(2, src, 30), at(2, 2, 5), at(2, 2, 6)))
    return fill, places, sets


@_kernel()
def test_lowest_index_wins_across_owner_and_inbox(eng, ora, want_sha):
    es, places, sets = _t4_corpus()
    ex = Ex(eng, ora, [0, 0, 0], want_sha, max_batch_entries=64)
    try:
        got, _ = ex.store(es)
        assert len(ex.plans[-1]) == 5
        for e, ps in places.items():
            assert got.was_unknown[ps].tolist() == [1] + [0] * (len(ps) - 1), ps
        for lo, a, b in sets:
            assert got.first_issuer_hour[[lo, a, b]].tolist() == [1, 0, 0]
            assert got.was_unknown[[lo, a, b]].tolist() == [1, 1, 1]
        ex.check()
    finally:
        ex.close()


# ------------------------------------------------------------------------------------------------ T5 byte-budget rounds

@_kernel()
def test_byte_budget_rounds(eng, ora, want_sha):
    rng = np.random.default_rng(5)
    W = 3
    es, made = [], []
    for j in range(1500):
        if made and j % 7 == 3:
            es.append(made[int(rng.integers(len(made)))])
            continue
        L = int(rng.choice([300, 600, 1500, 3000, 6000])) + int(rng.integers(0, 40))
        o = int(rng.integers(W))
        e = X.owned_leaf(600_000 + j, W, o, X.BASE_HOUR + j % 9, L) + (o,)
        made.append(e)
        es.append(e)
    ex = Ex(eng, ora, [0] * W, want_sha, max_batch_entries=256, max_batch_bytes=96 * 1024)
    try:
        for lo, hi in ((0, 900), (900, 1500)):
            ex.store(es[lo:hi])
        shrunk = 0
        for call in ex.plans:
            rest = sum(max(0, hi - lo) for rnd in call for _, lo, hi in rnd)
            for rnd in call:
                q = max(hi - lo for _, lo, hi in rnd)
                shrunk += q < min(ex.E, -(-rest // W))
                rest -= sum(hi - lo for _, lo, hi in rnd)
        assert shrunk > 0
        ex.check()
    finally:
        ex.close()


# ------------------------------------------------------------------------------------------------ T6 preload and eviction

@_kernel()
@pytest.mark.parametrize("W", (3, 5))
def test_preload_and_eviction_per_shard(eng, ora, W, want_sha):
    """Preloaded sets on every shard, eviction at a cut that splits each shard's sets, exact histograms on every shard (the
    owner adds and the owner subtracts: no shard's count wraps), a replay."""
    cut_hour = X.BASE_HOUR + 500
    ex = Ex(eng, ora, [0] * W, want_sha)
    try:
        pre = []
        for o in range(W):
            for v, after in enumerate((X.BASE_HOUR, cut_hour + 10)):
                iss = (3 * o + v) % X.N_ISSUERS
                h = X.hour_for(iss, W, o, after)
                serials = [D.serial_bytes(10, salt=700_000 + 100 * o + 10 * v + j) for j in range(4)]
                ex.preload(h, iss, serials)
                pre.append((h, iss, serials))
        ex.check()
        es = []
        for j in range(600):
            o = j % W
            es.append(X.owned_leaf(710_000 + j, W, o, X.BASE_HOUR if j % 2 else cut_hour + 10) + (o,))
        for h, iss, serials in pre:   # leaves carrying preloaded serials: known
            es.append((D.cert(serial=serials[1], not_after=h * 3600 + 1).der, iss, X.key_owner(h, iss, W)))
        got, _ = ex.store(es)
        assert not got.was_unknown[600:].any()
        ex.check()
        ex.evict(cut_hour * 3600)
        shards = M.decode_group_snapshot(ex.g.snapshot(), 1 << PAIR_LOG2, 1 << META_LOG2)
        for r, sh in enumerate(shards):
            hist = sh["issuer_counts"].astype(np.uint64)
            assert (hist < np.uint64(1 << 32)).all(), ("a shard's histogram wrapped", r)
            live = [k for k in ex.keys.first if X.key_owner(k[0], k[1], W) == r]
            assert live and int(hist.sum()) == len(live)
        ex.check()
        got, _ = ex.store(es)
        assert got.was_unknown[1:600:2].all() and not got.was_unknown[0:600:2].any()   # evicted sets are new again
        ex.check()
    finally:
        ex.close()


# ------------------------------------------------------------------------------------------------ the collective device call

X_ENTRIES, STAGE = 256, 128


def _peer_own(rank, j):
    o = 1 - rank if (j // X_ENTRIES) % 2 == 0 else rank
    return X.owned_leaf(800_000 + 10_000 * rank + j, 2, o, X.BASE_HOUR + j % 11) + (o,)


def _peer_corpus(rank, n, m):
    """Rank r's first m entries for rounds of X: keys owned by the other rank in even rounds, by r itself in odd rounds.
    Some entries of an even round repeat the other rank's key one round later (owned by that rank: still remote), so the
    lower index is the copy that arrives through the inbox."""
    out = [_peer_own(rank, j) for j in range(m)]
    for j in range(0, n - X_ENTRIES, 37):
        if (j // X_ENTRIES) % 2 == 0:
            out[j] = _peer_own(1 - rank, j + X_ENTRIES)
    return out


def _peer_worker(rank, world, n, n_big):
    os.environ["CTMR_PEER_TIMEOUT_MS"] = "20000"
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi, engine, sharded
    assert capi.peer_rounds() == 8 and sharded.round_entries(n) == X_ENTRIES and sharded.round_entries(n_big) == X_ENTRIES + 1
    iblob, ioffs = pack(X.issuers())
    db = engine.GpuCertDatabase(device=0, table_capacity=1 << 13, issuer_cn_filter=X.CN_FILTER, max_issuers=64,
                                max_batch_entries=STAGE, max_round_entries=X_ENTRIES, pair_capacity_log2=PAIR_LOG2,
                                meta_capacity_log2=META_LOG2)
    sharded.attach_peers(db)
    dense = db.register_issuers(iblob, ioffs)
    es = _peer_corpus(rank, n, n_big)
    blob, offs = pack([e[0] for e in es])
    dblob = torch.from_numpy(np.concatenate([blob, np.zeros(64, np.uint8)])).to(dev)
    doffs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    didx = torch.from_numpy(np.array([dense[e[1]] for e in es], np.int32)).to(dev)
    t = {k: torch.zeros((n_big,) + sh, dtype=dt, device=dev) for k, sh, dt in (
        ("status", (), torch.uint8), ("sha", (32,), torch.uint8), ("exp_hour", (), torch.int64), ("wu", (), torch.uint8),
        ("fi", (), torch.uint8))}
    o = capi.DevOut(t["status"].data_ptr(), t["sha"].data_ptr(), t["exp_hour"].data_ptr(), None, None, t["wu"].data_ptr(),
                    t["fi"].data_ptr(), None)

    def batch(m):
        b = capi.DevBatch()
        b.blob, b.blob_bytes, b.offsets, b.n = dblob.data_ptr(), int(offs[m]), doffs.data_ptr(), m
        b.issuer_idx, b.issuer_map, b.issuer_map_len = didx.data_ptr(), None, 0
        b.first_index, b.now_unix_ns = 0, NOW_NS
        return b

    torch.cuda.synchronize(dev)
    dist.barrier()
    db.process_device(batch(n), o)
    torch.cuda.synchronize(dev)
    db.check_device()
    res = {k: v[:n].cpu().numpy() for k, v in t.items()}
    res["counts"] = db.issuer_counts()
    res["status_counts"] = db.status_counters()
    res["used"] = db.table_stats()[0]
    dist.barrier()
    # one entry more per round than the regions hold: both ranks refuse before any barrier, nothing changes
    try:
        db.process_device(batch(n_big), o)
        res["refused"] = None
    except capi.CtmrError as e:
        res["refused"] = e.code
    torch.cuda.synchronize(dev)
    res["after"] = (db.issuer_counts(), db.status_counters(), db.table_stats()[0])
    dist.barrier()
    db.close()
    dist.destroy_process_group()
    return res


@pytest.mark.timeout(600)
def test_collective_device_call_rounds_of_exactly_x(ora):
    from ct_mapreduce_b200 import capi, sharded
    world = 2
    n = next(m for m in range(1, 4000) if X.device_round_entries(m, 8) == X_ENTRIES)
    n_big = next(m for m in range(n, 4000) if X.device_round_entries(m, 8) == X_ENTRIES + 1)
    outs = run_ranks(_peer_worker, world, (n, n_big), timeout=500)
    # the oracle over the order the collective call defines
    shard = [_peer_corpus(r, n, n) for r in range(world)]
    slices = list(sharded.sequential_order(n, world, 8))
    order = [shard[r][j] for r, lo, hi in slices for j in range(lo, hi)]
    blob, offs = pack([e[0] for e in order])
    iblob, ioffs = pack(X.issuers())
    odb = ora.DB(X.CN_FILTER, False)
    idx = np.array([e[1] for e in order], np.uint32)
    want = odb.process(blob, offs, iblob, ioffs, idx, NOW_NS)
    pos = 0
    for r, lo, hi in slices:
        k = hi - lo
        for name, w in (("status", want.status), ("sha", want.sha256), ("wu", want.was_unknown), ("fi", want.first_issuer_hour)):
            assert np.array_equal(outs[r][name][lo:hi], w[pos:pos + k]), (name, r, lo)
        pos += k
    # the even rounds filled both ranks' regions exactly; the odd ones left them empty
    for r in range(world):
        owners = X.owners_of(shard[r])
        for k in range(8):
            lo, hi = k * X_ENTRIES, min(n, (k + 1) * X_ENTRIES)
            away = int((owners[lo:hi] == 1 - r).sum())
            assert away == ((hi - lo) if k % 2 == 0 else 0), (r, k, away)
    # every rank's histogram is exactly the keys it owns
    km = K.KeyModel()
    km.add(blob, offs, want, idx, first_index=0)
    exp = X.shard_expectations(km, world)
    oc = odb.issuer_counts()
    for r in range(world):
        got = {d: v for d, v in outs[r]["counts"].items() if v}
        assert sum(got.values()) == len(exp[r].model.first) == outs[r]["used"]
    total = {}
    for r in range(world):
        for d, v in outs[r]["counts"].items():
            total[d] = total.get(d, 0) + v
    assert {d: v for d, v in total.items() if v} == oc
    assert np.array_equal(outs[0]["status_counts"] + outs[1]["status_counts"], odb.filter_counters())
    for r in range(world):
        assert outs[r]["refused"] == capi.E_BATCH_TOO_LARGE
        assert outs[r]["after"][0] == outs[r]["counts"] and np.array_equal(outs[r]["after"][1], outs[r]["status_counts"])
        assert outs[r]["after"][2] == outs[r]["used"]
