"""ctmr_reset_device empties the known-certificate, pair and string-identity tables by advancing an epoch, not by clearing
them: slots of an earlier epoch stay in memory and must count as empty everywhere.  A ctx that processes X, resets and
processes Y must agree with a ctx that processes Y alone on every output: the map outputs and membership bits, the
IssuerMetadata first-seen bits, the issuer and status counters, table_stats, the cardinality of every (issuer, hour) set,
and the contents of its snapshot and checkpoint.  Y repeats serials and sets of X, and the tables are small enough for
Y's probe chains to cross X's stale slots.  The same holds on a group, on two peer ranks, across the epoch's wrap
(after 2^16 - 1 resets), and for the CRL calls, which must not see X's certificates.  Marked gpu."""
import numpy as np
import pytest

import checkpoint_model as ckm
import crl_build as cb
from conftest import NOW_NS
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

N = 1200
NOW = NOW_NS // 10**9
KW = dict(table_capacity=1 << 12, log_expired_entries=True, max_issuers=1024, pair_capacity_log2=12, meta_capacity_log2=12)
FIELDS = ("status", "sha256", "exp_hour", "was_unknown", "first_issuer_hour", "first_issuer_dn", "first_crldp")


def corpus():
    """the same entries in the workers and in the parent: X = [0, N), Y = [N/2, 3N/2) repeats half of X"""
    from oracle import oracle
    cfg = oracle.synth_cfg(2 * N, n_issuers=24, len_mode=1, len_lo=512, len_hi=2500, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, 2 * N)
    iblob, ioffs = oracle.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def batch(c, lo, hi):
    blob, offs, idx, iblob, ioffs = c
    return blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi]


X, Y = (0, N), (N // 2, N // 2 + N)
EARLIER = [(N // 4, N // 4 + N // 2), (N, 2 * N)]   # further batches before Y in the wrap test
EPOCH_MAX = 0xFFFF   # the last epoch (ctmr_common.cuh kEpochMax); the reset after it clears the tables


def records(ck) -> dict:
    """a checkpoint's contents independent of where the keys landed in the tables: header fields and sorted records"""
    p = ckm.decode_part(ck)
    out = {k: p[k] for k in ("n_issuers", "next_index", "n_keys", "n_pairs", "n_meta")}
    out["status"] = p["status"].tolist()
    out["digests"] = p["digests"]
    for k in ("keys", "pairs", "meta"):
        out[k] = sorted(r.tobytes() for r in p[k])
    return out


def observe(db, res, c, digs, lo, hi, snapshot=True) -> dict:
    """everything the comparison covers, after db processed entries [lo, hi) into res"""
    _, _, idx, _, _ = c
    out = {f: getattr(res, f).copy() for f in FIELDS}
    out["counts"] = {d: v for d, v in db.issuer_counts().items() if v}
    out["status_counts"] = db.status_counters().tolist()
    out["stats"] = db.table_stats()
    ok = res.status == 0
    sets = {(int(h), digs[int(i)]) for h, i in zip(res.exp_hour[ok], idx[lo:hi][ok])}
    sets |= {(h + 1, d) for h, d in sorted(sets)[:20]}   # sets next to them, never written
    out["card"] = {s: db.get_known_certificates(*s).count() for s in sorted(sets)}
    out["checkpoint"] = records(db.checkpoint())
    if snapshot:
        out["snapshot"] = db.snapshot().copy()
    return out


def x_sets(db, res, c, digs):
    """the (hour, digest) sets of X's stored entries"""
    _, _, idx, _, _ = c
    ok = res.status == 0
    return sorted({(int(h), digs[int(i)]) for h, i in zip(res.exp_hour[ok], idx[X[0]:X[1]][ok])})


def assert_same(got, want):
    assert got.keys() == want.keys()
    for k in want:
        if isinstance(want[k], np.ndarray):
            assert np.array_equal(got[k], want[k]), k
        else:
            assert got[k] == want[k], k


def snapshot_contents(snap, make):
    """a snapshot's contents, as the checkpoint of a ctx it is restored into; and that ctx's own snapshot"""
    with make() as t:
        t.restore(snap)
        return records(t.checkpoint()), t.snapshot().copy()


def run_reset_then_y(make, c, empty_resets=0, earlier=()):
    """db: X, `empty_resets` resets, then for each earlier batch a reset and the batch, then a reset and Y.  Returns
    (observations of Y, the snapshot right after the last reset, the digests)"""
    db = make()
    try:
        digs = [db.issuer_digest(int(d)) for d in db.register_issuers(c[3], c[4])]
        rx = db.store_batch(*batch(c, *X), NOW_NS, want_meta=True)
        sets_x = x_sets(db, rx, c, digs)
        for _ in range(empty_resets):
            db.reset_device()
        for lo, hi in earlier:
            db.reset_device()
            db.store_batch(*batch(c, lo, hi), NOW_NS, want_meta=True)
        db.reset_device()
        assert db.table_stats()[0] == 0 and not any(db.issuer_counts().values()) and not db.status_counters().any()
        assert all(db.get_known_certificates(*s).count() == 0 for s in sets_x)
        snap0 = db.snapshot().copy()
        ry = db.store_batch(*batch(c, *Y), NOW_NS, want_meta=True)
        return observe(db, ry, c, digs, *Y), snap0, digs
    finally:
        db.close()


def fresh_y(make, c, snap0=None):
    """a fresh ctx (restored from snap0 when given: the same next index and registry) processes Y alone"""
    with make() as db:
        if snap0 is not None:
            db.restore(snap0)
        digs = [db.issuer_digest(int(d)) for d in db.register_issuers(c[3], c[4])]
        ry = db.store_batch(*batch(c, *Y), NOW_NS, want_meta=True)
        return observe(db, ry, c, digs, *Y)


def compare(make, c, empty_resets=0, earlier=()):
    got, snap0, _ = run_reset_then_y(make, c, empty_resets, earlier)
    want = fresh_y(make, c, snap0)
    # the slots keys land in depend on the order of concurrent inserts: snapshots are compared by their contents, and
    # byte for byte after a restore (a snapshot is canonical: no epoch in it)
    sg, sw = got.pop("snapshot"), want.pop("snapshot")
    assert sg.size == sw.size
    cg, rg = snapshot_contents(sg, make)
    cw, _ = snapshot_contents(sw, make)
    assert cg == cw == got["checkpoint"]
    assert np.array_equal(rg, sg), "a snapshot restored and saved again is the same bytes"
    assert_same(got, want)
    # and a ctx that never saw anything (its own indices): every output but the index-carrying checkpoint
    alone = fresh_y(make, c)
    alone.pop("snapshot")
    for k in ("checkpoint",):
        got.pop(k), alone.pop(k)
    assert_same(got, alone)
    return got


def test_reset_then_y_equals_y_alone():
    from ct_mapreduce_b200 import engine
    c = corpus()
    got = compare(lambda: engine.GpuCertDatabase(device=0, **KW), c)
    assert got["was_unknown"].any() and got["first_issuer_dn"].any() and got["stats"][0] > KW["table_capacity"] // 8


def test_epoch_wrap_clears_the_tables():
    """X at epoch 1, then resets up to the last epoch with a batch at each of the last two, and a reset that wraps to
    epoch 1 again: X's slots carry epoch 1, so only the wrap's real clear keeps them out of Y"""
    from ct_mapreduce_b200 import engine
    c = corpus()
    compare(lambda: engine.GpuCertDatabase(device=0, **KW), c, empty_resets=EPOCH_MAX - 3, earlier=EARLIER)


def test_group_reset_then_y_equals_y_alone():
    from ct_mapreduce_b200 import engine
    c = corpus()

    def run(first):
        with engine.GpuCertGroup([0, 0], **dict(KW, table_capacity=1 << 11)) as g:
            digs = [g.issuer_digest(int(d)) for d in g.register_issuers(c[3], c[4])]
            if first:
                g.store_batch(*batch(c, *X), NOW_NS, want_meta=True)
                g.reset()
                assert g.table_stats()[0] == 0
            ry = g.store_batch(*batch(c, *Y), NOW_NS, want_meta=True)
            out = {f: getattr(ry, f).copy() for f in FIELDS}
            out["counts"] = {d: v for d, v in g.issuer_counts().items() if v}
            out["status_counts"] = g.status_counters().tolist()
            out["stats"] = g.table_stats()
            ok = ry.status == 0
            sets = sorted({(int(h), digs[int(i)]) for h, i in zip(ry.exp_hour[ok], c[2][Y[0]:Y[1]][ok])})
            out["card"] = {s: g.get_known_certificates(*s).count() for s in sets}
            return out

    assert_same(run(True), run(False))


def test_crl_calls_do_not_see_certificates_of_an_earlier_epoch():
    """CRLs that list X's serials: after a reset and Y' (disjoint from X), revoked_known, revoked_cascade and
    revoked_stash answer as on a ctx that processed Y' alone"""
    from ct_mapreduce_b200 import engine
    c = corpus()
    y2 = (N, 2 * N)

    def run(first):
        """an open db (the caller closes it): X and a reset when `first`, then Y'"""
        db = engine.GpuCertDatabase(device=0, **dict(KW, table_capacity=1 << 13))
        db.register_issuers(c[3], c[4])
        if first:
            db.store_batch(*batch(c, *X), NOW_NS)
            db.reset_device()
        db.store_batch(*batch(c, *y2), NOW_NS)
        return db

    with engine.GpuCertDatabase(device=0, **dict(KW, table_capacity=1 << 13)) as t:
        t.register_issuers(c[3], c[4])
        t.store_batch(*batch(c, *X), NOW_NS)
        part = ckm.decode_part(t.checkpoint())
    by_issuer = {}
    for r in part["keys"]:
        b = r["body"].tobytes()
        by_issuer.setdefault(part["digests"][int(r["body"][1])], set()).add(b[9:9 + b[8]])
    crls, cdigs = [], []
    for d, serials in sorted(by_issuer.items())[:6]:
        crls.append(cb.crl(entries=[cb.entry(s, 1767000000) for s in sorted(serials)]))
        cdigs.append(d)
    assert sum(len(s) for s in by_issuer.values()) > 200

    def answers(db):
        rk = db.revoked_known(crls, cdigs)
        known = (rk.n_entries, rk.crl_status.tolist(), rk.known.tolist(), rk.known_exp_hour.tolist(), rk.known_sets.tolist())
        cas = db.revoked_cascade(crls, cdigs, NOW, b"epoch")
        st = db.revoked_stash(crls, cdigs, NOW, cas.bytes)
        return known, (cas.bytes, cas.revoked, cas.valid), (st.bytes, st.revoked, st.serials)

    a = run(True)
    try:
        got = answers(a)
    finally:
        a.close()
    b = run(False)
    try:
        want = answers(b)
    finally:
        b.close()
    assert got == want
    with engine.GpuCertDatabase(device=0, **dict(KW, table_capacity=1 << 13)) as x_only:
        x_only.register_issuers(c[3], c[4])
        x_only.store_batch(*batch(c, *X), NOW_NS)
        assert sum(answers(x_only)[0][2]) > sum(got[0][2]), "the CRLs do list X's certificates"


# ---- two peer ranks on one GPU --------------------------------------------------------------------------------------
def _peer_worker(rank, world, first, early_resets=0):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import engine, sharded
    c = corpus()
    db = engine.GpuCertDatabase(device=0, **dict(KW, max_batch_entries=1024))
    if rank == 0:   # a rank whose epoch is ahead when it attaches: the ranks agree on one epoch there
        for _ in range(early_resets):
            db.reset_device()
    sharded.attach_peers(db)
    try:
        half = N // 2
        if first:   # each rank its half of X, then the collective reset
            db.store_batch(*batch(c, X[0] + rank * half, X[0] + (rank + 1) * half), NOW_NS, want_meta=True)
            db.reset_device()
            assert db.table_stats()[0] == 0
        ry = db.store_batch(*batch(c, Y[0] + rank * half, Y[0] + (rank + 1) * half), NOW_NS, want_meta=True)
        out = {f: getattr(ry, f).copy() for f in FIELDS}
        out["counts"] = {d: v for d, v in db.issuer_counts().items() if v}
        out["status_counts"] = db.status_counters().tolist()
        out["stats"] = db.table_stats()
    finally:
        db.close()
    dist.barrier()
    dist.destroy_process_group()
    return out


@pytest.mark.timeout(900)
def test_peer_ranks_reset_then_y_equals_y_alone():
    from ct_mapreduce_b200 import build
    build.build()
    got = run_ranks(_peer_worker, 2, args=(True,), timeout=400)
    want = run_ranks(_peer_worker, 2, args=(False,), timeout=400)
    for r in range(2):
        assert_same(got[r], want[r])


@pytest.mark.timeout(900)
def test_peer_ranks_attached_at_different_epochs():
    """rank 0 resets its tables before it attaches: without one epoch across the ranks, the cross-GPU string-identity
    inserts would read the other rank's slots as empty and claim them again"""
    from ct_mapreduce_b200 import build
    build.build()
    want = run_ranks(_peer_worker, 2, args=(False,), timeout=400)
    for early in (1, 3):
        got = run_ranks(_peer_worker, 2, args=(True, early), timeout=400)
        for r in range(2):
            assert_same(got[r], want[r])
