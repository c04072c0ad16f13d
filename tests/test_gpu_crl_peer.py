"""ctmr_revoked_known on one process per GPU: two ranks (on one GPU, and on two GPUs when the box has them) fill their
shards with a collective store_batch of half a synthetic corpus each and with preloads on the owning rank, then each
joins its own CRLs in collective calls.  Every output of every rank must equal ctmr_revoked_known on a one-ctx twin
that loads both ranks' checkpoint parts and runs the same rank's CRLs, and must pass the crl_oracle checks over the union
of the sets.  Also covered: round and chunk edges with 512 records per round, the read-only property, each failure rule
and the next call after it, and one rank joining a 2 M-entry CRL while the other joins 10,000 small CRLs.  Marked gpu."""

import numpy as np
import pytest

import crl_build as cb
import crl_oracle as co
import xchg_model as XM
from conftest import NOW_NS
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

H = 2048       # corpus entries each rank stores first
TAIL = 60      # entries each rank stores after the joins: one round of the collective store_batch each
X = 512        # max_batch_entries = max_round_entries: records per inbox region, i.e. per rank and round
KW = dict(table_capacity=1 << 15, max_issuers=1024, max_batch_entries=X, max_round_entries=X, max_batch_bytes=1 << 17)
SCALE_KW = dict(table_capacity=1 << 16)
FAR = 900000   # hours of the crafted sets: past every expiry of the corpus
CRL_FIELDS = ("crl_status", "crl_flags", "this_update", "next_update", "tbs_off", "tbs_len", "issuer_name_off", "issuer_name_len",
              "crl_first", "crl_entries")
ENTRY_FIELDS = ("serial_off", "serial_len", "revoked_at", "reason", "entry_status", "known", "known_exp_hour", "known_sets")
SCALE_N = 2_000_000
SCALE_STRIDE = 19997


def corpus():
    """the same entries in the workers and in the parent"""
    from oracle import oracle
    n = 2 * H + 2 * TAIL
    cfg = oracle.synth_cfg(n, n_issuers=16, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, n)
    iblob, ioffs = oracle.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def part(c, lo, hi):
    blob, offs, idx, iblob, ioffs = c
    return blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi]


def corpus_sets(c, dig):
    """{(hour, digest): serials} of the entries both ranks store first"""
    from oracle import oracle
    blob, offs, idx, iblob, ioffs = c
    want = oracle.DB().process(blob, offs[:2 * H + 1], iblob, ioffs, idx[:2 * H], NOW_NS)
    sets = {}
    for i in np.nonzero(want.status == 0)[0]:
        s = bytes(blob[offs[i] + want.serial_off[i]: offs[i] + want.serial_off[i] + want.serial_len[i]])
        sets.setdefault((int(want.exp_hour[i]), dig[idx[i]]), set()).add(s)
    return sets


def crafted(dense, dig, x_dense, x_dig):
    """[(owner rank, hour, digest, serials)]: 66 01 in two sets of issuer 0 on different ranks (the lower hour on rank 1),
    66 02 in two sets on rank 0, 66 03 in a set of the issuer only rank 0 registered (owned by rank 1).  Each rank preloads
    five serials: a preload takes indices, and the ranks' checkpoint parts must agree on the next one."""
    i0 = int(dense[0])
    a = XM.hour_for(i0, 2, 1, FAR)
    b = XM.hour_for(i0, 2, 0, a)
    c1 = XM.hour_for(i0, 2, 0, FAR + 1000)
    c2 = XM.hour_for(i0, 2, 0, c1)
    e = XM.hour_for(x_dense, 2, 1, FAR)
    f = XM.hour_for(i0, 2, 1, FAR + 2000)
    return [(1, a, dig[0], [b"\x66\x01"]), (0, b, dig[0], [b"\x66\x01", b"\x00\xaa"]), (0, c1, dig[0], [b"\x66\x02"]),
            (0, c2, dig[0], [b"\x66\x02", b"\x05"]), (1, e, x_dig, [b"\x66\x03"]), (1, f, dig[0], [b"\x66\x10", b"\x66\x11", b"\x66\x12"])]


def cases(dig, x_dig, sets):
    """[(name, (crls, digests, entry_cap) of rank 0, the same of rank 1)]; entry_cap None: the bound that suffices"""
    rng = np.random.default_rng(5)
    e = lambda s, **kw: cb.entry(s, 1767000000 - int(rng.integers(0, 10**6)), **kw)  # noqa: E731
    known = lambda d: sorted(s for (h, g), ss in sets.items() if g == d for s in ss)  # noqa: E731
    k0, k1 = known(dig[0]), known(dig[1])
    shared = cb.crl(entries=[e(s) for s in k0[50:120]] + [e(b"\x66\x01"), e(b"\x66\x02")])
    r0 = [(cb.crl(entries=[e(s) for s in k0[:200]] + [e(b"\x00\xaa"), e(b"\x66\x01"), e(b"\x66\x02", reason=1), e(b"\x05", cert_issuer=True),
                                                     e(b"\x01" * 40), e(k1[0]), e(b"\x42", seconds=False), e(k0[0], generalized=True)]), dig[0]),
          (cb.crl(entries_raw=e(b"\x05") + b"\x30\x01\x02"), dig[0]),                                   # bad entries
          (cb.crl(entries=[e(s) for s in k1[:50]], delta=True, idp=True), dig[1]),
          (shared, dig[0])]
    r1 = [(cb.crl(entries=[e(s) for s in k1[:300]] + [e(b"\x66\x01")]), dig[1]),
          (cb.crl(entries=[e(b"\x66\x01")])[:-1], dig[0]),                                                # truncated
          (cb.crl(entries=[e(s) for s in k0[:30]]), b"\xee" * 32),                                       # unknown issuer
          (cb.crl(entries=None, version=None, next_update=None), dig[1]),                                # v1, no entries
          (cb.crl(entries=[e(b"\x66\x03"), e(b"\x66\x05"), e(b"\x66\x01")]), x_dig),                     # registered by rank 0 only
          (shared, dig[0]),
          (cb.crl(entries=[e(b"\x66\x01"), e(b"\x66\x02"), e(b"\x05")]), dig[0])]
    unz = lambda lst, cap=None: ([c for c, _ in lst], [d for _, d in lst], cap)  # noqa: E731
    out = [("mix", unz(r0), unz(r1))]

    def one(n):  # one CRL of n valid entries: every third a known serial of issuer 0, the rest unknown
        ents = [e(k0[i % len(k0)] if i % 3 == 0 else b"\x7e" + int(i).to_bytes(3, "big")) for i in range(n)]
        return [cb.crl(entries=ents or None)], [dig[0]]

    for n0, n1 in ((0, X + 1), (X - 1, X), (X, 5 * X + 3), (X + 1, 0), (5 * X + 3, X - 1), (X, X)):
        out.append(("rounds_%d_%d" % (n0, n1), one(n0) + (None,), one(n1) + (None,)))
    many = [cb.crl(entries=[e(k0[(7 * j + i) % len(k0)] if i % 5 == 0 else b"\x7d" + int(600 * j + i).to_bytes(3, "big")) for i in range(600)])
            for j in range(20)]
    out.append(("chunks_vs_one", (many, [dig[0]] * 20, None), one(7) + (None,)))
    out.append(("chunks_vs_none", ([], [], None), (many[:13], [dig[0]] * 13, None)))
    out.append(("both_empty", ([], [], None), ([], [], None)))
    invalid = [cb.crl(entries=[e(s, cert_issuer=True) for s in k0[:40]]), cb.crl(entries=[e(s) for s in k0[:40]])]
    out.append(("all_invalid", (invalid, [dig[0], b"\xee" * 32], None), ([invalid[1][:-3]], [dig[0]], None)))
    return out


def capped(cases_, need0):
    """the mix with entry_cap one short on rank 0 only"""
    name, a, b = cases_[0]
    return ("cap_short", (a[0], a[1], need0 - 1), b)


def _join(db, crls, digs, cap):
    """{code, n_entries, every output array} of one call"""
    from ct_mapreduce_b200 import capi
    try:
        r = db.revoked_known(crls, digs, entry_cap=cap)
        out = {f: getattr(r, f).copy() for f in CRL_FIELDS + ENTRY_FIELDS}
        out.update(code=0, n_entries=r.n_entries)
    except capi.CtmrError as ex:
        out = dict(code=ex.code, n_entries=getattr(ex, "n_entries", None))
    return out


def _state(db):
    return (db.checkpoint().tobytes(), db.next_index(), db.status_counters().tolist(), db.issuer_counts(), db.table_stats())


def _worker(rank, world, same_gpu):
    import torch
    import torch.distributed as dist
    dev = 0 if same_gpu else rank
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi, engine, sharded
    c = corpus()
    res = {}
    db = engine.GpuCertDatabase(device=dev, **KW)
    sharded.attach_peers(db)
    dense = db.register_issuers(c[3], c[4])
    dig = [db.issuer_digest(int(d)) for d in dense]
    x = None
    if rank == 0:  # an issuer only rank 0 registers
        der = np.frombuffer(XM.ca(3).der, np.uint8)
        xd = int(db.register_issuers(der, np.array([0, der.size], np.uint64))[0])
        x = (xd, db.issuer_digest(xd))
    xs = [None] * world
    dist.all_gather_object(xs, x)
    x_dense, x_dig = xs[0]
    db.store_batch(*part(c, rank * H, (rank + 1) * H), NOW_NS)
    for owner, hour, d, serials in crafted(dense, dig, x_dense, x_dig):
        if owner == rank:
            db.preload_known(hour, d, serials)
    dist.barrier()
    sets = corpus_sets(c, dig)
    cs = cases(dig, x_dig, sets)
    res["parts"] = db.checkpoint().copy()
    res["dig"], res["x_dig"] = dig, x_dig
    before = _state(db)
    res["calls"] = {}
    for name, a, b in cs:
        crls, digs, cap = (a, b)[rank]
        res["calls"][name] = _join(db, crls, digs, cap)
    res["read_only"] = _state(db) == before
    need0 = [None] * world
    dist.all_gather_object(need0, res["calls"]["mix"]["n_entries"])
    name, a, b = capped(cs, need0[0])
    res["calls"][name] = _join(db, *(a, b)[rank])
    # failures, each followed by the mix again: a CRL outside data, a CRL above the staging budget, and a digest count
    # the binding refuses (the call is made anyway, with no batch)
    mix = cs[0][1 + rank]
    data, offs, lens = engine.pack_crls(mix[0])
    fails = {
        "outside": ((data, offs, lens + np.uint64(1) * (np.arange(lens.size) == lens.size - 1)), mix[1]),
        "too_large": ([cb.crl(entries=[cb.entry(bytes([1, i >> 8, i & 255]), 1767000000) for i in range(7000)])], [dig[0]]),
        "refused": (mix[0], mix[1][:-1]),
    }
    res["fail"] = {}
    for fname, (crls, digs) in fails.items():
        got = None
        if rank == 1:
            try:
                db.revoked_known(crls, digs)
            except capi.CtmrError as ex:
                got = (ex.code, ex.n_entries)
            except ValueError:
                got = ("ValueError", None)
        else:
            got = _join(db, *mix)
            got = (got["code"], got["n_entries"])
        res["fail"][fname] = (got, _join(db, *mix))
    after = db.store_batch(*part(c, 2 * H + rank * TAIL, 2 * H + (rank + 1) * TAIL), NOW_NS)
    res["after"] = {f: getattr(after, f) for f in ("status", "was_unknown", "first_issuer_hour")}
    db.close()
    # scale: a 2 M-entry CRL on rank 0, 10,000 small CRLs on rank 1, hits seeded in sets of both ranks' shards
    db = engine.GpuCertDatabase(device=dev, **SCALE_KW)
    sharded.attach_peers(db)
    dense = db.register_issuers(c[3], c[4])
    dig = [db.issuer_digest(int(d)) for d in dense]
    rng = np.random.default_rng(11)
    rows = rng.integers(0, 256, (SCALE_N, 16), dtype=np.uint8)
    rows[:, 0] = rng.integers(1, 0x80, SCALE_N, dtype=np.uint8)
    seeded = list(range(0, SCALE_N, SCALE_STRIDE))
    i2 = int(dense[2])
    small_seed = [7, 1234, 5555, 9999]
    for j, pos in enumerate(seeded):  # alternate owners
        owner = j & 1
        if owner == rank:
            db.preload_known(XM.hour_for(i2, 2, owner, FAR + j), dig[2], [rows[pos].tobytes()])
    small_serial = lambda i: bytes([1 + i % 100, i >> 8 & 0x7F])  # noqa: E731
    for j, i in enumerate(small_seed):
        owner = j & 1
        if owner == rank:
            ii = int(dense[i % 3])
            db.preload_known(XM.hour_for(ii, 2, owner, FAR + j), dig[i % 3], [small_serial(i)])
    dist.barrier()
    if rank == 0:
        r = db.revoked_known([cb.bulk_crl(rows)], [dig[2]])
        res["scale"] = (int(r.crl_status[0]), r.n_entries, sorted(np.nonzero(r.known)[0].tolist()), seeded)
    else:
        small = [cb.crl(entries=[cb.entry(small_serial(i), 1767000000)]) for i in range(10_000)]
        r = db.revoked_known(small, [dig[i % 3] for i in range(10_000)])
        res["scale"] = (bool((r.crl_status == co.CRL_OK).all()), r.n_entries, sorted(np.nonzero(r.known)[0].tolist()), small_seed)
    db.close()
    if rank == 0:
        res["cases"] = cs + [capped(cs, need0[0])]
    dist.barrier()
    dist.destroy_process_group()
    return res


def _oracle_check(got, crls, digs, sets, registered):
    """the crl_oracle rules over the union of the sets (test_gpu_crl's checks)"""
    from ct_mapreduce_b200 import engine
    data, offs, _ = engine.pack_crls(crls)
    e = 0
    for k, der in enumerate(crls):
        p = co.parse_crl(der)
        j = co.join(p, digs[k], sets, registered)
        assert got["crl_status"][k] == j["status"], k
        if j["status"] not in (co.CRL_OK, co.CRL_UNKNOWN_ISSUER):
            assert got["crl_entries"][k] == 0
            continue
        assert got["crl_first"][k] == e and got["crl_entries"][k] == len(p["entries"]), k
        for i, pe in enumerate(p["entries"]):
            g = e + i
            o = int(got["serial_off"][g])
            assert bytes(data[o:o + int(got["serial_len"][g])]) == pe["serial"]
            assert (got["revoked_at"][g], got["reason"][g], got["entry_status"][g]) == (pe["revoked_at"], pe["reason"], pe["status"])
            assert (got["known"][g], got["known_exp_hour"][g], got["known_sets"][g]) == j["answers"][i], (k, i, pe["serial"])
        e += len(p["entries"])
    assert got["n_entries"] == e


def _run(same_gpu):
    from ct_mapreduce_b200 import build
    build.build()
    world = 2
    return run_ranks(_worker, world, (same_gpu,), timeout=1700)


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("same_gpu", [True, False], ids=["two_ranks_one_gpu", "one_rank_per_gpu"])
def test_collective_join_equals_one_ctx(same_gpu):
    import torch
    from ct_mapreduce_b200 import capi, engine
    if not same_gpu and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    outs = _run(same_gpu)
    o0 = outs[0]
    dig, x_dig = o0["dig"], o0["x_dig"]
    c = corpus()
    sets = corpus_sets(c, dig)
    # the union of every rank's sets: the corpus and the crafted preloads (hours recomputed from the twin's registry)
    with engine.GpuCertDatabase(device=0, **dict(KW, table_capacity=1 << 16)) as twin:
        twin.load_checkpoint([outs[r]["parts"] for r in (1, 0)])
        dense = twin.register_issuers(c[3], c[4])
        assert [twin.issuer_digest(int(d)) for d in dense] == dig
        der = np.frombuffer(XM.ca(3).der, np.uint8)
        x_dense = int(twin.register_issuers(der, np.array([0, der.size], np.uint64))[0])
        assert twin.issuer_digest(x_dense) == x_dig
        for _, hour, d, serials in crafted(dense, dig, x_dense, x_dig):
            sets.setdefault((hour, d), set()).update(serials)
        registered = set(dig) | {x_dig}
        for name, *per_rank in o0["cases"]:
            for r in range(2):
                crls, digs, cap = per_rank[r]
                got, want = outs[r]["calls"][name], None
                want = {}
                try:
                    w = twin.revoked_known(crls, digs, entry_cap=cap)
                    want = {f: getattr(w, f) for f in CRL_FIELDS + ENTRY_FIELDS}
                    want.update(code=0, n_entries=w.n_entries)
                except capi.CtmrError as ex:
                    want = dict(code=ex.code, n_entries=ex.n_entries)
                assert (got["code"], got["n_entries"]) == (want["code"], want["n_entries"]), (name, r)
                if got["code"]:
                    continue
                for f in CRL_FIELDS + ENTRY_FIELDS:
                    assert np.array_equal(got[f], want[f]), (name, r, f)
                _oracle_check(got, crls, digs, sets, registered)
        # the crafted sets are seen across ranks: 66 01 in two sets, the lower hour on rank 1's shard
        mix = outs[0]["calls"]["mix"]
        data, _, _ = engine.pack_crls(o0["cases"][0][1][0])
        hits = {bytes(data[int(o):int(o) + int(n)]): (k, h, s) for o, n, k, h, s in
                zip(mix["serial_off"], mix["serial_len"], mix["known"], mix["known_exp_hour"], mix["known_sets"])}
        low = min(h for (h, d), ss in sets.items() if d == dig[0] and b"\x66\x01" in ss)
        assert hits[b"\x66\x01"] == (1, low, 2) and XM.key_owner(low, int(dense[0]), 2) == 1
        assert hits[b"\x66\x02"][2] == 2
    assert o0["calls"]["mix"]["known"].sum() > 200
    # entry_cap one short on rank 0 only: its count, and rank 1's complete answers (compared above)
    assert o0["calls"]["cap_short"]["code"] == capi.E_BATCH_TOO_LARGE
    assert o0["calls"]["cap_short"]["n_entries"] == o0["calls"]["mix"]["n_entries"]
    assert outs[1]["calls"]["cap_short"]["code"] == 0
    for r in range(2):
        assert outs[r]["read_only"], r
        # failures: the failing rank's own code, CTMR_E_PEER_FAILED on the other, n_entries 0; the next call is normal
        for fname, want1 in (("outside", capi.E_INVALID), ("too_large", capi.E_BATCH_TOO_LARGE), ("refused", "ValueError")):
            got, again = outs[r]["fail"][fname]
            if r == 1:
                assert got[0] == want1, fname
                assert got[1] in (0, None), fname
            else:
                assert got == (capi.E_PEER_FAILED, 0), fname
            for f in CRL_FIELDS + ENTRY_FIELDS + ("code", "n_entries"):
                assert np.array_equal(again[f], outs[r]["calls"]["mix"][f]), (fname, r, f)
    # a collective store_batch after the joins: the oracle after the first halves (set membership does not depend on the
    # order), then rank 0's tail, then rank 1's
    from oracle import oracle
    blob, offs, idx, iblob, ioffs = c
    odb = oracle.DB()
    odb.process(blob, offs[:2 * H + 1], iblob, ioffs, idx[:2 * H], NOW_NS)
    wt = odb.process(blob, offs[2 * H:], iblob, ioffs, idx[2 * H:], NOW_NS)
    for r in range(2):
        for f, a in outs[r]["after"].items():
            assert np.array_equal(a, getattr(wt, f)[r * TAIL:(r + 1) * TAIL]), (r, f)
    # scale
    st0, n0, hits0, seeded0 = outs[0]["scale"]
    assert st0 == co.CRL_OK and n0 == SCALE_N and hits0 == seeded0
    ok1, n1, hits1, seeded1 = outs[1]["scale"]
    assert ok1 and n1 == 10_000 and hits1 == seeded1


def test_empty_batch_on_one_ctx():
    """An empty list of CRLs is a call with n_crls == 0 on one ctx too: an empty result (the peer ranks above pass one
    whenever they have no CRLs); a digest count that does not match the CRLs is still refused before the call."""
    from ct_mapreduce_b200 import engine
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 12) as db:
        r = db.revoked_known([], [])
        assert r.n_entries == 0 and r.crl_status.size == 0 and all(getattr(r, f).size == 0 for f in ENTRY_FIELDS)
        with pytest.raises(ValueError):
            db.revoked_known([cb.crl(entries=[cb.entry(b"\x01", 1767000000)])], [])
