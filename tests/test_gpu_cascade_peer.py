"""ctmr_revoked_cascade on one process per GPU: ranks (two on one GPU, two on two GPUs when the box has them, and three on
one GPU) fill their shards with a collective store_batch of a part of a synthetic corpus each and with preloads on the
owning rank, then build cascades in collective calls, each rank with its own CRLs.  Every rank's outputs must equal each
other's and those of ctmr_revoked_cascade on a one-ctx twin that holds every rank's shard and runs the ranks' CRLs in rank
order; the bytes must be cascade_model's, with R and S derived from the checkpoint parts and crl_oracle.  Also covered:
round and chunk edges with 512 records per round, levels and coverage bitmaps over several exchange slices, a rank whose
lists grow after level 1, salts, each failure rule and the next call after it, the cap rule, the read-only property, and
two 2^22-slot shards.  Marked gpu."""
import ctypes as C

import numpy as np
import pytest

import cascade_model as cm
import checkpoint_model as ckm
import crl_build as cb
import crl_oracle as co
import xchg_model as XM
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

NOW = 1767225600          # a whole hour: sets of that hour are expired, the next hour's are live
NOW_NS = NOW * 10**9
HOUR = NOW // 3600
H = 2048                  # corpus entries each rank stores first
TAIL = 60                 # entries each rank stores after the cascades
X = 512                   # max_batch_entries = max_round_entries: records per inbox region, i.e. per rank and round
KW = dict(table_capacity=1 << 15, max_issuers=1024, max_batch_entries=X, max_round_entries=X, max_batch_bytes=1 << 17)
OUT = ("code", "bytes", "issuers", "levels", "revoked", "valid")
SLICE_BITS = X * 64 * 8   # one slice of the OR all-reduce: X records of 64 bytes = 32 KiB = 262,144 bits


def corpus(world):
    """the same entries in the workers and in the parent"""
    from oracle import oracle
    n = world * (H + TAIL)
    cfg = oracle.synth_cfg(n, n_issuers=16, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, n)
    iblob, ioffs = oracle.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def part(c, lo, hi):
    blob, offs, idx, iblob, ioffs = c
    return blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi]


def corpus_serials(c, world, dig):
    """{digest: sorted serials} of the entries the ranks store first"""
    from oracle import oracle
    blob, offs, idx, iblob, ioffs = c
    want = oracle.DB().process(blob, offs[:world * H + 1], iblob, ioffs, idx[:world * H], NOW_NS)
    out = {}
    for i in np.nonzero(want.status == 0)[0]:
        s = bytes(blob[offs[i] + want.serial_off[i]: offs[i] + want.serial_off[i] + want.serial_len[i]])
        out.setdefault(dig[idx[i]], set()).add(s)
    return {d: sorted(v) for d, v in out.items()}


def crafted(world, dense, dig, x, y):
    """[(hour, digest, serials)], each preloaded on the rank that owns its set: 77 77 of issuer 0 under hours owned by
    ranks 0 and 1 (revoked twice), sets of issuer 0 exactly at now and one hour past it, y's records (registered by rank 0,
    CRLs on rank 1) on rank 0 only, x's records (registered by rank 0 only, CRL on rank 1) on rank 1"""
    i0 = int(dense[0])
    a = XM.hour_for(i0, world, 0, HOUR + 10)
    b = XM.hour_for(i0, world, 1, HOUR + 10)
    return [(a, dig[0], [b"\x77\x77", b"\x77\x01"]), (b, dig[0], [b"\x77\x77", b"\x77\x02"]), (HOUR, dig[0], [b"\x66\x01", b"\x66\x03"]),
            (HOUR + 1, dig[0], [b"\x66\x02", b"\x66\x04"]), (XM.hour_for(y[0], world, 0, HOUR + 20), y[1], [b"\x55\x01", b"\x55\x02", b"\x55\x03"]),
            (XM.hour_for(x[0], world, 1, HOUR + 30), x[1], [b"\x33\x01", b"\x33\x02"])]


def cases(world, dig, x_dig, y_dig, known):
    """[(name, [(crls, digests) of each rank], salt)]"""
    e = lambda s, **kw: cb.entry(s, 1767000000, **kw)  # noqa: E731
    k0, k1, k2, k4 = (known.get(dig[i], []) for i in (0, 1, 2, 4))
    shared = cb.crl(entries=[e(s) for s in k0[1::7]] + [e(b"\x77\x01")])
    r0 = [(cb.crl(entries=[e(s) for s in k0[::3]] + [e(b"\x77\x77"), e(b"\x66\x01"), e(b"\x66\x02"), e(b"\x01" * 40),
                                                     e(k0[1], cert_issuer=True), e(b"\x12\x34\x56")]), dig[0]),
          (cb.crl(entries=[e(s) for s in k1[::2]]), dig[1]),
          (shared, dig[0]),
          (cb.crl(entries=[e(s) for s in k0[:20]]), b"\xee" * 32)]                                  # unknown issuer
    r1 = [(cb.crl(entries=[e(b"\x05")])[:-1], dig[1]),                                            # truncated: issuer 1 uncovered
          (cb.crl(entries=[e(b"\x55\x01")]), y_dig),                                              # y's records are on rank 0
          (cb.crl(entries=[e(b"\x33\x01")]), x_dig),                                              # registered by rank 0 only
          (shared, dig[0]),
          (cb.crl(entries=[e(s, cert_issuer=True) for s in k4[:20]] + [e(b"\x01" * 40)]), dig[4]),  # all invalid: issuer 4 all S
          (cb.crl(entries=[e(s) for s in k2[::4]]), dig[2])]
    rest = [[(cb.crl(entries=[e(s) for s in k2[1::5]]), dig[2])] for _ in range(world - 2)]
    unz = lambda lst: ([c for c, _ in lst], [d for _, d in lst])  # noqa: E731
    mix = [unz(r0), unz(r1)] + [unz(r) for r in rest]
    out = [("mix", mix, b""), ("mix_salt_1", mix, b"\x01"), ("mix_salt_32", mix, bytes(range(32)))]

    def one(n):  # one CRL of issuer 0 with n valid entries: every third a known serial, the rest unknown
        ents = [e(k0[i % len(k0)] if i % 3 == 0 else b"\x7e" + int(i).to_bytes(3, "big")) for i in range(n)]
        return [cb.crl(entries=ents or None)], [dig[0]]

    none = ([], [])
    edges = ((0, X + 1), (X - 1, X), (X, 5 * X + 3), (X + 1, 0)) if world == 2 else ((X - 1, X),)
    for n0, n1 in edges:
        out.append(("rounds_%d_%d" % (n0, n1), [one(n0), one(n1)] + [none] * (world - 2), b"r"))
    many = [cb.crl(entries=[e(k0[(7 * j + i) % len(k0)] if i % 5 == 0 else b"\x7d" + int(600 * j + i).to_bytes(3, "big")) for i in range(600)])
            for j in range(13)]
    if world == 2:
        out.append(("chunks_vs_none", [(many, [dig[0]] * 13), none], b"c"))
    out.append(("both_empty", [none] * world, b""))
    return out


def _cascade(db, crls, digs, salt, now=NOW, cap=None):
    """{OUT fields, crl_status} of one call, or {code} of its failure"""
    from ct_mapreduce_b200 import capi
    try:
        r = db.revoked_cascade(crls, digs, now, salt, cap=cap)
        return dict(code=0, bytes=r.bytes, issuers=r.issuers, levels=r.levels, revoked=r.revoked, valid=r.valid, crl_status=r.crl_status.tolist())
    except capi.CtmrError as ex:
        return dict(code=ex.code)
    except ValueError:
        return dict(code="ValueError")


def _raw(db, crls, digs, salt, cap, sentinel=0xAB):
    """ctmr_revoked_cascade straight through the C ABI into a sentinel-filled buffer of `cap` bytes (+ 64)"""
    from ct_mapreduce_b200 import capi, engine
    lib = capi.load()
    b, keep = engine._crl_batch(crls, digs)
    sbuf = (C.c_uint8 * max(len(salt), 1)).from_buffer_copy(salt or b"\0")
    buf = np.full(cap + 64, sentinel, np.uint8)
    status = np.full(max(len(crls), 1), 0xCD, np.uint8)
    o = capi.CascadeOut(buf.ctypes.data, cap, 0, status.ctypes.data)
    rc = lib.ctmr_revoked_cascade(db.handle, C.byref(b), NOW, sbuf, len(salt), C.byref(o))
    return rc, int(o.bytes), buf, status


def _state(db):
    return (db.checkpoint().tobytes(), db.next_index(), db.status_counters().tolist(), db.issuer_counts(), db.table_stats())


def _known_outputs(db, crls, digs):
    r = db.revoked_known(crls, digs)
    return [getattr(r, f).tolist() for f in ("crl_status", "crl_entries", "known", "known_exp_hour", "known_sets")]


def _bulk(world, rank, n, frac, per_crl, seed):
    """n random 16-octet serials per rank over issuers 0..3 (each rank's under hours it owns, `dense` known by the caller),
    `frac` of them revoked by CRLs of issuers 0..2 of at most per_crl entries, dealt to the ranks in turn"""
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, 256, (world * n, 16), dtype=np.uint8)
    rows[:, 0] = rng.integers(1, 0x80, world * n, dtype=np.uint8)
    who = rng.integers(0, 4, world * n)
    rev = rng.random(world * n) < frac
    return rows, who, rev


def _bulk_preload(db, rows, who, hours, digs):
    from ct_mapreduce_b200 import capi
    lib = capi.load()
    for i, d in enumerate(digs):
        sel = np.nonzero(who == i)[0]
        blob = np.ascontiguousarray(rows[sel]).reshape(-1)
        offs = np.arange(sel.size + 1, dtype=np.uint64) * 16
        dd = (C.c_uint8 * 32).from_buffer_copy(d)
        assert lib.ctmr_preload_known(db.handle, hours[i], dd, capi.ptr(blob), capi.ptr(offs), sel.size) == 0


def _bulk_crls(rows, who, rev, digs, per_crl):
    crls, ds = [], []
    for i in range(3):
        sel = np.nonzero(rev & (who == i))[0]
        for lo in range(0, sel.size, per_crl):
            crls.append(cb.bulk_crl(rows[sel[lo:lo + per_crl]]))
            ds.append(digs[i])
    return crls, ds


BULK = {  # name: (rows per rank, revoked fraction, entries per CRL, seed, config)
    # issuers 0..2 of 0..3 covered: |R| ~ 0.95 * 3/4 * 2 * 450,000 = 641,000 and |S| ~ 34,000 < |R| / sqrt(2), so p_1 = 0.5,
    # k_1 = 1 and m_1 = ceil(|R| / ln 2) ~ 925,000 bits: 3.5 slices of 262,144 bits.  max_issuers = 2^20 makes the seen
    # and bad bitmaps 2 x 32,769 words: 8 slices of 8,192 words, the last one partly filled
    "slices": (450_000, 0.95, 60_000, 21, dict(table_capacity=1 << 20, max_issuers=1 << 20, max_batch_entries=X, max_round_entries=X,
                                                max_batch_bytes=4 << 20)),
    # two 2^22-slot shards about half full, 1 % revoked, CRLs of 8,000 entries (~300 KB) in chunks of 512 KiB
    "scale": (2_000_000, 0.01, 8_000, 22, dict(table_capacity=1 << 22, max_issuers=1024, max_batch_entries=X, max_round_entries=X,
                                                max_batch_bytes=1 << 19)),
}


def _worker(rank, world, same_gpu, big):
    import torch
    import torch.distributed as dist
    dev = 0 if same_gpu else rank
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi, engine, sharded
    c = corpus(world)
    res = {}
    db = engine.GpuCertDatabase(device=dev, **KW)
    sharded.attach_peers(db)
    dense = db.register_issuers(c[3], c[4])
    dig = [db.issuer_digest(int(d)) for d in dense]
    xy = None
    if rank == 0:  # issuers only rank 0 registers
        got = []
        for k in (3, 5):
            der = np.frombuffer(XM.ca(k).der, np.uint8)
            d = int(db.register_issuers(der, np.array([0, der.size], np.uint64))[0])
            got.append((d, db.issuer_digest(d)))
        xy = got
    xys = [None] * world
    dist.all_gather_object(xys, xy)
    x, y = xys[0]
    db.store_batch(*part(c, rank * H, (rank + 1) * H), NOW_NS)
    # a preload takes indices, and the ranks' checkpoint parts must agree on the next one: every rank preloads as many
    # serials, the crafted sets on their owners and fillers of an expired hour
    mine = []
    for hour, d, serials in crafted(world, dense, dig, x, y):
        i = int(dense[dig.index(d)]) if d in dig else (x[0] if d == x[1] else y[0])
        if XM.key_owner(hour, i, world) == rank:
            db.preload_known(hour, d, serials)
            mine += serials
    counts = [None] * world
    dist.all_gather_object(counts, len(mine))
    if max(counts) > len(mine):
        db.preload_known(XM.hour_for(int(dense[0]), world, rank, 100), dig[0], [b"\xf0" + bytes([k]) for k in range(max(counts) - len(mine))])
    dist.barrier()
    known = corpus_serials(c, world, dig)
    cs = cases(world, dig, x[1], y[1], known)
    res["parts"] = db.checkpoint().copy()
    res["dig"], res["x"], res["y"] = dig, x, y
    before = _state(db)
    res["known_before"] = _known_outputs(db, *cs[0][1][rank])
    res["calls"] = {name: _cascade(db, *per[rank], salt) for name, per, salt in cs}
    mix, want = cs[0][1][rank], res["calls"]["mix"]
    if world == 2:
        # failures on rank 1 only, each followed by the mix again
        data, offs, lens = engine.pack_crls(mix[0])
        too_large = [cb.crl(entries=[cb.entry(bytes([1, i >> 8, i & 255]), 1767000000) for i in range(7000)])]
        fails = {"salt_33": (mix[0], mix[1], b"\0" * 33, NOW), "too_large": (too_large, [dig[0]], b"", NOW),
                 "now": (mix[0], mix[1], b"", NOW + 1), "salt": (mix[0], mix[1], b"\x01", NOW), "refused": (mix[0], mix[1][:-1], b"", NOW)}
        res["fail"] = {}
        for fname, (crls, digs, salt, now) in fails.items():
            got = _cascade(db, crls, digs, salt, now) if rank == 1 else _cascade(db, *mix, b"")
            res["fail"][fname] = (got["code"], _cascade(db, *mix, b""))
        if rank == 1:
            o = capi.CascadeOut()
            got = capi.load().ctmr_revoked_cascade(db.handle, None, NOW, None, 0, C.byref(o))
        else:
            got = _cascade(db, *mix, b"")["code"]
        res["fail"]["null_batch"] = (got, _cascade(db, *mix, b""))
        # the cap: one byte short on rank 1 only, then exactly the bytes, then the binding's retry from 16 bytes
        n = len(want["bytes"])
        rc, nb, buf, status = _raw(db, *mix, b"", n - 1 if rank == 1 else n + 1000)
        res["cap_short"] = (rc, nb, bool((buf == 0xAB).all()), bool((status == 0xCD).all()))
        rc, nb, buf, status = _raw(db, *mix, b"", n)
        res["cap_exact"] = (rc, nb, buf[:nb].tobytes() == want["bytes"], bool((buf[nb:] == 0xAB).all()), status[:len(mix[0])].tolist())
        res["cap_retry"] = _cascade(db, *mix, b"", cap=16)
    res["read_only"] = _state(db) == before
    res["known_after"] = _known_outputs(db, *cs[0][1][rank])
    after = db.store_batch(*part(c, world * H + rank * TAIL, world * H + (rank + 1) * TAIL), NOW_NS)
    res["after"] = {f: getattr(after, f) for f in ("status", "was_unknown", "first_issuer_hour")}
    db.close()
    # a rank whose shard holds only S records of the covered issuer: its lists grow after level 1
    with engine.GpuCertDatabase(device=dev, **KW) as g:
        sharded.attach_peers(g)
        d0 = int(g.register_issuers(c[3], c[4])[0])
        rng = np.random.default_rng(4)
        serials = [b"\x01" + rng.bytes(15) for _ in range(2200)]
        rev, s0, s1 = serials[:200], serials[200:1200], serials[1200:]
        if rank < 2:
            g.preload_known(XM.hour_for(d0, world, rank, HOUR + 10), dig[0], (rev + s0) if rank == 0 else s1)
        dist.barrier()
        crls = [cb.crl(entries=[cb.entry(s, 1767000000) for s in rev])] if rank == 0 else []
        res["grow"] = (_cascade(g, crls, [dig[0]] * len(crls), b"grow"), [dig[0] + s for s in rev], [dig[0] + s for s in s0 + s1])
    # bulk: the slices and the scale cases, the twin built by the parent from the same seeds
    res["bulk"] = {}
    for name, (n, frac, per_crl, seed, kw) in BULK.items() if big else ():
        with engine.GpuCertDatabase(device=dev, **kw) as g:
            sharded.attach_peers(g)
            bdense = [int(d) for d in g.register_issuers(c[3], c[4])][:4]
            bdig = [g.issuer_digest(d) for d in bdense]
            rows, who, rev = _bulk(world, rank, n, frac, per_crl, seed)
            mine = slice(rank * n, (rank + 1) * n)
            hours = [XM.hour_for(d, world, rank, HOUR + 10) for d in bdense]
            _bulk_preload(g, rows[mine], who[mine], hours, bdig)
            crls, digs = _bulk_crls(rows, who, rev, bdig, per_crl)
            dist.barrier()
            res["bulk"][name] = (_cascade(g, crls[rank::world], digs[rank::world], name.encode()), hours)
    dist.barrier()
    dist.destroy_process_group()
    return res


def _records(parts):
    """(hour, digest, serial) of every key record of the checkpoint parts"""
    out = []
    for p in parts:
        d = ckm.decode_part(p)
        for r in d["keys"]:
            b = r["body"].tobytes()
            out.append((ckm.signed32(int(r["body"][0])), d["digests"][int(r["body"][1])], b[9:9 + b[8]]))
    return out


def _model(records, crls, digs, registered):
    """(R, S, covered issuers, per-CRL status) of the header's rules"""
    parsed = [co.parse_crl(c) for c in crls]
    status = [co.join(p, d, {}, registered)["status"] for p, d in zip(parsed, digs)]
    issuers = {d for d in digs if d in registered}
    covered = {d for d in issuers if all(s == co.CRL_OK for s, dd in zip(status, digs) if dd == d)}
    revoked = {(d, e["serial"]) for p, d, s in zip(parsed, digs, status) if s == co.CRL_OK for e in p["entries"] if e["status"] == co.RV_OK}
    R, S = [], []
    for h, d, s in records:
        if h * 3600 > NOW and d in covered:
            (R if (d, s) in revoked else S).append(d + s)
    return R, S, covered, status


def _same(got, want):
    assert all(got[f] == want[f] for f in OUT), ({f: got.get(f) for f in OUT[2:]}, {f: want.get(f) for f in OUT[2:]})


def _twin_call(twin, per_rank, salt, cap=None):
    crls = [c for cr, _ in per_rank for c in cr]
    digs = [d for _, ds in per_rank for d in ds]
    return _cascade(twin, crls, digs, salt, cap=cap), crls, digs


def _check_ranks(outs, world):
    from ct_mapreduce_b200 import engine
    o0 = outs[0]
    dig, x, y = o0["dig"], o0["x"], o0["y"]
    c = corpus(world)
    registered = set(dig) | {x[1], y[1]}
    records = _records([outs[r]["parts"] for r in range(world)])
    with engine.GpuCertDatabase(device=0, **dict(KW, table_capacity=1 << 17)) as twin:
        twin.load_checkpoint([outs[r]["parts"] for r in range(world)])
        known = corpus_serials(c, world, dig)
        for name, per, salt in cases(world, dig, x[1], y[1], known):
            want, crls, digs = _twin_call(twin, per, salt)
            assert want["code"] == 0, name
            lo = 0
            for r in range(world):
                got = outs[r]["calls"][name]
                assert got["code"] == 0, (name, r, got["code"])
                _same(got, want)
                n = len(per[r][0])
                assert got["crl_status"] == want["crl_status"][lo:lo + n], (name, r)
                lo += n
            R, S, covered, status = _model(records, crls, digs, registered)
            assert want["bytes"] == cm.build(R, S, salt), name
            assert want["crl_status"] == status and (want["issuers"], want["revoked"], want["valid"]) == (len(covered), len(R), len(S)), name
            d = cm.decode(want["bytes"])
            assert want["levels"] == len(d["levels"])
            assert all(cm.query(d, q) for q in R) and not any(cm.query(d, q) for q in S), name
            if name == "mix":
                assert dig[1] not in covered and {dig[0], dig[2], dig[4], x[1], y[1]} <= covered
                assert R.count(dig[0] + b"\x77\x77") == 2 and y[1] + b"\x55\x01" in R and x[1] + b"\x33\x01" in R
                assert dig[0] + b"\x66\x02" in R and dig[0] + b"\x66\x01" not in R + S and dig[0] + b"\x66\x04" in S
                assert len(R) > 50 and len(S) > 200
            if name == "both_empty":
                assert want["bytes"] == cm.build([], []) and (want["issuers"], want["levels"]) == (0, 1)
    return o0["calls"]["mix"]


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("same_gpu", [True, False], ids=["two_ranks_one_gpu", "one_rank_per_gpu"])
def test_collective_cascade_equals_one_ctx(same_gpu):
    import torch
    from ct_mapreduce_b200 import build, capi, engine
    if not same_gpu and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    build.build()
    world = 2
    outs = run_ranks(_worker, world, (same_gpu, True), timeout=1700)
    mix = _check_ranks(outs, world)
    for r in range(world):
        o = outs[r]
        # failures: the failing rank's own code, CTMR_E_PEER_FAILED on the other; the next call is normal
        for fname, want1 in (("salt_33", capi.E_INVALID), ("too_large", capi.E_BATCH_TOO_LARGE), ("now", capi.E_INVALID),
                             ("salt", capi.E_INVALID), ("refused", "ValueError"), ("null_batch", capi.E_INVALID)):
            got, again = o["fail"][fname]
            assert got == (want1 if r == 1 else capi.E_PEER_FAILED), (fname, r, got)
            _same(again, o["calls"]["mix"])
            assert again["crl_status"] == o["calls"]["mix"]["crl_status"]
        # the cap: too small on rank 1 is too small on both, with the same bytes and nothing else written
        n = len(mix["bytes"])
        assert o["cap_short"] == (capi.E_BATCH_TOO_LARGE, n, True, True), r
        assert o["cap_exact"][:4] == (0, n, True, True) and o["cap_exact"][4] == o["calls"]["mix"]["crl_status"], r
        _same(o["cap_retry"], o["calls"]["mix"])
        # read-only: state, the revoked_known calls around the cascades, and the store_batch after them
        assert o["read_only"], r
        assert o["known_before"] == o["known_after"], r
    from oracle import oracle
    blob, offs, idx, iblob, ioffs = corpus(world)
    odb = oracle.DB()
    odb.process(blob, offs[:world * H + 1], iblob, ioffs, idx[:world * H], NOW_NS)
    wt = odb.process(blob, offs[world * H:], iblob, ioffs, idx[world * H:], NOW_NS)
    for r in range(world):
        for f, a in outs[r]["after"].items():
            assert np.array_equal(a, getattr(wt, f)[r * TAIL:(r + 1) * TAIL]), (r, f)
    # list growth after level 1 on the rank with S records only
    for r in range(world):
        got, R, S = outs[r]["grow"]
        assert got["code"] == 0 and (got["revoked"], got["valid"]) == (len(R), len(S)) and got["bytes"] == cm.build(R, S, b"grow"), r
    # bulk cases against a one-ctx twin built from the same seeds
    for name, (n, frac, per_crl, seed, kw) in BULK.items():
        got = [outs[r]["bulk"][name][0] for r in range(world)]
        hours = [outs[r]["bulk"][name][1] for r in range(world)]
        for g in got:
            assert g["code"] == 0, (name, g["code"])
            _same(g, got[0])
        with engine.GpuCertDatabase(device=0, **dict(kw, table_capacity=kw["table_capacity"] * 2)) as twin:
            bdig = [twin.issuer_digest(int(d)) for d in twin.register_issuers(corpus(world)[3], corpus(world)[4])][:4]
            rows, who, rev = _bulk(world, 0, n, frac, per_crl, seed)
            for r in range(world):
                mine = slice(r * n, (r + 1) * n)
                _bulk_preload(twin, rows[mine], who[mine], hours[r], bdig)
            crls, digs = _bulk_crls(rows, who, rev, bdig, per_crl)
            per = [(crls[r::world], digs[r::world]) for r in range(world)]
            want, _, _ = _twin_call(twin, per, name.encode())
        _same(got[0], want)
        assert (want["issuers"], want["revoked"], want["valid"]) == (3, int((rev & (who < 3)).sum()), int((~rev & (who < 3)).sum())), name
        d = cm.decode(want["bytes"])
        rng = np.random.default_rng(seed + 100)
        for i in rng.choice(np.nonzero(who < 3)[0], 2000, replace=False).tolist():
            assert cm.query(d, bdig[who[i]] + rows[i].tobytes()) == bool(rev[i]), (name, i)
        if name == "slices":
            m1 = d["levels"][0][2]
            assert m1 > 3 * SLICE_BITS and (m1 + 31) // 32 % (SLICE_BITS // 32) != 0, m1
        else:
            assert len(crls) // world >= 3


@pytest.mark.timeout(900)
def test_three_ranks_on_one_gpu():
    from ct_mapreduce_b200 import build
    build.build()
    outs = run_ranks(_worker, 3, (True, False), timeout=800)
    _check_ranks(outs, 3)
    for r in range(3):
        assert outs[r]["read_only"] and outs[r]["known_before"] == outs[r]["known_after"], r
        got, R, S = outs[r]["grow"]
        assert got["code"] == 0 and got["bytes"] == cm.build(R, S, b"grow"), r
