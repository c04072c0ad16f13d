"""ctmr_revoked_verify / ctmr_group_revoked_verify on the GPU against verify_model: R and S, with each key record's hour
and first index, are derived on the host from a checkpoint of the table and crl_oracle's parse of the CRLs
(test_gpu_cascade's rules), and the counts and the list the GPU returns must be the model's."""
import ctypes as C
import random
import struct
import subprocess

import numpy as np
import pytest

import cascade_model as cm
import checkpoint_model as ckm
import crl_build as cb
import crl_oracle as co
import stash_model as sm
import test_gpu_cascade as tgc
import test_gpu_stash as tgs
import verify_model as vm
from conftest import ROOT
from ct_mapreduce_b200 import capi, engine
from ct_mapreduce_b200.capi import CtmrError
from oracle import oracle

gpu = pytest.mark.gpu

NOW, NOW_NS, HOUR = tgc.NOW, tgc.NOW_NS, tgc.HOUR
MASK = 2**64 - 1


def test_verify_structs_match_header(tmp_path):
    src = tmp_path / "probe.c"
    probes = [("ctmr_verify_counts", n) for n in ("revoked", "missed", "valid", "blocked")] + \
             [("ctmr_verify_miss", n) for n in ("digest", "exp_hour", "first_index", "serial_len", "serial", "blocked", "pad")] + \
             [("ctmr_verify_out", n) for n in ("crl_status", "issuers", "levels", "before", "since", "list", "list_cap", "n_list")]
    src.write_text('#include "include/ctmr.h"\n#include <stdio.h>\n#include <stddef.h>\nint main(){' +
                   "".join(f'printf("%zu ", sizeof({s}));' for s in ("ctmr_verify_counts", "ctmr_verify_miss", "ctmr_verify_out")) +
                   "".join(f'printf("%zu ", offsetof({s}, {n}));' for s, n in probes) + "return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", ROOT, str(src), "-o", str(exe)], check=True, cwd=ROOT)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    py = {"ctmr_verify_counts": capi.VerifyCounts, "ctmr_verify_miss": capi.VerifyMiss, "ctmr_verify_out": capi.VerifyOut}
    assert got == [C.sizeof(py[s]) for s in py] + [getattr(py[s], n).offset for s, n in probes]
    assert C.sizeof(capi.VerifyMiss) == 96 == engine.MISS_DTYPE.itemsize
    assert all(engine.MISS_DTYPE.fields[n][1] == getattr(capi.VerifyMiss, n).offset for n, _ in capi.VerifyMiss._fields_)


def _records(db):
    """(hour, digest, serial, first index) of every key record of the db, from its checkpoint"""
    part = ckm.decode_part(db.checkpoint())
    out = []
    for r in part["keys"]:
        b = r["body"].tobytes()
        out.append((ckm.signed32(int(r["body"][0])), part["digests"][int(r["body"][1])], b[9:9 + b[8]], ~int(r["inv_first"]) & MASK))
    return out


def _model(records, crls, digs, registered, now=NOW):
    """(R, S) as verify_model's key records (x, hour, first), and the covered issuers, by the header's rules"""
    parsed = [co.parse_crl(c) for c in crls]
    status = [co.join(p, d, {}, registered)["status"] for p, d in zip(parsed, digs)]
    covered = {d for d in digs if d in registered and all(s == co.CRL_OK for s, dd in zip(status, digs) if dd == d)}
    revoked = {(d, e["serial"]) for p, d, s in zip(parsed, digs, status) if s == co.CRL_OK for e in p["entries"] if e["status"] == co.RV_OK}
    R, S = [], []
    for h, d, s, f in records:
        if h * 3600 > now and d in covered:
            (R if (d, s) in revoked else S).append((d + s, h, f))
    return R, S, covered, status


def _check(res, R, S, flt, stashes=b"", covered_below=MASK):
    counts, lst = vm.verify(R, S, flt, stashes, covered_below)
    assert (res.before, res.since) == (counts["before"], counts["since"])
    assert res.entries() == lst
    assert res.levels == len(cm.decode(flt)["levels"])
    return counts, lst


@gpu
def test_a_fresh_filter_verifies_clean():
    corpus = tgs._corpus()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dig = tgc._fill(db, corpus)
        crls, digs = tgc._crls(db, dig)
        ck = db.checkpoint()
        for salt in (b"", b"\x01\x02"):
            cas = db.revoked_cascade(crls, digs, NOW, salt)
            res = db.revoked_verify(crls, digs, NOW, cas.bytes)
            assert res.before == {"revoked": cas.revoked, "missed": 0, "valid": cas.valid, "blocked": 0}, salt
            assert res.since == dict.fromkeys(vm.NAMES, 0) and res.entries() == []
            assert (res.issuers, res.levels) == (cas.issuers, cas.levels) and np.array_equal(res.crl_status, cas.crl_status)
            assert cas.revoked > 100 and cas.valid > 300
            for w in (1, 2, 3, 8):
                with engine.GpuCertGroup([0] * w, table_capacity=1 << 16) as g:
                    g.load_checkpoint(ck)
                    got = g.revoked_verify(crls, digs, NOW, cas.bytes)
                    assert (got.before, got.since, got.issuers, got.levels) == (res.before, res.since, res.issuers, res.levels), (salt, w)
                    assert got.entries() == [] and np.array_equal(got.crl_status, res.crl_status)


def _day_two(db, dig):
    """day 0's CRLs and filter and the next index then; day two: more certificates, CRLs that revoke more of them and of
    the old ones, and one serial revoked on day 0 that is no longer.  Returns (flt, next index, day-two CRLs and digests,
    the un-revoked serial)."""
    rec = _records(db)
    crls0, digs0 = tgc._crls(db, dig)
    flt = db.revoked_cascade(crls0, digs0, NOW, b"day0").bytes
    nb = db.next_index()
    R0, _, _, _ = _model(rec, crls0, digs0, set(dig))
    k2 = sorted({s for h, d, s, f in rec if d == dig[2]})
    live0 = {x for x, _, _ in R0}
    u = next(s for s in k2[4::4] if dig[2] + s in live0)                   # revoked by crls0[4] on day 0
    cfg2 = oracle.synth_cfg(tgc.N, seed=7, n_issuers=16, dup_mode=1)
    b2, o2, i2 = oracle.synth_corpus(cfg2, 0, tgc.N)
    ib2, io2 = oracle.synth_issuers(cfg2)
    db.store_batch(b2, o2, ib2, io2, i2, NOW_NS)
    fresh = [bytes([0x21, n]) * (1 + n % 19) for n in range(60)]
    db.preload_known(HOUR + 30, dig[0], fresh)
    db.preload_known(HOUR + 32, dig[0], fresh[:5])                          # serials under two hours
    rec = _records(db)
    k0 = sorted({s for h, d, s, f in rec if d == dig[0]})
    e = lambda s: cb.entry(s, 1767100000)  # noqa: E731
    crls = list(crls0)
    crls[4] = cb.crl(entries=[e(s) for s in k2[::4] if s != u] + [e(k2[0])])  # tgc._crls's issuer-2 CRL without u
    crls.append(cb.crl(entries=[e(s) for s in k0[2::5] + fresh[::2]]))
    return flt, nb, crls, digs0 + [dig[0]], u


@gpu
def test_a_day_later():
    corpus = tgs._corpus()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dig = tgc._fill(db, corpus)
        flt, nb, crls, digs, u = _day_two(db, dig)
        R, S, covered, status = _model(_records(db), crls, digs, set(dig))
        assert any(f >= nb for _, _, f in R + S) and any(f < nb for _, _, f in R + S)
        for cb_ in (MASK, nb, nb // 2):
            res = db.revoked_verify(crls, digs, NOW, flt, covered_below=cb_)
            counts, lst = _check(res, R, S, flt, b"", cb_)
            assert res.issuers == len(covered) and list(res.crl_status) == status
        every = db.revoked_verify(crls, digs, NOW, flt)
        assert every.before["missed"] > 20 and every.before["blocked"] >= 1
        split = db.revoked_verify(crls, digs, NOW, flt, covered_below=nb)
        assert [e for e in split.entries() if e[4]] == [(dig[2], u, h, f, True) for x, h, f in sorted(S, key=lambda r: r[1])
                                                           if x == dig[2] + u and f < nb]
        assert split.since["missed"] > 5                                   # the fresh serials revoked on day two
        # the stash of day two makes every missed record revoked
        stash = db.revoked_stash(crls, digs, NOW, flt).bytes
        res = db.revoked_verify(crls, digs, NOW, flt, stash)
        _check(res, R, S, flt, stash)
        assert res.before["missed"] == res.since["missed"] == 0 and res.before["revoked"] + res.since["revoked"] == len(R)
        ck = db.checkpoint()
    for w in (2, 3):
        with engine.GpuCertGroup([0] * w, table_capacity=1 << 16) as g:
            g.load_checkpoint(ck)
            got = g.revoked_verify(crls, digs, NOW, flt, covered_below=nb)
            assert (got.before, got.since, got.entries()) == (split.before, split.since, split.entries()), w


@pytest.fixture(scope="module")
def walk():
    """a db whose live records are one universe of keys with serials of 1 to 39 octets under three issuers, every other
    one revoked by the CRLs, plus a serial under two hours; filters from cascade_model.build over other splits of it"""
    rng = random.Random(11)                                                # test_gpu_stash's universe: every level is reached
    corpus = tgs._corpus()
    db = engine.GpuCertDatabase(device=0, table_capacity=1 << 16)
    try:
        dense = [int(d) for d in db.register_issuers(corpus[3], corpus[4])]
        dig = [db.issuer_digest(d) for d in dense[:3]]
        keys = list(dict.fromkeys(dig[i % 3] + bytes([rng.randrange(1, 128)]) + rng.randbytes(i % 39) for i in range(6400)))
        for d in dig:
            db.preload_known(HOUR + 50, d, [x[32:] for x in keys if x[:32] == d])
        db.preload_known(HOUR + 51, keys[3001][:32], [keys[3001][32:]])     # one serial under two hours
        crls = [cb.crl(entries=[cb.entry(x[32:], 1767000000) for x in keys[::2] if x[:32] == d]) for d in dig]
        filters = [cm.build(keys[:nr], keys[nr:nr + ns], salt) for salt, (nr, ns) in zip(tgs.SALTS, tgs.SIZES)]
        R, S, _, _ = _model(_records(db), crls, dig, set(dig))
        yield db, dig, crls, R, S, filters
    finally:
        db.close()


@gpu
def test_every_level_of_the_walk(walk):
    db, dig, crls, R, S, filters = walk
    parity = set()
    for flt in filters:
        d = cm.decode(flt)
        L = len(d["levels"])
        parity.add(L % 2)
        assert {tgs._stops(d, x) for x, _, _ in R + S} == set(range(L + 1))
        counts, lst = _check(db.revoked_verify(crls, dig, NOW, flt), R, S, flt)
        assert counts["before"]["missed"] > 1000 and counts["before"]["blocked"] > 1000
    assert parity == {0, 1}


@gpu
def test_stash_entries_that_never_match(walk):
    db, dig, crls, R, S, filters = walk
    flt = filters[0]
    want = db.revoked_verify(crls, dig, NOW, flt)
    missed = [e for e in want.entries() if not e[4]]
    unknown = struct.pack("<IB", 1, 32) + b"\xee" * 32 + bytes([len(missed[0][1])]) + missed[0][1]
    long = struct.pack("<IB", 2, 32) + dig[1] + b"\x2d" + b"\x01" * 45 + b"\x28" + b"\x01" * 40
    for stashes in (unknown, long, unknown + long):
        got = db.revoked_verify(crls, dig, NOW, flt, stashes)
        assert (got.before, got.since, got.entries()) == (want.before, want.since, want.entries())
        _check(got, R, S, flt, stashes)
    some = sm.encode([(e[0], e[1]) for e in want.entries()[::3]])
    _check(db.revoked_verify(crls, dig, NOW, flt, unknown + some + long), R, S, flt, unknown + some + long)


@gpu
def test_a_filter_that_blocks_every_record(walk):
    """one level with every bit set answers every record revoked: every S record is blocked, more listed records than
    the lists cascade_front sized for R, so the pass runs again with longer lists"""
    db, dig, crls, R, S, filters = walk
    flt = tgs.HDR + tgs._level(1, 3, 16, b"\xff\xff")
    assert len(S) > len(R)
    counts, lst = _check(db.revoked_verify(crls, dig, NOW, flt), R, S, flt)
    assert counts["before"] == {"revoked": len(R), "missed": 0, "valid": 0, "blocked": len(S)} and len(lst) == len(S)


@gpu
def test_refusals(walk):
    db, dig, crls, R, S, filters = walk
    lib = capi.load()
    b, keep = engine._crl_batch(crls, dig)
    for f in tgs.BAD_FILTERS:
        with pytest.raises(CtmrError) as ei:
            db.revoked_verify(crls, dig, NOW, f)
        assert ei.value.code == capi.E_INVALID, f
    for s in tgs.BAD_STASHES:
        with pytest.raises(CtmrError) as ei:
            db.revoked_verify(crls, dig, NOW, filters[0], s)
        assert ei.value.code == capi.E_INVALID, s
    flt = tgs._ctypes(filters[0])
    o = capi.VerifyOut()
    assert lib.ctmr_revoked_verify(db.handle, None, NOW, flt, len(filters[0]), None, 0, MASK, C.byref(o)) == capi.E_INVALID
    assert lib.ctmr_revoked_verify(db.handle, C.byref(b), NOW, flt, len(filters[0]), None, 0, MASK, None) == capi.E_INVALID
    assert lib.ctmr_revoked_verify(db.handle, C.byref(b), NOW, None, len(filters[0]), None, 0, MASK, C.byref(o)) == capi.E_INVALID
    assert lib.ctmr_revoked_verify(db.handle, C.byref(b), NOW, flt, len(filters[0]), None, 5, MASK, C.byref(o)) == capi.E_INVALID
    with engine.GpuCertGroup([0, 0], table_capacity=1 << 15) as g:
        member = lib.ctmr_group_member(g.handle, 1)
        assert lib.ctmr_revoked_verify(member, C.byref(b), NOW, flt, len(filters[0]), None, 0, MASK, C.byref(o)) == capi.E_INVALID
    assert db.revoked_verify([], [], NOW, filters[0]).before == dict.fromkeys(vm.NAMES, 0)   # still usable


@gpu
def test_cap_and_read_only():
    corpus = tgs._corpus()
    lib = capi.load()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dig = tgc._fill(db, corpus)
        flt, nb, crls, digs, u = _day_two(db, dig)
        before = (db.checkpoint().tobytes(), db.next_index(), list(db.status_counters()), db.issuer_counts())
        want = db.revoked_verify(crls, digs, NOW, flt)
        assert (db.checkpoint().tobytes(), db.next_index(), list(db.status_counters()), db.issuer_counts()) == before
        n = len(want.list)
        assert n > 20
        b, keep = engine._crl_batch(crls, digs)
        fb = tgs._ctypes(flt)
        raw = np.full((n + 4) * 96, 0xAB, np.uint8)
        status = np.full(len(crls), 0xCD, np.uint8)
        o = capi.VerifyOut(status.ctypes.data, 0, 0, capi.VerifyCounts(), capi.VerifyCounts(), raw.ctypes.data, n - 1, 0)
        assert lib.ctmr_revoked_verify(db.handle, C.byref(b), NOW, fb, len(flt), None, 0, MASK, C.byref(o)) == capi.E_BATCH_TOO_LARGE
        assert o.n_list == n and (raw == 0xAB).all() and (status == 0xCD).all()
        assert (o.issuers, o.levels, o.before.revoked, o.since.valid) == (0, 0, 0, 0)
        o = capi.VerifyOut(status.ctypes.data, 0, 0, capi.VerifyCounts(), capi.VerifyCounts(), 0, 0, 0)   # NULL list
        assert lib.ctmr_revoked_verify(db.handle, C.byref(b), NOW, fb, len(flt), None, 0, MASK, C.byref(o)) == capi.E_BATCH_TOO_LARGE
        assert o.n_list == n
        o = capi.VerifyOut(status.ctypes.data, 0, 0, capi.VerifyCounts(), capi.VerifyCounts(), raw.ctypes.data, n, 0)
        assert lib.ctmr_revoked_verify(db.handle, C.byref(b), NOW, fb, len(flt), None, 0, MASK, C.byref(o)) == 0
        assert raw[:n * 96].tobytes() == want.list.tobytes() and (raw[n * 96:] == 0xAB).all()
        assert np.array_equal(status, want.crl_status) and o.n_list == n
        got = db.revoked_verify(crls, digs, NOW, flt, cap=3)                 # the binding grows a short list
        assert got.list.tobytes() == want.list.tobytes()
        assert (db.checkpoint().tobytes(), db.next_index(), list(db.status_counters()), db.issuer_counts()) == before


@gpu
def test_2_26_slots_several_chunks():
    rng = np.random.default_rng(14)
    _, _, _, iblob, ioffs = tgs._corpus()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 26, max_batch_bytes=4 << 20) as db:
        dig = [db.issuer_digest(int(d)) for d in db.register_issuers(iblob, ioffs)][:4]
        n = 1 << 24
        rows, who, when = tgc._bulk_fill(db, dig, n, rng, [HOUR - 5, HOUR + 3, HOUR + 40])
        crls0, digs0, rev0 = tgc._bulk_crls(rows, who, dig[:3], 0.01, rng, 60_000)
        flt = db.revoked_cascade(crls0, digs0, NOW).bytes
        more = (rng.random(n) < 0.001) & ~rev0
        rev = rev0 | more
        crls, digs = [], []
        for i, d in enumerate(dig[:3]):
            sel = np.nonzero(rev & (who == i))[0]
            for lo in range(0, sel.size, 60_000):
                crls.append(cb.bulk_crl(rows[sel[lo:lo + 60_000]]))
                digs.append(d)
        assert len(crls) >= 3
        res = db.revoked_verify(crls, digs, NOW, flt)
        stash = db.revoked_stash(crls, digs, NOW, flt).bytes
        clean = db.revoked_verify(crls, digs, NOW, flt, stash)
    live = (when > 0) & (who < 3)
    assert res.before == {"revoked": int((live & rev0).sum()), "missed": int((live & more).sum()), "valid": int((live & ~rev).sum()),
                          "blocked": 0}
    assert res.since == dict.fromkeys(vm.NAMES, 0) and res.issuers == 3
    missed = sorted((dig[who[i]], rows[i].tobytes(), [HOUR - 5, HOUR + 3, HOUR + 40][when[i]]) for i in np.nonzero(live & more)[0].tolist())
    assert [e[:3] for e in res.entries()] == missed
    assert clean.before["missed"] == 0 and clean.before["revoked"] == int((live & rev).sum())
