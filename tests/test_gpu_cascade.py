"""ctmr_revoked_cascade / ctmr_group_revoked_cascade on the GPU against cascade_model: R and S are derived on the host
from a checkpoint of the table and crl_oracle's parse of the CRLs, and the filter the GPU serializes must be the model's
byte for byte."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import cascade_model as cm
import checkpoint_model as ckm
import crl_build as cb
import crl_oracle as co
import xchg_model as X
from conftest import ROOT
from ct_mapreduce_b200 import capi, engine
from ct_mapreduce_b200.capi import CtmrError
from oracle import oracle

gpu = pytest.mark.gpu

NOW = 1767225600          # a whole hour: sets of that hour are expired, the next hour's are live
NOW_NS = NOW * 10**9
HOUR = NOW // 3600
N = 4096


def test_cascade_out_layout_matches_header(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text('#include "include/ctmr.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(ctmr_cascade_out), offsetof(ctmr_cascade_out, bytes),'
                   'offsetof(ctmr_cascade_out, crl_status), offsetof(ctmr_cascade_out, issuers), offsetof(ctmr_cascade_out, levels),'
                   'offsetof(ctmr_cascade_out, revoked), offsetof(ctmr_cascade_out, valid));return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", ROOT, str(src), "-o", str(exe)], check=True, cwd=ROOT)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    O = capi.CascadeOut
    assert got == [C.sizeof(O), O.bytes.offset, O.crl_status.offset, O.issuers.offset, O.levels.offset, O.revoked.offset,
                   O.valid.offset]


@pytest.fixture(scope="module")
def corpus():
    cfg = oracle.synth_cfg(N, n_issuers=16, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, N)
    iblob, ioffs = oracle.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def _fill(db, corpus):
    """The corpus through ctmr_process_batch, then crafted preloads: one serial under several hours, serials of 1 to 39
    octets with and without a leading 00, and sets exactly at and one hour past now.  Returns the issuers' digests."""
    blob, offs, idx, iblob, ioffs = corpus
    db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
    dig = [db.issuer_digest(int(d)) for d in db.register_issuers(iblob, ioffs)]
    for h in (HOUR + 5, HOUR + 900, 500000):
        db.preload_known(h, dig[0], [b"\x77\x77", b"\x05"])
    lens = [bytes([0x11 + n]) * n for n in range(1, 40)] + [b"\x00" + bytes([0x80 + n]) * (n - 1) for n in range(2, 40)]
    db.preload_known(HOUR + 7, dig[0], lens)
    db.preload_known(HOUR + 8, dig[2], lens[::3])
    db.preload_known(HOUR, dig[0], [b"\x66\x01", b"\x77\x77"])       # expires exactly at now
    db.preload_known(HOUR + 1, dig[0], [b"\x66\x02", b"\x05"])       # one hour past now
    db.preload_known(HOUR, dig[2], [b"\x66\x03"])
    return dig


def _records(db):
    """(hour, digest, serial) of every key record of the db, from its checkpoint"""
    part = ckm.decode_part(db.checkpoint())
    out = []
    for r in part["keys"]:
        b = r["body"].tobytes()
        out.append((ckm.signed32(int(r["body"][0])), part["digests"][int(r["body"][1])], b[9:9 + b[8]]))
    return out


def _crls(db, dig):
    """CRLs over the issuers: 0 and 2 covered, 1 uncovered by a second, bad CRL, 3 without a CRL, 4 covered by a CRL
    without entries, and a digest nobody registered.  Indirect entries and serials too long are never joined."""
    rec = _records(db)
    known = lambda d: sorted({s for h, dg, s in rec if dg == d})
    e = lambda s, **kw: cb.entry(s, 1767000000, **kw)
    k0, k1, k2 = known(dig[0]), known(dig[1]), known(dig[2])
    crls, digs = [], []
    crls.append(cb.crl(entries=[e(s) for s in k0[::3]] + [e(b"\x77\x77"), e(b"\x66\x01"), e(b"\x66\x02"), e(b"\x01" * 40),
                                                          e(k0[1], cert_issuer=True), e(b"\x12\x34\x56")])); digs.append(dig[0])
    crls.append(cb.crl(entries=[e(s) for s in k0[1::7]] + [e(b"\x77\x77")])); digs.append(dig[0])
    crls.append(cb.crl(entries=[e(s) for s in k1[::2]])); digs.append(dig[1])
    crls.append(cb.crl(entries=[e(b"\x05")])[:-1]); digs.append(dig[1])                       # truncated: issuer 1 uncovered
    crls.append(cb.crl(entries=[e(s) for s in k2[::4]] + [e(k2[0])])); digs.append(dig[2])
    crls.append(cb.crl(entries=None)); digs.append(dig[4])
    crls.append(cb.crl(entries=[e(s) for s in k0[:20]])); digs.append(b"\xee" * 32)
    return crls, digs


def _model(records, crls, digs, registered, now=NOW):
    """(R, S, covered issuers, per-CRL status) of the header's rules"""
    parsed = [co.parse_crl(c) for c in crls]
    status = [co.join(p, d, {}, registered)["status"] for p, d in zip(parsed, digs)]
    issuers = {d for d in digs if d in registered}
    covered = {d for d in issuers if all(s == co.CRL_OK for s, dd in zip(status, digs) if dd == d)}
    revoked = {(d, e["serial"]) for p, d, s in zip(parsed, digs, status) if s == co.CRL_OK
               for e in p["entries"] if e["status"] == co.RV_OK}
    R, S = [], []
    for h, d, s in records:
        if h * 3600 > now and d in covered:
            (R if (d, s) in revoked else S).append(d + s)
    return R, S, covered, status


def _check(res, R, S, covered, status, salt):
    assert res.bytes == cm.build(R, S, salt)
    assert list(res.crl_status) == status
    assert (res.issuers, res.revoked, res.valid) == (len(covered), len(R), len(S))
    d = cm.decode(res.bytes)
    assert res.levels == len(d["levels"])
    assert all(cm.query(d, x) for x in R) and not any(cm.query(d, x) for x in S)


@gpu
def test_every_output_against_the_model(corpus):
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dig = _fill(db, corpus)
        crls, digs = _crls(db, dig)
        R, S, covered, status = _model(_records(db), crls, digs, set(dig))
        assert len(covered) == 3 and len(R) > 100 and len(S) > 300
        assert len(R) > len({x for x in R})  # a revoked serial under several hours
        for salt in (b"", b"\x01", bytes(range(32))):
            _check(db.revoked_cascade(crls, digs, NOW, salt), R, S, covered, status, salt)
        empty = db.revoked_cascade([], [], NOW)
        assert empty.bytes == cm.build([], []) and (empty.issuers, empty.levels) == (0, 1)


@gpu
def test_groups_and_other_capacities_give_the_same_bytes(corpus):
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dig = _fill(db, corpus)
        crls, digs = _crls(db, dig)
        want = db.revoked_cascade(crls, digs, NOW, b"salt")
        ck = db.checkpoint()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 18) as other:
        other.load_checkpoint(ck)
        assert other.revoked_cascade(crls, digs, NOW, b"salt").bytes == want.bytes
    for w in (1, 2, 3, 8):
        with engine.GpuCertGroup([0] * w, table_capacity=1 << 16) as g:
            g.load_checkpoint(ck)
            got = g.revoked_cascade(crls, digs, NOW, b"salt")
            assert got.bytes == want.bytes, w
            assert (got.issuers, got.levels, got.revoked, got.valid) == (want.issuers, want.levels, want.revoked, want.valid)
            assert np.array_equal(got.crl_status, want.crl_status)


@gpu
def test_read_only(corpus):
    cfg2 = oracle.synth_cfg(N, seed=7, n_issuers=16, dup_mode=1)
    b2, o2, i2 = oracle.synth_corpus(cfg2, 0, N)
    ib2, io2 = oracle.synth_issuers(cfg2)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db, \
            engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as twin:
        dig = _fill(db, corpus)
        crls, digs = _crls(db, dig)
        twin.load_checkpoint(db.checkpoint())
        before = (db.checkpoint().tobytes(), db.next_index(), list(db.status_counters()), db.issuer_counts())
        db.revoked_cascade(crls, digs, NOW)
        assert (db.checkpoint().tobytes(), db.next_index(), list(db.status_counters()), db.issuer_counts()) == before
        got, want = db.revoked_known(crls, digs), twin.revoked_known(crls, digs)  # the CRL call that follows
        for name, _ in engine.RevokedResult._CRL + engine.RevokedResult._ENTRY:
            assert np.array_equal(getattr(got, name), getattr(want, name)), name
        got, want = (x.store_batch(b2, o2, ib2, io2, i2, NOW_NS) for x in (db, twin))  # and the batch that follows
        for name in ("status", "exp_hour", "serial_off", "serial_len", "was_unknown", "first_issuer_hour"):
            assert np.array_equal(getattr(got, name), getattr(want, name)), name
        assert want.was_unknown.sum() > 1000
        assert (db.next_index(), list(db.status_counters()), db.issuer_counts()) == \
            (twin.next_index(), list(twin.status_counters()), twin.issuer_counts())
        assert ckm.as_sets(ckm.decode_part(db.checkpoint())) == ckm.as_sets(ckm.decode_part(twin.checkpoint()))


@gpu
def test_a_shard_without_revoked_records_grows_its_lists(corpus):
    """A group of two whose shard 1 holds S records only: its R list is empty, so the records of its S that level 1
    contains outgrow its lists, which are grown before the level-1 test runs again.  The bytes must not change."""
    _, _, _, iblob, ioffs = corpus
    rng = np.random.default_rng(4)
    serials = [b"\x01" + rng.bytes(15) for _ in range(2200)]
    rev, s0, s1 = serials[:200], serials[200:1200], serials[1200:]
    with engine.GpuCertGroup([0, 0], table_capacity=1 << 15) as g:
        dense = [int(d) for d in g.register_issuers(iblob, ioffs)]
        dig = [g.issuer_digest(d) for d in dense]
        h0, h1 = (X.hour_for(dense[0], 2, owner, HOUR + 10) for owner in (0, 1))
        g.preload_known(h0, dig[0], rev + s0)
        g.preload_known(h1, dig[0], s1)
        crls = [cb.crl(entries=[cb.entry(x, 1767000000) for x in rev])]
        got = g.revoked_cascade(crls, [dig[0]], NOW, b"grow")
        ck = g.checkpoint()
    R, S = [dig[0] + x for x in rev], [dig[0] + x for x in s0 + s1]
    assert (got.revoked, got.valid) == (len(R), len(S))
    assert got.bytes == cm.build(R, S, b"grow")
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        db.load_checkpoint(ck)
        assert db.revoked_cascade(crls, [dig[0]], NOW, b"grow").bytes == got.bytes


@gpu
def test_errors(corpus):
    lib = capi.load()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dig = _fill(db, corpus)
        crls, digs = _crls(db, dig)
        with pytest.raises(CtmrError) as ei:
            db.revoked_cascade(crls, digs, NOW, b"\0" * 33)
        assert ei.value.code == capi.E_INVALID
        b, keep = engine._crl_batch(crls, digs)
        o = capi.CascadeOut()
        assert lib.ctmr_revoked_cascade(db.handle, None, NOW, None, 0, C.byref(o)) == capi.E_INVALID
        assert lib.ctmr_revoked_cascade(db.handle, C.byref(b), NOW, None, 0, None) == capi.E_INVALID
        assert lib.ctmr_revoked_cascade(db.handle, C.byref(b), NOW, None, 4, C.byref(o)) == capi.E_INVALID
        want = db.revoked_cascade(crls, digs, NOW, b"x")
        salt = (C.c_uint8 * 1)(ord("x"))
        buf = np.full(len(want.bytes) + 64, 0xAB, np.uint8)
        status = np.full(len(crls), 0xCD, np.uint8)
        o = capi.CascadeOut(buf.ctypes.data, len(want.bytes) - 1, 0, status.ctypes.data)
        assert lib.ctmr_revoked_cascade(db.handle, C.byref(b), NOW, salt, 1, C.byref(o)) == capi.E_BATCH_TOO_LARGE
        assert o.bytes == len(want.bytes) and (buf == 0xAB).all() and (status == 0xCD).all()
        assert (o.issuers, o.levels, o.revoked, o.valid) == (0, 0, 0, 0)
        o = capi.CascadeOut(buf.ctypes.data, o.bytes, 0, status.ctypes.data)
        assert lib.ctmr_revoked_cascade(db.handle, C.byref(b), NOW, salt, 1, C.byref(o)) == 0
        assert buf[:o.bytes].tobytes() == want.bytes and (buf[o.bytes:] == 0xAB).all()
        assert np.array_equal(status, want.crl_status)
    with engine.GpuCertGroup([0, 0], table_capacity=1 << 15) as g:
        member = lib.ctmr_group_member(g.handle, 1)
        o = capi.CascadeOut()
        assert lib.ctmr_revoked_cascade(member, C.byref(b), NOW, None, 0, C.byref(o)) == capi.E_INVALID
    big = cb.crl(entries=[cb.entry(b"\x01", 1767000000)] * 600)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16, max_batch_bytes=4096) as db:
        with pytest.raises(CtmrError) as ei:
            db.revoked_cascade([big], [b"\x00" * 32], NOW)
        assert ei.value.code == capi.E_BATCH_TOO_LARGE


def _bulk_fill(db, digests, n, rng, hours):
    """n random 16-octet serials (first octet 01..7f) spread over the issuers and hours, preloaded from numpy; returns
    the rows and each row's (issuer, hour)"""
    rows = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    rows[:, 0] = rng.integers(1, 0x80, n, dtype=np.uint8)
    who = rng.integers(0, len(digests), n)
    when = rng.integers(0, len(hours), n)
    lib = capi.load()
    for i, d in enumerate(digests):
        for j, h in enumerate(hours):
            sel = np.nonzero((who == i) & (when == j))[0]
            blob = np.ascontiguousarray(rows[sel]).reshape(-1)
            offs = np.arange(sel.size + 1, dtype=np.uint64) * 16
            dd = (C.c_uint8 * 32).from_buffer_copy(d)
            assert lib.ctmr_preload_known(db.handle, h, dd, capi.ptr(blob), capi.ptr(offs), sel.size) == 0
    return rows, who, when


def _bulk_crls(rows, who, digests, frac, rng, per_crl):
    """CRLs revoking `frac` of each issuer's rows, at most per_crl entries each; returns (crls, digests, revoked mask)"""
    rev = rng.random(rows.shape[0]) < frac
    crls, digs = [], []
    for i, d in enumerate(digests):
        sel = np.nonzero(rev & (who == i))[0]
        for lo in range(0, sel.size, per_crl):
            crls.append(cb.bulk_crl(rows[sel[lo:lo + per_crl]]))
            digs.append(d)
    return crls, digs, rev


@gpu
def test_four_million_keys_byte_for_byte(corpus):
    rng = np.random.default_rng(7)
    _, _, _, iblob, ioffs = corpus
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 23) as db:
        dig = [db.issuer_digest(int(d)) for d in db.register_issuers(iblob, ioffs)][:8]
        rows, who, when = _bulk_fill(db, dig, 1 << 22, rng, [HOUR + 10, HOUR + 2000])
        crls, digs, rev = _bulk_crls(rows, who, dig[:6], 0.02, rng, 1 << 20)
        res = db.revoked_cascade(crls, digs, NOW, b"scale")
    covered = set(range(6))
    keys = [dig[w] + rows[i].tobytes() for i, w in enumerate(who.tolist())]
    R = [keys[i] for i in np.nonzero(rev & (who < 6))[0]]
    S = [keys[i] for i in np.nonzero(~rev & (who < 6))[0]]
    assert (res.issuers, res.revoked, res.valid) == (len(covered), len(R), len(S))
    assert res.bytes == cm.build(R, S, b"scale")


@gpu
def test_2_26_slots_several_chunks_counts_and_sampled_queries(corpus):
    rng = np.random.default_rng(8)
    _, _, _, iblob, ioffs = corpus
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 26, max_batch_bytes=4 << 20) as db:
        dig = [db.issuer_digest(int(d)) for d in db.register_issuers(iblob, ioffs)][:4]
        n = 1 << 25
        rows, who, when = _bulk_fill(db, dig, n, rng, [HOUR - 5, HOUR + 3, HOUR + 40])
        crls, digs, rev = _bulk_crls(rows, who, dig[:3], 0.01, rng, 60_000)
        assert len(crls) == 6  # 2.3 MB each: one CRL per 4 MiB chunk
        res = db.revoked_cascade(crls, digs, NOW)
    live = (when > 0) & (who < 3)
    assert (res.issuers, res.revoked, res.valid) == (3, int((live & rev).sum()), int((live & ~rev).sum()))
    d = cm.decode(res.bytes)
    for i in rng.choice(np.nonzero(live)[0], 100_000, replace=False).tolist():
        assert cm.query(d, dig[who[i]] + rows[i].tobytes()) == bool(rev[i]), i
