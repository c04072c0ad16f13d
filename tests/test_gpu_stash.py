"""ctmr_revoked_stash / ctmr_group_revoked_stash on the GPU against stash_model: R is derived on the host from a
checkpoint of the table and crl_oracle's parse of the CRLs (test_gpu_cascade's helpers), and the stash the GPU
serializes, with every count, must be the model's byte for byte."""
import ctypes as C
import random
import struct
import subprocess

import numpy as np
import pytest

import cascade_model as cm
import crl_build as cb
import stash_model as sm
import test_gpu_cascade as tgc
from conftest import ROOT
from ct_mapreduce_b200 import capi, engine
from ct_mapreduce_b200.capi import CtmrError
from oracle import oracle
from peer_ranks import run_ranks

gpu = pytest.mark.gpu

NOW, NOW_NS, HOUR = tgc.NOW, tgc.NOW_NS, tgc.HOUR
FIELDS = ("issuers", "stash_issuers", "revoked", "in_filter", "in_stashes", "serials")


def test_stash_out_layout_matches_header(tmp_path):
    src = tmp_path / "probe.c"
    names = ("bytes", "crl_status") + FIELDS
    src.write_text('#include "include/ctmr.h"\n#include <stdio.h>\n#include <stddef.h>\nint main(){printf("%zu", sizeof(ctmr_stash_out));' +
                   "".join(f'printf(" %zu", offsetof(ctmr_stash_out, {n}));' for n in names) + "return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", ROOT, str(src), "-o", str(exe)], check=True, cwd=ROOT)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    O = capi.StashOut
    assert got == [C.sizeof(O)] + [getattr(O, n).offset for n in names]


def _check(res, R, flt, stashes, covered=None, status=None):
    data, n = sm.stash(R, flt, stashes)
    assert res.bytes == data
    assert {f: getattr(res, f) for f in FIELDS[1:]} == n
    if covered is not None:
        assert res.issuers == len(covered)
    if status is not None:
        assert list(res.crl_status) == status
    return n


def _day1(db, dig, crls0, digs0):
    """a day later: more certificates, CRLs that revoke more of them, some revocations dropped, some sets expired"""
    cfg2 = oracle.synth_cfg(tgc.N, seed=7, n_issuers=16, dup_mode=1)
    b2, o2, i2 = oracle.synth_corpus(cfg2, 0, tgc.N)
    ib2, io2 = oracle.synth_issuers(cfg2)
    db.store_batch(b2, o2, ib2, io2, i2, NOW_NS)
    fresh = [bytes([0x21, n]) * (1 + n % 19) for n in range(60)]
    db.preload_known(HOUR + 30, dig[0], fresh)
    db.preload_known(HOUR + 31, dig[2], fresh[:20])
    db.preload_known(HOUR + 32, dig[0], fresh[:5])                          # serials under two hours
    rec = tgc._records(db)
    known = lambda d: sorted({s for h, dg, s in rec if dg == d})  # noqa: E731
    e = lambda s: cb.entry(s, 1767100000)  # noqa: E731
    crls = [crls0[0], crls0[2], crls0[3], crls0[4], crls0[5]]                # crls0[1] gone: its revocations are dropped
    digs = [digs0[0], digs0[2], digs0[3], digs0[4], digs0[5]]
    crls.append(cb.crl(entries=[e(s) for s in known(dig[0])[2::5] + fresh[::2]])); digs.append(dig[0])
    crls.append(cb.crl(entries=[e(s) for s in known(dig[2])[1::6] + fresh[:20:3]])); digs.append(dig[2])
    return crls, digs, fresh


@gpu
def test_a_day_later_and_a_second_day():
    corpus = _corpus()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dig = tgc._fill(db, corpus)
        crls0, digs0 = tgc._crls(db, dig)
        flt = db.revoked_cascade(crls0, digs0, NOW, b"day0").bytes
        R0, _, _, _ = tgc._model(tgc._records(db), crls0, digs0, set(dig))
        same = db.revoked_stash(crls0, digs0, NOW, flt)                       # the filter's own day: nothing new
        assert same.bytes == b"" and (same.revoked, same.in_filter, same.serials) == (len(R0), len(R0), 0)
        crls, digs, fresh = _day1(db, dig, crls0, digs0)
        now1 = NOW + 8 * 3600                                                # sets of hours up to HOUR + 8 expire
        R, S, covered, status = tgc._model(tgc._records(db), crls, digs, set(dig), now1)
        res = db.revoked_stash(crls, digs, now1, flt)
        n = _check(res, R, flt, b"", covered, status)
        assert n["serials"] > 20 and n["in_filter"] > 50 and len(R) > len(set(R))
        # a second day: the first stash has been published; more revocations
        e = lambda s: cb.entry(s, 1767200000)  # noqa: E731
        crls2 = crls + [cb.crl(entries=[e(s) for s in fresh[1::2]])]
        digs2 = digs + [dig[0]]
        R2, _, covered2, status2 = tgc._model(tgc._records(db), crls2, digs2, set(dig), now1)
        res2 = db.revoked_stash(crls2, digs2, now1, flt, res.bytes)
        n2 = _check(res2, R2, flt, res.bytes, covered2, status2)
        assert n2["in_stashes"] >= n["serials"] and 0 < n2["serials"] < n["serials"] + 40


def _corpus():
    cfg = oracle.synth_cfg(tgc.N, n_issuers=16, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, tgc.N)
    iblob, ioffs = oracle.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


SALTS = (b"", b"\x01", bytes(range(18)), bytes(range(1, 20)), bytes(range(7, 39)))
SIZES = ((3000, 3000), (2500, 3000), (3000, 2600), (2800, 2800), (3000, 2900))


def _stops(d, x):
    """the level x stops at in the decoded filter d, or 0 when every level contains it"""
    for level, k, m, bits in d["levels"]:
        if not cm._contains(bits, d["salt"], level, k, m, x):
            return level
    return 0


@pytest.fixture(scope="module")
def walk():
    """a db whose live records are one universe of keys with serials of 1 to 39 octets under three issuers, every one
    revoked by the CRLs, plus a serial under two hours; filters from cascade_model.build over parts of that universe"""
    rng = random.Random(11)
    corpus = _corpus()
    db = engine.GpuCertDatabase(device=0, table_capacity=1 << 16)
    try:
        dense = [int(d) for d in db.register_issuers(corpus[3], corpus[4])]
        dig = [db.issuer_digest(d) for d in dense[:3]]
        keys = list(dict.fromkeys(dig[i % 3] + bytes([rng.randrange(1, 128)]) + rng.randbytes(i % 39) for i in range(6400)))
        for i, d in enumerate(dig):
            db.preload_known(HOUR + 50, d, [x[32:] for x in keys if x[:32] == d])
        two = keys[3000]                                                     # in every filter's S: always new
        db.preload_known(HOUR + 51, two[:32], [two[32:]])                    # one serial under two hours
        crls = [cb.crl(entries=[cb.entry(x[32:], 1767000000) for x in keys if x[:32] == d]) for d in dig]
        filters = []
        for salt, (nr, ns) in zip(SALTS, SIZES):
            R0, S0 = keys[:nr], keys[nr:nr + ns]                             # keys[nr + ns:]: outside the filter's universe
            filters.append(cm.build(R0, S0, salt))
        R = keys + [two]
        yield db, dig, crls, R, filters
    finally:
        db.close()


@gpu
def test_every_level_of_the_walk(walk):
    db, dig, crls, R, filters = walk
    parity = set()
    for flt in filters:
        d = cm.decode(flt)
        L = len(d["levels"])
        assert L >= 12
        parity.add(L % 2)
        assert any(m % 8 for _, _, m, _ in d["levels"]) and any(m % 32 for _, _, m, _ in d["levels"])
        assert {_stops(d, x) for x in R} == set(range(L + 1))               # every level, and all L levels
        res = db.revoked_stash(crls, dig, NOW, flt)
        n = _check(res, R, flt, b"", {*dig}, [0, 0, 0])
        assert n["in_filter"] > 2000 and n["serials"] > 2000
    assert parity == {0, 1}


@gpu
def test_earlier_stashes(walk):
    db, dig, crls, R, filters = walk
    flt = filters[0]
    new, _ = sm.stash(R, flt)
    units = sm.decode(new)
    pairs = [(d, s) for d, ss in units for s in ss]
    assert any(d + s == R[-1] for d, s in pairs)                             # the serial under two hours is new
    first, second = sm.encode(pairs[::3]), sm.encode(pairs[1::3] + [(R[-1][:32], R[-1][32:])])
    unknown = struct.pack("<IB", 2, 32) + b"\xee" * 32 + b"\x01\x05" + bytes([len(pairs[2][1])]) + pairs[2][1]
    long = struct.pack("<IB", 2, 32) + dig[1] + b"\x2d" + b"\x01" * 45 + b"\x28" + b"\x01" * 40
    zero = struct.pack("<IB", 0, 32) + dig[0] + struct.pack("<IB", 0, 32) + b"\x00" * 32
    for stashes in (b"", first, first + second, unknown, long, zero, zero + first + unknown + long + second):
        n = _check(db.revoked_stash(crls, dig, NOW, flt, stashes), R, flt, stashes)
        if stashes and second in stashes:
            assert n["in_stashes"] == len(set(pairs[::3] + pairs[1::3] + [(R[-1][:32], R[-1][32:])])) + 1  # two hours: twice


def _ctypes(b):
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")


@gpu
def test_groups_and_other_capacities_give_the_same_bytes():
    corpus = _corpus()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        dig = tgc._fill(db, corpus)
        crls0, digs0 = tgc._crls(db, dig)
        flt = db.revoked_cascade(crls0, digs0, NOW, b"g").bytes
        crls, digs, _ = _day1(db, dig, crls0, digs0)
        want = db.revoked_stash(crls, digs, NOW, flt)
        assert want.serials > 20
        ck = db.checkpoint()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 18) as other:
        other.load_checkpoint(ck)
        assert other.revoked_stash(crls, digs, NOW, flt).bytes == want.bytes
    for w in (1, 2, 3, 8):
        with engine.GpuCertGroup([0] * w, table_capacity=1 << 16) as g:
            g.load_checkpoint(ck)
            got = g.revoked_stash(crls, digs, NOW, flt)
            assert got.bytes == want.bytes, w
            assert all(getattr(got, f) == getattr(want, f) for f in FIELDS), w
            assert np.array_equal(got.crl_status, want.crl_status)


def _level(level, k, m, bits):
    return struct.pack("<BIIB", 2, m, k, level) + bits


HDR = struct.pack("<HBB", 2, 0, 0)
ONE = _level(1, 1, 8, b"\x00")
BAD_FILTERS = [b"", b"\x02\x00\x00", struct.pack("<HBB", 1, 0, 0) + ONE, struct.pack("<HBB", 2, 1, 0) + ONE,
               struct.pack("<HBB", 2, 0, 33) + b"\x00" * 33 + ONE, HDR + b"\x00" * 3, HDR, HDR + ONE + b"\x00",
               HDR + struct.pack("<BIIB", 1, 8, 1, 1) + b"\x00", HDR + _level(1, 0, 8, b"\x00"), HDR + _level(1, 65, 8, b"\x00"),
               HDR + _level(1, 1, 7, b"\x00"), HDR + _level(2, 1, 8, b"\x00"), HDR + _level(1, 1, 9, b"\x00"),
               HDR + _level(1, 1, 9, b"\x00\x02"), HDR + ONE + _level(3, 1, 8, b"\x00"), HDR + ONE + b"\x02" + b"\x00" * 8]
D = b"\x01" * 32
BAD_STASHES = [b"\x01", struct.pack("<IB", 1, 32) + D, struct.pack("<IB", 1, 32) + D + b"\x03\x01\x02",
               struct.pack("<IB", 0, 20) + D, struct.pack("<IB", 0, 32) + D[:31], sm.encode([(D, b"\x01")]) + b"\x00"]


@gpu
def test_refusals(walk):
    db, dig, crls, R, filters = walk
    lib = capi.load()
    b, keep = engine._crl_batch(crls, dig)
    for f in BAD_FILTERS:
        with pytest.raises(ValueError):
            sm.check_filter(f)
        with pytest.raises(CtmrError) as ei:
            db.revoked_stash(crls, dig, NOW, f)
        assert ei.value.code == capi.E_INVALID, f
    assert db.revoked_stash(crls, dig, NOW, HDR + _level(1, 64, 9, b"\x00\x01")).serials > 0   # k = 64 is allowed
    for s in BAD_STASHES:
        with pytest.raises(CtmrError) as ei:
            db.revoked_stash(crls, dig, NOW, filters[0], s)
        assert ei.value.code == capi.E_INVALID, s
    flt = _ctypes(filters[0])
    o = capi.StashOut()
    assert lib.ctmr_revoked_stash(db.handle, None, NOW, flt, len(filters[0]), None, 0, C.byref(o)) == capi.E_INVALID
    assert lib.ctmr_revoked_stash(db.handle, C.byref(b), NOW, flt, len(filters[0]), None, 0, None) == capi.E_INVALID
    assert lib.ctmr_revoked_stash(db.handle, C.byref(b), NOW, None, len(filters[0]), None, 0, C.byref(o)) == capi.E_INVALID
    assert lib.ctmr_revoked_stash(db.handle, C.byref(b), NOW, flt, len(filters[0]), None, 5, C.byref(o)) == capi.E_INVALID
    assert lib.ctmr_revoked_stash(db.handle, C.byref(b), NOW, flt, len(filters[0]), None, 0, C.byref(o)) == capi.E_BATCH_TOO_LARGE
    with engine.GpuCertGroup([0, 0], table_capacity=1 << 15) as g:
        member = lib.ctmr_group_member(g.handle, 1)
        assert lib.ctmr_revoked_stash(member, C.byref(b), NOW, flt, len(filters[0]), None, 0, C.byref(o)) == capi.E_INVALID
    big = cb.crl(entries=[cb.entry(b"\x01", 1767000000)] * 600)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16, max_batch_bytes=4096) as small:
        with pytest.raises(CtmrError) as ei:
            small.revoked_stash([big], [b"\x00" * 32], NOW, filters[0])
        assert ei.value.code == capi.E_BATCH_TOO_LARGE
        assert small.revoked_stash([], [], NOW, filters[0]).bytes == b""      # still usable


def _peer_worker(rank, world, flt):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi, engine, sharded
    db = engine.GpuCertDatabase(device=0, table_capacity=1 << 15, max_batch_entries=512, max_round_entries=512)
    sharded.attach_peers(db)
    try:
        db.revoked_stash([], [], NOW, flt)
        code = 0
    except capi.CtmrError as e:
        code = e.code
    # the ranks are still in step: a collective call after the refusal completes on both
    empty = db.revoked_cascade([], [], NOW)
    db.close()
    dist.destroy_process_group()
    return code, empty.levels


@gpu
def test_a_ctx_attached_to_peers_is_refused_on_every_rank():
    flt = cm.build([], [])
    outs = run_ranks(_peer_worker, 2, (flt,), timeout=300)
    assert outs == {0: (capi.E_INVALID, 1), 1: (capi.E_INVALID, 1)}


@gpu
def test_caps_and_read_only():
    corpus = _corpus()
    lib = capi.load()
    cfg2 = oracle.synth_cfg(tgc.N, seed=9, n_issuers=16, dup_mode=1)
    b2, o2, i2 = oracle.synth_corpus(cfg2, 0, tgc.N)
    ib2, io2 = oracle.synth_issuers(cfg2)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db, \
            engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as twin:
        dig = tgc._fill(db, corpus)
        crls0, digs0 = tgc._crls(db, dig)
        flt = db.revoked_cascade(crls0, digs0, NOW).bytes
        crls, digs, _ = _day1(db, dig, crls0, digs0)
        twin.load_checkpoint(db.checkpoint())
        before = (db.checkpoint().tobytes(), db.next_index(), list(db.status_counters()), db.issuer_counts())
        want = db.revoked_stash(crls, digs, NOW, flt)
        assert (db.checkpoint().tobytes(), db.next_index(), list(db.status_counters()), db.issuer_counts()) == before
        assert len(want.bytes) > 100
        # a cap one byte short: only bytes is written; the retry with that cap gives exactly those bytes
        b, keep = engine._crl_batch(crls, digs)
        fb = _ctypes(flt)
        buf = np.full(len(want.bytes) + 64, 0xAB, np.uint8)
        status = np.full(len(crls), 0xCD, np.uint8)
        o = capi.StashOut(buf.ctypes.data, len(want.bytes) - 1, 0, status.ctypes.data)
        assert lib.ctmr_revoked_stash(db.handle, C.byref(b), NOW, fb, len(flt), None, 0, C.byref(o)) == capi.E_BATCH_TOO_LARGE
        assert o.bytes == len(want.bytes) and (buf == 0xAB).all() and (status == 0xCD).all()
        assert all(getattr(o, f) == 0 for f in FIELDS)
        o = capi.StashOut(buf.ctypes.data, o.bytes, 0, status.ctypes.data)
        assert lib.ctmr_revoked_stash(db.handle, C.byref(b), NOW, fb, len(flt), None, 0, C.byref(o)) == 0
        assert buf[:o.bytes].tobytes() == want.bytes and (buf[o.bytes:] == 0xAB).all()
        assert np.array_equal(status, want.crl_status)
        # a small default buffer is grown by the binding
        assert db.revoked_stash(crls, digs, NOW, flt, cap=16).bytes == want.bytes
        # the calls that follow give what they give on the untouched twin
        got, exp = db.revoked_cascade(crls, digs, NOW, b"z"), twin.revoked_cascade(crls, digs, NOW, b"z")
        assert got.bytes == exp.bytes
        got, exp = db.revoked_known(crls, digs), twin.revoked_known(crls, digs)
        for name, _ in engine.RevokedResult._CRL + engine.RevokedResult._ENTRY:
            assert np.array_equal(getattr(got, name), getattr(exp, name)), name
        got, exp = (x.store_batch(b2, o2, ib2, io2, i2, NOW_NS) for x in (db, twin))
        for name in ("status", "exp_hour", "serial_off", "serial_len", "was_unknown", "first_issuer_hour"):
            assert np.array_equal(getattr(got, name), getattr(exp, name)), name
        assert (db.next_index(), list(db.status_counters()), db.issuer_counts()) == \
            (twin.next_index(), list(twin.status_counters()), twin.issuer_counts())


@gpu
def test_2_26_slots_several_chunks_counts_and_bytes():
    rng = np.random.default_rng(12)
    _, _, _, iblob, ioffs = _corpus()
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
        res = db.revoked_stash(crls, digs, NOW, flt)
    live = (when > 0) & (who < 3)
    R = [dig[who[i]] + rows[i].tobytes() for i in np.nonzero(live & rev)[0].tolist()]
    n_ = _check(res, R, flt, b"")
    assert res.issuers == 3 and n_["serials"] > 0.9 * int((live & more).sum())
