"""ctmr_revoked_known / ctmr_group_revoked_known on the GPU against crl_oracle: the CRLs are parsed byte by byte on the
host and joined with the serials:: sets the test put into the table (ctmr_process_batch over the synthetic corpus, and
preloads of crafted serials)."""
import numpy as np
import pytest

import crl_build as cb
import crl_oracle as co
from ct_mapreduce_b200 import capi, engine
from ct_mapreduce_b200.capi import CtmrError
from oracle import oracle

pytestmark = pytest.mark.gpu

NOW_NS = 1767225600 * 10**9
N = 4096


@pytest.fixture(scope="module")
def corpus():
    cfg = oracle.synth_cfg(N, n_issuers=16, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, N)
    iblob, ioffs = oracle.synth_issuers(cfg)
    want = oracle.DB().process(blob, offs, iblob, ioffs, idx, NOW_NS)
    return blob, offs, idx, iblob, ioffs, want


def _digests(db, iblob, ioffs):
    dense = db.register_issuers(iblob, ioffs)
    return [db.issuer_digest(int(d)) for d in dense]


def _fill(db, corpus):
    """The table: the corpus through ctmr_process_batch and crafted preloads; returns (sets, digests of the issuers)."""
    blob, offs, idx, iblob, ioffs, want = corpus
    db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
    dig = _digests(db, iblob, ioffs)
    sets = {}
    for i in np.nonzero(want.status == 0)[0]:
        s = bytes(blob[offs[i] + want.serial_off[i]: offs[i] + want.serial_off[i] + want.serial_len[i]])
        sets.setdefault((int(want.exp_hour[i]), dig[idx[i]]), set()).add(s)
    crafted = [(500000, 0, [b"\x00\xaa", b"\x05", b"\x77\x77"]), (500100, 0, [b"\x77\x77"]), (500200, 1, [b"\x05"])]
    for hour, k, ss in crafted:
        db.preload_known(hour, dig[k], ss)
        sets.setdefault((hour, dig[k]), set()).update(ss)
    return sets, dig


def _crls(corpus, dig, sets):
    """A mix of CRLs: known and unknown serials, serials known under another issuer, 00aa and non-minimal encodings, one
    serial under two hours, duplicates across CRLs, indirect entries, a delta CRL, malformed CRLs between good ones and
    an unknown issuer digest."""
    rng = np.random.default_rng(5)
    known0 = sorted(s for (h, d), ss in sets.items() if d == dig[0] for s in ss)
    known1 = sorted(s for (h, d), ss in sets.items() if d == dig[1] for s in ss)
    e = lambda s, **kw: cb.entry(s, 1767000000 - int(rng.integers(0, 10**6)), **kw)
    crls, digs = [], []
    ents0 = [e(s) for s in known0[:200]] + [e(b"\x00\xaa"), e(b"\x00\x05"), e(b"\x77\x77", reason=1), e(b"\x12\x34" * 5),
                                             e(known1[0]), e(b"\x05", cert_issuer=True), e(b"\x01" * 40), e(known0[0], generalized=True),
                                             e(b"\x42", seconds=False)]
    crls.append(cb.crl(entries=ents0)); digs.append(dig[0])
    crls.append(cb.crl(entries=[e(s) for s in known0[100:300]] + [e(b"\x05", reason=4)])); digs.append(dig[0])  # duplicates
    crls.append(cb.crl(entries_raw=e(b"\x05") + b"\x30\x01\x02")); digs.append(dig[0])                      # bad entries
    crls.append(cb.crl(entries=[e(s) for s in known1[:50]], delta=True, idp=True)); digs.append(dig[1])
    crls.append(cb.crl(entries=[e(b"\x05")])[:-1]); digs.append(dig[1])                                      # truncated
    crls.append(cb.crl(entries=[e(s) for s in known1[:50]])); digs.append(b"\xee" * 32)                     # unknown issuer
    crls.append(cb.crl(entries=None, version=None, next_update=None)); digs.append(dig[1])                  # v1, no entries
    crls.append(cb.crl(entries=[e(s) for s in known1[:80]] + [e(b"\x05")], trailing=b"\x00")); digs.append(dig[1])  # trailing
    crls.append(cb.crl(entries=[e(s) for s in known1[:80]] + [e(b"\x05")])); digs.append(dig[1])
    return crls, digs


def _check(res, crls, digs, sets, registered):
    data, offs, _ = engine.pack_crls(crls)
    e = 0
    for k, der in enumerate(crls):
        p = co.parse_crl(der)
        j = co.join(p, digs[k], sets, registered)
        assert res.crl_status[k] == j["status"], k
        if j["status"] not in (co.CRL_OK, co.CRL_UNKNOWN_ISSUER):
            assert res.crl_entries[k] == 0
            continue
        assert res.crl_flags[k] == p["flags"] and res.this_update[k] == p["this_update"] and res.next_update[k] == p["next_update"]
        assert (res.tbs_off[k] - offs[k], res.tbs_len[k]) == p["tbs"]
        assert (res.issuer_name_off[k] - offs[k], res.issuer_name_len[k]) == p["name"]
        assert res.crl_first[k] == e and res.crl_entries[k] == len(p["entries"]), k
        for i, pe in enumerate(p["entries"]):
            g = e + i
            assert res.serial(data, g) == pe["serial"]
            assert res.serial_off[g] == offs[k] + pe["serial_pos"]
            assert (res.revoked_at[g], res.reason[g], res.entry_status[g]) == (pe["revoked_at"], pe["reason"], pe["status"]), (k, i)
            assert (res.known[g], res.known_exp_hour[g], res.known_sets[g]) == j["answers"][i], (k, i, pe["serial"])
        e += len(p["entries"])
    assert res.n_entries == e


def test_every_output_against_the_oracle(corpus):
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        sets, dig = _fill(db, corpus)
        crls, digs = _crls(corpus, dig, sets)
        res = db.revoked_known(crls, digs)
        _check(res, crls, digs, sets, set(dig))
        assert res.known.sum() > 200 and (res.known_sets > 1).any()
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16, max_batch_bytes=8192) as db:  # chunks of 8 KiB
        _fill(db, corpus)
        small = db.revoked_known(crls, digs)
        for name, _ in engine.RevokedResult._CRL + engine.RevokedResult._ENTRY:
            assert np.array_equal(getattr(small, name), getattr(res, name)), name


def test_entry_cap_too_small_reports_the_count(corpus):
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        sets, dig = _fill(db, corpus)
        crls, digs = _crls(corpus, dig, sets)
        need = db.revoked_known(crls, digs).n_entries
        with pytest.raises(CtmrError) as ei:
            db.revoked_known(crls, digs, entry_cap=need - 1)
        assert ei.value.code == capi.E_BATCH_TOO_LARGE and ei.value.n_entries == need
        big = cb.crl(entries=[cb.entry(b"\x01", 1767000000)] * 600)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16, max_batch_bytes=4096) as db:
        with pytest.raises(CtmrError) as ei:
            db.revoked_known([big], [b"\x00" * 32])
        assert ei.value.code == capi.E_BATCH_TOO_LARGE


def test_read_only_and_eviction_and_checkpoint(corpus):
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        sets, dig = _fill(db, corpus)
        crls, digs = _crls(corpus, dig, sets)
        before = (db.checkpoint().tobytes(), db.next_index(), list(db.status_counters()), db.issuer_counts())
        res = db.revoked_known(crls, digs)
        assert (db.checkpoint().tobytes(), db.next_index(), list(db.status_counters()), db.issuer_counts()) == before
        ck = db.checkpoint()
        with engine.GpuCertDatabase(device=0, table_capacity=1 << 18) as other:
            other.load_checkpoint(ck)
            again = other.revoked_known(crls, digs)
            for name, _ in engine.RevokedResult._ENTRY:
                assert np.array_equal(getattr(again, name), getattr(res, name)), name
        db.evict_expired(500150 * 3600)
        live = {(h, d): ss for (h, d), ss in sets.items() if h * 3600 > 500150 * 3600}
        _check(db.revoked_known(crls, digs), crls, digs, live, set(dig))


def test_group_equals_one_ctx_and_refusals(corpus):
    import torch
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        sets, dig = _fill(db, corpus)
        crls, digs = _crls(corpus, dig, sets)
        want = db.revoked_known(crls, digs)
    for devs in ([0, 0, 0], list(range(torch.cuda.device_count()))):
        if len(devs) < 2:
            continue
        with engine.GpuCertGroup(devs, table_capacity=1 << 15) as g:
            gsets, gdig = _fill(g, corpus)
            assert gdig == dig
            got = g.revoked_known(crls, digs)
            for name, _ in engine.RevokedResult._CRL + engine.RevokedResult._ENTRY:
                assert np.array_equal(getattr(got, name), getattr(want, name)), (devs, name)
            lib = capi.load()
            member = lib.ctmr_group_member(g.handle, 1)
            data, offs, lens = engine.pack_crls(crls[:1])
            b = capi.CrlBatch(data.ctypes.data, data.size, offs.ctypes.data, lens.ctypes.data,
                              np.frombuffer(digs[0], np.uint8).ctypes.data, 1)
            o = engine.RevokedResult(1, 1000).to_c()
            assert lib.ctmr_revoked_known(member, b, o) == capi.E_INVALID


def test_two_million_entries_and_ten_thousand_small_crls(corpus):
    rng = np.random.default_rng(11)
    n = 2_000_000
    rows = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    rows[:, 0] = rng.integers(1, 0x80, n, dtype=np.uint8)
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 16) as db:
        sets, dig = _fill(db, corpus)
        known = sorted({x for (h, d), ss in sets.items() if d == dig[2] for x in ss if len(x) == 16})
        for j, s in enumerate(known[:100]):
            rows[j * 19997] = np.frombuffer(s, np.uint8)
        big = cb.bulk_crl(rows)
        res = db.revoked_known([big], [dig[2]])
        assert res.crl_status[0] == co.CRL_OK and res.n_entries == n
        hits = set(np.nonzero(res.known)[0].tolist())
        assert hits == {j * 19997 for j in range(min(100, len(known)))}
        small = [cb.crl(entries=[cb.entry(bytes([1 + i % 100, i >> 8 & 0x7F]), 1767000000)]) for i in range(10_000)]
        r2 = db.revoked_known(small, [dig[i % 3] for i in range(10_000)])
        assert (r2.crl_status == co.CRL_OK).all() and r2.n_entries == 10_000
        assert np.array_equal(r2.crl_first, np.arange(10_000))
