"""Whole get-entries bodies on the GPU (ctmr_process_raw_bodies, include/ctmr_frontend.h) against a twin db fed by
ctmr_process_raw with the spans tests/bodies_oracle.py finds (escaped strings replaced by their unescaped text): every
per-entry output, the body statuses and counts, the string spans, the next index and the counters.  Marked gpu."""
import ctypes as C

import numpy as np
import pytest

import bodies_oracle as bo
from conftest import NOW_NS

pytestmark = pytest.mark.gpu

RAW_FIELDS = ("entry_status", "entry_type", "timestamp_ms", "issuer", "leaf_src", "leaf_off", "leaf_len")
PATH_FIELDS = ("status", "sha256", "exp_hour", "serial_off", "serial_len", "was_unknown", "first_issuer_hour")


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def synth_bodies(n, page=1000, seed=20260922):
    """n synthetic entries as back-to-back bodies of `page` entries (ctmr_synth_raw_pages_host)"""
    from ct_mapreduce_b200 import capi
    L = capi.load()
    cfg = capi.synth_cfg(n, seed=seed, n_issuers=64)
    need = L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, page, None, 0, None, None, None, None)
    text = np.zeros(need, np.uint8)
    lo, ll, xo, xl = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    assert L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, page, capi.ptr(text), need, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo),
                                       capi.ptr(xl)) == need
    starts = [int(lo[a]) - len(b'{"entries":[{"leaf_input":"') for a in range(0, n, page)] + [need]
    return text.tobytes(), [text[starts[k]:starts[k + 1]].tobytes() for k in range(len(starts) - 1)]


def next_idx(d):
    from ct_mapreduce_b200 import engine
    if isinstance(d, engine.GpuCertGroup):  # a group's next index is in its snapshot header
        return int(np.frombuffer(d.snapshot()[48:56].tobytes(), np.uint64)[0])
    return d.next_index()


def run_pair(db, twin, bodies, maxes, text=None, offs=None, **kw):
    """the bodies call on db and the twin's ctmr_process_raw call; compares everything"""
    if text is None:
        text = b"".join(bodies)
        offs = np.cumsum([0] + [len(b) for b in bodies[:-1]]).astype(np.uint64)
    lens = np.array([len(b) for b in bodies], np.uint32)
    ttext, lo, ll, xo, xl, sts, cnts = bo.twin_batch(bodies, maxes)
    n0 = next_idx(db)
    t0 = twin.next_index()
    r = db.store_raw_bodies(text, offs, lens, np.array(maxes, np.uint32), NOW_NS, **kw)
    t = twin.store_raw_entries(ttext, np.array(lo, np.uint64), np.array(ll, np.uint32), np.array(xo, np.uint64), np.array(xl, np.uint32),
                               NOW_NS, **kw)
    assert r.body_status.tolist() == sts
    assert r.body_entries.tolist() == cnts
    assert r.body_first.tolist() == np.cumsum([0] + cnts[:-1]).tolist()
    assert r.n_entries == sum(cnts) and next_idx(db) - n0 == sum(cnts) == twin.next_index() - t0
    for f in RAW_FIELDS:
        if f != "issuer":
            assert np.array_equal(getattr(r, f), getattr(t, f)), f
    # dense issuer indices are handed out in the order a parallel look-up meets new Chain[0]s: compare the issuers
    dense = r.issuer < 0xFFFFFFFE
    assert np.array_equal(dense, t.issuer < 0xFFFFFFFE) and np.array_equal(r.issuer[~dense], t.issuer[~dense])
    assert [db.issuer_digest(int(i)) for i in r.issuer[dense]] == [twin.issuer_digest(int(i)) for i in t.issuer[dense]]
    for f in PATH_FIELDS + (("issuer_name_off", "issuer_name_len", "crldp_off", "crldp_len", "first_issuer_dn", "first_crldp")
                            if kw.get("want_meta") else ()):
        assert np.array_equal(getattr(r.path, f), getattr(t.path, f)), f
    if kw.get("want_pem"):
        assert np.array_equal(r.path.pem_off, t.path.pem_off) and r.path.pem[:int(r.path.pem_off[-1])].tobytes() == \
            t.path.pem[:int(t.path.pem_off[-1])].tobytes()
    # the spans as found, in the caller's text
    k = 0
    for body, off, mx in zip(bodies, offs, maxes):
        st, ents = bo.parse_body(body, mx)
        for leaf, extra in ents:
            for s, o_, l_, bit in ((leaf, r.leaf_input_off, r.leaf_input_len, 1), (extra, r.extra_data_off, r.extra_data_len, 2)):
                assert (int(o_[k]), int(l_[k])) == ((0, 0) if s is None else (int(off) + s.off, s.len)), k
                assert bool(r.escaped[k] & bit) == bool(s is not None and s.escaped), k
            k += 1
    assert {a: v for a, v in db.issuer_counts().items() if v} == {a: v for a, v in twin.issuer_counts().items() if v}
    assert np.array_equal(db.status_counters(), twin.status_counters())
    return r


def corpus():
    """the rule corpus around real synthetic entries: (body, max) pairs"""
    _, pages = synth_bodies(12, page=3, seed=5)
    s, ents = bo.parse_body(pages[0], 3)
    assert s == bo.BODY_OK
    (l0, x0), (l1, x1), (l2, x2) = [(e[0].data, e[1].data) for e in ents]
    _, ents = bo.parse_body(pages[1], 3)
    (l3, x3), (l4, x4), _ = [(e[0].data, e[1].data) for e in ents]

    def esc(s):  # every '/' as '\/', a '\n' and a 'A'-style escape in the middle
        h = len(s) // 2
        return s[:h].replace(b"/", b"\\/") + b"\\n\\r\\u00" + b"%02x" % s[h] + s[h + 1:]
    out = [
        (pages[0], 3),
        (b' {\n\t"entries" : [ {"extra_data" :"' + x0 + b'" , "leaf_input": "' + l0 + b'" } , null ,{} ]\r\n} ', 3),
        (b'{"ENTRIES":[{"Leaf_Input":"' + l1 + b'","EXTRA_DATA":"' + x1 + b'","leaf_input":"' + l2 + b'"}]}', 1),
        ('{"entrieſ":[{"leaf_input":"'.encode() + l3 + b'"}]}', 2),
        (b'{"ent\\u0072ies":[{"leaf\\u005finput":"' + esc(l4) + b'","extra_data":"' + esc(x4) + b'"}]}', 1),
        (b'{"x":{"entries":[{"leaf_input":"' + l0 + b'"}]},"entries":[{"y":{"leaf_input":"' + l1 + b'","extra_data":[' + b"[" * 100 +
         b"]" * 100 + b']},"leaf_input":"' + l2 + b'","extra_data":"' + x2 + b'","z":[[[{"extra_data":"AA=="}]]]}],"w":' +
         b"[" * 300 + b"]" * 300 + b"}", 1),
        (b'{"entries":[{"leaf_input":"A\\u00e9AA","extra_data":null}]}', 1),
        (b'{"entries":null}', 0), (b'{"entries":[]}', 0), (b"null", 0), (b"{}", 5), (b"", 1), (b"\xef\xbb\xbf{}", 1),
        (pages[1], 2),                                                 # TOO_MANY
        (b'{"entries":[],"Entries":[]}', 1),                           # REPEATED_ENTRIES
        (pages[2], 3),
    ]
    for bad in (b"{", b"{}}", b"{} x", b"[1,]", b'{"a":01}', b"NaN", b'{"a":"\x01"}', b'{"a":"\\x"}', b'{"a":"\\u12g4"}', b'{"a":tru}',
                b'{"entries":[{"leaf_input":"abc}]}', b'{"a" 1}'):
        out.append((bad, 1))                                           # BAD_JSON
    for bad in (b"[]", b"1", b'"s"', b'{"entries":{}}', b'{"entries":[1]}', b'{"entries":[{"leaf_input":1}]}',
                b'{"entries":[{"extra_data":{}}]}'):
        out.append((bad, 1))                                           # BAD_TYPE
    out.append((pages[3], 3))
    return out


def test_rule_corpus_mixed_in_one_call(eng):
    bodies, maxes = zip(*corpus())
    statuses = {bo.parse_body(b, m)[0] for b, m in zip(bodies, maxes)}
    assert statuses == {0, 1, 2, 3, 4}
    with eng.GpuCertDatabase(table_capacity=1 << 14, log_expired_entries=True) as db, \
            eng.GpuCertDatabase(table_capacity=1 << 14, log_expired_entries=True) as twin:
        r = run_pair(db, twin, list(bodies), list(maxes))
        assert r.escaped.any() and (r.entry_status == 0).sum() >= 8
        # the same bodies again, out of order in the text (packed on the host), and one at a time
        order = list(range(len(bodies)))[::-1]
        text = b"".join(bodies[i] for i in order)
        pos = np.cumsum([0] + [len(bodies[i]) for i in order[:-1]])
        offs = np.zeros(len(bodies), np.uint64)
        offs[order] = pos
        run_pair(db, twin, list(bodies), list(maxes), text=text, offs=offs)
        for b, m in zip(bodies, maxes):
            run_pair(db, twin, [b], [m])
        assert db.bodies_profile_last() > 0


def test_synthetic_pages_over_several_chunks(eng, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(12 << 20))  # about two bodies per chunk
    _, pages = synth_bodies(6000, page=500)
    with eng.GpuCertDatabase(table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=1500) as db, \
            eng.GpuCertDatabase(table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=1500) as twin:
        r = run_pair(db, twin, pages, [500] * len(pages))
        assert r.n_entries == 6000 and (r.entry_status == 0).all()
        fe_ms, path_ms, launches = db.frontend_profile_last()
        assert 0 < db.bodies_profile_last() < fe_ms
        run_pair(db, twin, pages[:3], [500] * 3)       # everything known now
        assert not (db.store_raw_bodies(b"{}", [0], [2], [1000], NOW_NS).n_entries)


def test_pem_and_string_identities(eng):
    bodies, maxes = zip(*corpus())
    with eng.GpuCertDatabase(table_capacity=1 << 14, log_expired_entries=True, max_batch_entries=8) as db, \
            eng.GpuCertDatabase(table_capacity=1 << 14, log_expired_entries=True, max_batch_entries=8) as twin:
        run_pair(db, twin, list(bodies), list(maxes), want_pem=True, want_meta=True)


def test_group_of_three_shards_on_one_gpu(eng, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(4 << 20))
    _, pages = synth_bodies(3000, page=250, seed=9)
    bodies = pages + [b for b, _ in corpus()]
    maxes = [250] * len(pages) + [m for _, m in corpus()]
    with eng.GpuCertGroup([0, 0, 0], table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=600) as g, \
            eng.GpuCertDatabase(table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=600) as twin:
        run_pair(g, twin, bodies, maxes, want_pem=True)
        run_pair(g, twin, bodies[:5], maxes[:5])


def test_arguments_and_budgets(eng):
    from ct_mapreduce_b200 import capi
    with eng.GpuCertDatabase(table_capacity=1 << 12, max_batch_entries=64) as db:
        with pytest.raises(capi.CtmrError) as e:
            db.store_raw_bodies(b"{}", [1], [2], [1], NOW_NS)              # outside the text
        assert e.value.code == capi.E_INVALID
        with pytest.raises(capi.CtmrError) as e:                           # a later body outside the text: no index taken
            db.store_raw_bodies(b"{}{}", [0, 3], [2, 2], [7, 9], NOW_NS)
        assert e.value.code == capi.E_INVALID and db.next_index() == 0
        with pytest.raises(capi.CtmrError) as e:
            db.store_raw_bodies(b"{}", [0], [2], [65], NOW_NS)             # more requested than a chunk holds
        assert e.value.code == capi.E_BATCH_TOO_LARGE
        assert db.next_index() == 0
        r = db.store_raw_bodies(b"", np.zeros(0, np.uint64), [], [], NOW_NS)
        assert r.n_entries == 0 and db.next_index() == 0


def test_bodies_in_order_with_junk_between_them(eng):
    """One copy of the caller's text, gaps included: an unclosed quote and a trailing backslash in the junk before a body
    must not carry into it (both carries restart at every body start, at every offset within a block)."""
    bodies, maxes = zip(*corpus())
    junks = [b'"', b'\\', b'"abc\\', b"x" * 63 + b'"\\', b'\\"{[', b"", b'"' * 3 + b"\\" * 5]
    text, offs = bytearray(), []
    for k, b in enumerate(bodies):
        text += junks[k % len(junks)]
        offs.append(len(text))
        text += b
    text += b'"\\'
    with eng.GpuCertDatabase(table_capacity=1 << 14, log_expired_entries=True) as db, \
            eng.GpuCertDatabase(table_capacity=1 << 14, log_expired_entries=True) as twin:
        r = run_pair(db, twin, list(bodies), list(maxes), text=bytes(text), offs=np.array(offs, np.uint64))
        assert (r.entry_status == 0).sum() >= 8
