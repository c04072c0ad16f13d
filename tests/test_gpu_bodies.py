"""Whole get-entries bodies on the GPU (ctmr_process_raw_bodies, include/ctmr_frontend.h) against a twin db fed by
ctmr_process_raw with the spans tests/bodies_oracle.py finds (escaped strings replaced by their unescaped text): every
per-entry output, the body statuses and counts, the string spans, the next index and the counters.  Marked gpu."""
import numpy as np
import pytest

import bodies_oracle as bo
from bodies_pair import PATH_FIELDS, RAW_FIELDS, next_idx, run_pair, synth_bodies  # noqa: F401 (re-exported)
from conftest import NOW_NS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


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
