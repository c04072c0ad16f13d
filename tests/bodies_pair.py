"""Whole get-entries bodies on the GPU (ctmr_process_raw_bodies) against a twin db fed by ctmr_process_raw with the spans
tests/bodies_oracle.py finds (escaped strings replaced by their unescaped text): `run_pair` compares every per-entry
output, the body statuses and counts, the string spans, the next index and the counters.  `lay_out` puts the bodies in
the caller's text the way each of Bodies::upload's two layouts is chosen."""
import ctypes as C

import numpy as np

import bodies_oracle as bo
from conftest import NOW_NS

RAW_FIELDS = ("entry_status", "entry_type", "timestamp_ms", "issuer", "leaf_src", "leaf_off", "leaf_len")
PATH_FIELDS = ("status", "sha256", "exp_hour", "serial_off", "serial_len", "was_unknown", "first_issuer_hour")
# junk between bodies in one copy of the caller's text: open quotes and dangling backslashes that must not carry into a body
JUNK = (b'"', b'\\', b'"abc\\', b"x" * 63 + b'"\\', b'\\"{[', b"", b'"' * 3 + b"\\" * 5)


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


def lay_out(bodies, layout, gaps=None):
    """(text, offs) for one of Bodies::upload's layouts.  "one_copy": the bodies in order, gaps[k] (JUNK in turn by
    default) before body k; a chunk whose bodies lie in order and close together is copied once as it is, so a body's
    staged offset is its offset minus the chunk's first.  "packed": the bodies in reverse order, which upload packs back to
    back in body order, so a body's staged offset is the sum of the lengths before it in its chunk."""
    if layout == "one_copy":
        text, offs = bytearray(), []
        for k, b in enumerate(bodies):
            text += JUNK[k % len(JUNK)] if gaps is None else gaps[k]
            offs.append(len(text))
            text += b
        text += b'"\\'
        return bytes(text), np.array(offs, np.uint64)
    assert layout == "packed", layout
    if not bodies:
        return b"", np.zeros(0, np.uint64)
    order = list(range(len(bodies)))[::-1]
    pos = np.cumsum([0] + [len(bodies[i]) for i in order[:-1]])
    offs = np.zeros(len(bodies), np.uint64)
    offs[order] = pos
    return b"".join(bodies[i] for i in order), offs


def run_pair(db, twin, bodies, maxes, text=None, offs=None, layout=None, gaps=None, **kw):
    """the bodies call on db and the twin's ctmr_process_raw call; compares everything.  The bodies are back to back in
    order unless text and offs say where they are, or layout (and gaps) has lay_out place them."""
    if layout is not None:
        text, offs = lay_out(bodies, layout, gaps)
    elif text is None:
        text = b"".join(bodies)
        offs = np.cumsum([0] + [len(b) for b in bodies[:-1]]).astype(np.uint64)
    lens = np.array([len(b) for b in bodies], np.uint32)
    ttext, lo, ll, xo, xl, sts, cnts = bo.twin_batch(bodies, maxes)
    n0 = next_idx(db)
    t0 = twin.next_index()
    r = db.store_raw_bodies(text, offs, lens, np.array(maxes, np.uint32), NOW_NS, **kw)
    t = twin.store_raw_entries(ttext, np.array(lo, np.uint64), np.array(ll, np.uint32), np.array(xo, np.uint64), np.array(xl, np.uint32),
                               NOW_NS, **kw)
    diff = [k for k in range(len(sts)) if int(r.body_status[k]) != sts[k]]
    assert not diff, [(k, int(r.body_status[k]), sts[k], len(bodies[k]), bodies[k][:96]) for k in diff[:4]]
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
