"""The front end at its byte edges, entry by entry against the oracle (no sampling): base64 at every text alignment,
length residue and padding; junk at every character position; RFC 6962 framing fuzz; precertificate TBS shapes;
Issuer.ID for SPKIs across two SHA-256 block boundaries; Chain[0] hash collisions crafted with fe_model, inside a
chunk, across chunks, across calls and after register_issuers; probe chains that wrap in the issuer mirror and the
pending table; the mirror's capacity; and the same pages through a group of three shards.  Marked gpu."""
import base64
import hashlib
import struct

import numpy as np
import pytest

import der_build as D
import fe_model as F
from conftest import NOW_NS, go_pem, pack
from ct_mapreduce_b200 import frontend as fe

pytestmark = pytest.mark.gpu

TS0 = 1_700_000_000_000
PATH_FIELDS = ("status", "was_unknown", "first_issuer_hour", "exp_hour", "serial_off", "serial_len")
JUNK = b"-_=.\n\x00\x80\xff"
FE_LAUNCHES_OUTSIDE_ROUNDS = 6  # per chunk: sizes, scan, decode, frame, tbs + finish; then one fe_issuer per round
CA0 = F.ca(7001, F.rsa_spki(162))


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def leaf(salt: int, **kw) -> bytes:
    kw.setdefault("subject", [[D.cn(b"leaf %d" % salt)]])
    return D.cert(serial=D.serial_bytes(8, salt=salt), **kw).der


def entry(ts: int, cert: bytes, chain, precert: bool = False, ext: bytes = b"", tbs: bytes | None = None):
    if precert:
        return (fe.merkle_tree_leaf_precert(ts, hashlib.sha256(chain[0] if chain else b"").digest(),
                                            fe.tbs_of(cert) if tbs is None else tbs, ext), fe.precert_chain_entry(cert, chain))
    return fe.merkle_tree_leaf_x509(ts, cert, ext), fe.certificate_chain(chain)


def layout(strings, align=None):
    """Base64 strings (already text) laid out in one buffer: string k starts at a chosen offset mod 16 (align[k]),
    separated by a quote.  Returns (text, offsets, lengths)."""
    out, offs = bytearray(b'{"'), []
    for k, s in enumerate(strings):
        if align is not None:
            out += b'"' * ((align[k] - len(out)) % 16)
        offs.append(len(out))
        out += s + b'"'
    return bytes(out), np.array(offs, np.uint64), np.array([len(s) for s in strings], np.uint32)


def raw_pages(entries, align=None, b64=None):
    """(text, lo, ll, xo, xl) for (leaf_input, extra_data) pairs; b64 overrides the encoded strings (for damage)."""
    strings = []
    for li, ed in entries:
        strings += [base64.b64encode(li), base64.b64encode(ed)]
    if b64 is not None:
        for k, s in b64.items():
            strings[k] = s
    text, offs, lens = layout(strings, align)
    return text, offs[0::2].copy(), lens[0::2].copy(), offs[1::2].copy(), lens[1::2].copy()


def issuer_digest_of(ora, der):
    rc, c = ora.parse_cert(der)
    return None if rc != 0 else ora.issuer_id(der[c.spki_off:c.spki_off + c.spki_len])[0]


def check(ora, db, odb, pages, want_pem=False, what=""):
    """Every entry against ora.raw_process: front-end fields, every path field, and the Issuer.ID digest of every
    stored entry.  Returns (gpu result, oracle result)."""
    text, lo, ll, xo, xl = pages
    r_o = ora.raw_process(odb, text, lo, ll, xo, xl, NOW_NS)
    r_g = db.store_raw_entries(text, lo, ll, xo, xl, NOW_NS, want_pem=want_pem)
    for f in ("entry_status", "entry_type", "timestamp_ms"):
        a, b = getattr(r_g, f), getattr(r_o, f)
        bad = np.nonzero(a != b)[0]
        assert bad.size == 0, (what, f, bad[:10], a[bad[:10]], b[bad[:10]])
    located = (r_o.entry_status == 0) | ((r_o.entry_status == ora.FE_BAD_CERT) & (r_o.entry_type == 0))
    for f in ("leaf_src", "leaf_off", "leaf_len"):
        bad = np.nonzero(getattr(r_g, f)[located] != getattr(r_o, f)[located])[0]
        assert bad.size == 0, (what, f, np.nonzero(located)[0][bad[:10]])
    assert not r_g.leaf_len[~located].any(), what
    for f in PATH_FIELDS:
        a, b = getattr(r_g.path, f), getattr(r_o.path, f)
        if f in ("exp_hour", "serial_off", "serial_len"):
            m = r_o.path.status != ora.ST_PARSE_ERR
            a, b = a[m], b[m]
        bad = np.nonzero(a != b)[0]
        assert bad.size == 0, (what, f, bad[:10], a[bad[:10]], b[bad[:10]])
    bad = np.nonzero((r_g.path.sha256 != r_o.path.sha256).any(axis=1))[0]
    assert bad.size == 0, (what, "sha256", bad[:10])
    memo = {}
    for i in np.nonzero(r_o.path.status == 0)[0]:
        der = r_o.issuer_der[i]
        if der not in memo:
            memo[der] = issuer_digest_of(ora, der)
        assert db.issuer_digest(int(r_g.issuer[i])) == memo[der], (what, "issuer", int(i))
    bad_iss = r_o.path.status == ora.ST_ISSUER_PARSE_ERR
    assert (r_g.issuer[bad_iss] == 0xFFFFFFFE).all(), what
    if want_pem:
        for i in range(lo.size):
            assert r_g.path.pem_of(i) == (go_pem(r_o.leaves[i]) if r_o.path.was_unknown[i] else b""), (what, i)
    return r_g, r_o


def same_results(a, b, what):
    """Equal outputs of two runs; dense issuer indices are handed out in registration order, so only their digests
    (checked by check()) are compared."""
    for f in ("entry_status", "entry_type", "timestamp_ms", "leaf_src", "leaf_off", "leaf_len"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), (what, f)
    for f in PATH_FIELDS + ("sha256",):
        assert np.array_equal(getattr(a.path, f), getattr(b.path, f)), (what, f)


# ------------------------------------------------------------------------------------------------ 1. base64 tails

def test_base64_every_alignment_length_and_padding(eng, ora):
    """Certificates of 500..580 bytes (every residue mod 48: mod 3 for the '=' padding, mod 16 for the lane group;
    480..576 include whole PEM lines) and some of 1500, CtExtensions of 0..5 bytes, x509 and precert framings, every
    string starting at each offset mod 16; strings up to ~2 100 characters (several iterations of a lane)."""
    entries = []
    lengths = list(range(500, 581)) + [1500, 1536, 1537, 1538]
    for k, L in enumerate(lengths):
        cert = F.cert_of_length(L, serial=D.serial_bytes(8, salt=100 + k), subject=[[D.cn(b"b64 leaf")]])
        for e in range(6):
            entries.append(entry(TS0 + 10 * k + e, cert.der, [CA0.der], precert=(k + e) % 3 == 0, ext=bytes(range(7, 7 + e))))
    align = [k % 16 for k in range(2 * len(entries))]
    pages = raw_pages(entries, align)
    ll, xl = pages[2], pages[4]
    for lens in (ll, xl):
        assert {int(x) % 16 for x in lens} == {0, 4, 8, 12} and lens.max() > 32 * 16
    text = pages[0]
    pads = {text[int(o) + int(n) - 2:int(o) + int(n)].count(b"=") for o, n in zip(pages[1], ll)}
    assert pads == {0, 1, 2}
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 14) as db:
        r_g, r_o = check(ora, db, odb, pages, want_pem=True, what="b64")
    assert (r_o.entry_status == 0).all() and r_o.path.was_unknown.sum() > 0
    assert {len(x) % 48 for x in r_o.leaves} == set(range(48))


# ------------------------------------------------------------------------------------------------ 2. junk

def test_junk_at_every_position(eng, ora):
    """Each of - _ = . \\n NUL 0x80 0xff at every character position of three strings (padding 0, 1 and 2), the last
    quantum rewritten ('A===', '====', 'QQ=A', 'Q=Q='), a lone '=' appended, a character dropped: FE_BAD_BASE64 exactly
    where the oracle says so; an untouched entry after every damaged one."""
    base = []
    for k, L in enumerate((300, 301, 302)):  # leaf_input of 12 + 3 + L + 2 bytes: padding differs
        cert = F.cert_of_length(L, serial=D.serial_bytes(8, salt=300 + k))
        base.append(entry(TS0 + k, cert.der, [CA0.der]))
    entries, b64 = [], {}

    def add(pair, which, s):
        b64[2 * len(entries) + which] = s
        entries.append(pair)
        entries.append(entry(TS0 + 50_000 + len(entries), leaf(900_000 + len(entries) % 64), [CA0.der]))

    for k, pair in enumerate(base):
        for which in (0, 1):
            s = base64.b64encode(pair[which])
            positions = range(len(s)) if which == 0 or k == 0 else list(range(0, 40)) + list(range(len(s) - 40, len(s)))
            for p in positions:
                for j in JUNK:
                    if s[p] != j:
                        add(pair, which, s[:p] + bytes([j]) + s[p + 1:])
            for q in (b"A===", b"====", b"QQ=A", b"Q=Q=", b"QQ==", b"QUI="):
                add(pair, which, s[:-4] + q)
            add(pair, which, s + b"=")
            add(pair, which, s[:-1])
            add(pair, which, s[:len(s) // 2] + s[len(s) // 2 + 1:])
    pages = raw_pages(entries, [k % 16 for k in range(2 * len(entries))], b64)
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        r_g, r_o = check(ora, db, odb, pages, what="junk")
    st = r_o.entry_status
    assert (st[1::2] == 0).all()  # the untouched neighbours
    assert (st[0::2] == ora.FE_BAD_BASE64).sum() > 10000 and (st[0::2] != ora.FE_BAD_BASE64).any()


# ------------------------------------------------------------------------------------------------ 3. framing fuzz

HOWS = ("ok", "trunc_li", "trunc_ed", "extra_li", "extra_ed", "flip_li", "flip_ed", "type", "leaftype")


def framing_corpus(n=3000, seed=2024):
    """The generator of test_framing_agrees_with_an_independent_reading_of_rfc6962 (all nine kinds of damage), driven by
    a seeded numpy RNG, with der_build certificates where the structure should parse; then fixed edges."""
    rng = np.random.default_rng(seed)
    pool = [D.cert(serial=D.serial_bytes(8, salt=5000 + k), subject=[[D.cn(b"fuzz %d" % k)]], sig_len=17 + k).der for k in range(40)]
    cas = [CA0.der, F.ca(7002, F.rsa_spki(98)).der]
    out = []
    for i in range(n):
        precert = bool(rng.integers(2))
        ts = int(rng.integers(0, 2**63)) * 2 + int(rng.integers(2))
        cert = pool[int(rng.integers(len(pool)))] if rng.integers(4) else rng.bytes(int(rng.integers(1, 41)))
        chain = [cas[int(rng.integers(2))]] if rng.integers(3) else []
        chain += [rng.bytes(int(rng.integers(1, 41))) for _ in range(int(rng.integers(0, 4)))]
        ext = rng.bytes(int(rng.integers(0, 7)))
        how, where = HOWS[int(rng.integers(len(HOWS)))], int(rng.integers(0, 10**6))
        li, ed = entry(ts, cert, chain, precert, ext, tbs=fe.tbs_of(cert) if cert in pool else cert)
        li, ed = bytearray(li), bytearray(ed)
        if how == "trunc_li": del li[where % len(li):]
        elif how == "trunc_ed": del ed[where % len(ed):]
        elif how == "extra_li": li += b"\x00" * (1 + where % 3)
        elif how == "extra_ed": ed += b"\x00" * (1 + where % 3)
        elif how == "flip_li": li[where % len(li)] ^= 1 << (where % 8)
        elif how == "flip_ed": ed[where % len(ed)] ^= 1 << (where % 8)
        elif how == "type": li[10:12] = struct.pack(">H", where % 65536)
        elif how == "leaftype": li[1] = where % 256
        out.append((bytes(li), bytes(ed)))
    good, big = pool[0], F.cert_of_length(70000, serial=D.serial_bytes(8, salt=77)).der
    out += [
        entry(2**64 - 1, good, [CA0.der]),
        (b"\x07" + entry(TS0, pool[1], [CA0.der])[0][1:], entry(TS0, pool[1], [CA0.der])[1]),  # Version is not checked
        (b"\xff" + entry(TS0, pool[2], [CA0.der], precert=True)[0][1:], entry(TS0, pool[2], [CA0.der], precert=True)[1]),
        entry(TS0, pool[3], [CA0.der], ext=b""),
        entry(TS0, pool[4], [CA0.der], ext=bytes(k % 251 for k in range(65535))),
        entry(TS0, pool[5], [CA0.der], precert=True, ext=b"\xee" * 65535),
        entry(TS0, big, [CA0.der]),
        entry(TS0, big, [CA0.der], precert=True),
        entry(TS0, pool[6], [CA0.der, b""]),                  # zero-length certificate at chain position 2
        entry(TS0, pool[7], [CA0.der, b"\x01", b""], precert=True),
        entry(TS0, pool[8], [b""]),                           # ... and at position 1
    ]
    for k in range(1, 6):                                      # chains of 1..5, garbage after Chain[0]
        for precert in (False, True):
            out.append(entry(TS0 + k, pool[9 + k], [CA0.der] + [bytes([k]) * (3 * j + 1) for j in range(k - 1)], precert))
    return out


def test_framing_fuzz(eng, ora):
    entries = framing_corpus()
    pages = raw_pages(entries)
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        r_g, r_o = check(ora, db, odb, pages, what="framing")
    seen = set(r_o.entry_status.tolist())
    assert seen == {0, 2, 3, 4, 5}, seen
    assert {0, 1, 5, 6} <= set(r_o.path.status.tolist())
    assert int(r_g.timestamp_ms[len(entries) - 21]) == 2**64 - 1


# ------------------------------------------------------------------------------------------------ 4. precert TBS shapes

def test_precert_tbs_shapes(eng, ora):
    """Every der_build shape of the walker-geometry corpus, accepted and rejected, as the TBS of a precert entry and as
    its pre_certificate, crossed; plus one trailing byte and one byte short."""
    from test_gpu_walker_geometry import SHAPES, build_shape
    good = [(n, build_shape(i, k, kn).der) for i, (n, bad, kn) in enumerate(SHAPES) if not bad for k in (0, 61)]
    bad = [(n, build_shape(i, k, kn).der) for i, (n, b, kn) in enumerate(SHAPES) if b for k in (0, 61)]
    plain = leaf(424242)
    entries = []
    for t, (_, der) in enumerate(good + bad):
        tbs = fe.tbs_of(der)
        for j, pre in enumerate((plain, der, good[t % len(good)][1], bad[t % len(bad)][1])):
            entries.append(entry(TS0 + 4 * t + j, pre, [CA0.der], precert=True, tbs=tbs))
        entries.append(entry(TS0 + t, plain, [CA0.der], precert=True, tbs=tbs + b"\x00"))
        entries.append(entry(TS0 + t, plain, [CA0.der], precert=True, tbs=tbs[:-1]))
        entries.append(entry(TS0 + t, der, [CA0.der]))  # and as an x509 leaf
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 14) as db:
        r_g, r_o = check(ora, db, odb, raw_pages(entries), what="tbs")
    st = r_o.entry_status
    assert (st == ora.FE_BAD_CERT).any() and (st == 0).any()
    assert (r_o.path.status[st == 0] == ora.ST_PARSE_ERR).any()  # TBS good, pre_certificate bad


# ------------------------------------------------------------------------------------------------ 5. Issuer.ID at block boundaries

ISSUER_KNOBS = [
    {},
    dict(version=1, extensions=None),
    dict(issuer_uid=b"\x01\x02", subject_uid=b"\x03"),
    dict(tbs_sig_alg=D.RSA_PSS, sig_alg=D.RSA_PSS),
    dict(subject=[[D.cn(b"Multi"), D.attr(D.long_oid(50), 0x16, b"x"), D.cn(b"Last", 0x13)]]),
    dict(subject=[[D.cn("BMP CA".encode("utf-16-be"), D.BMP_STRING)]]),
    dict(issuer=[[D.attr(D.long_oid(44), 0x0C, b"far value")], [D.cn(b"Geo CA")]], filler=300),
    dict(extensions=[D.Ext(D.long_oid(22), b"\x30\x00", critical=True), D.basic_constraints(True)]),
    dict(extensions=[D.key_usage(True), D.basic_constraints(True, 3), D.crl_distribution_points(b"http://c.example/crl")]),
]
REJECTED_ISSUER_KNOBS = [
    dict(issuer=[[D.attr(D.long_oid(44), 0x0C, b"value", value_hdr=b"\x0c\x06")], [D.cn(b"Geo CA")]]),
    dict(extensions=[D.Ext(D.long_oid(30), b"\x05\x00", critical=b"\x01\x01\x01")]),
    dict(extensions=[D.Ext(D.long_oid(30), b"\x05\x00", value_tag=0x05)]),
    dict(sig_raw=D.tlv(0x04, b"\x00" + b"\x5a" * 40)),
    dict(sig_raw=D.hdr(0x03, 42) + b"\x00" + b"\x5a" * 40),
]


def block_boundary_cas():
    """Two CAs per SPKI length (another serial, the same key), with the issuer-side knobs in turn, then rejected ones."""
    out = []
    for n in F.SPKI_LENGTHS:
        spki = F.rsa_spki(n)
        for r in range(2):
            out.append(F.ca(10_000 + 2 * n + r, spki, **ISSUER_KNOBS[(n + 5 * r) % len(ISSUER_KNOBS)]).der)
    for k, kn in enumerate(REJECTED_ISSUER_KNOBS):
        out.append(F.ca(20_000 + k, F.rsa_spki(56 + 64 * (k % 2)), **kn).der)
    return out


def check_registered(ora, db, ders, dense):
    by_spki = {}
    for der, d in zip(ders, dense):
        rc, c = ora.parse_cert(der)
        if rc != 0:
            assert d == 0xFFFFFFFE
            continue
        spki = der[c.spki_off:c.spki_off + c.spki_len]
        assert db.issuer_digest(int(d)) == hashlib.sha256(spki).digest() == ora.issuer_id(spki)[0], len(spki)
        by_spki.setdefault(spki, set()).add(int(d))
    assert all(len(v) == 1 for v in by_spki.values())
    assert len({next(iter(v)) for v in by_spki.values()}) == len(by_spki)


def test_issuer_id_at_sha256_block_boundaries(eng, ora):
    cas = block_boundary_cas()
    rejected = [ora.parse_cert(d)[0] != 0 for d in cas]
    assert all(rejected[-len(REJECTED_ISSUER_KNOBS):]) and rejected.count(False) > 150
    with eng.GpuCertDatabase(table_capacity=1 << 12) as db:
        blob, offs = pack(cas)
        dense = db.register_issuers(blob, offs)
        check_registered(ora, db, cas, dense)
    entries = [entry(TS0 + k, leaf(30_000 + k), [der], precert=k % 2 == 1) for k, der in enumerate(cas)]
    entries += [entry(TS0 + k, leaf(40_000 + k), [der, CA0.der]) for k, der in enumerate(cas)]
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 12) as db:
        r_g, r_o = check(ora, db, odb, raw_pages(entries), what="block boundaries")
        n = len(cas)
        check_registered(ora, db, cas, r_g.issuer[:n])
        assert np.array_equal(r_g.issuer[:n], r_g.issuer[n:])
        assert {k: v for k, v in db.issuer_counts().items() if v} == odb.issuer_counts()


# ------------------------------------------------------------------------------------------------ 6. Chain[0] collisions

def chunks_of(ll, xl, cap_entries, cap_text):
    """Pages::fit (ctmr_frontend_api.cu): entries per chunk under the entry budget and half the character budget."""
    out, lo = [], 0
    while lo < ll.size:
        hi, chars = lo, 0
        while hi < ll.size and hi - lo < cap_entries:
            add = int(ll[hi]) + int(xl[hi])
            if chars + add > cap_text // 2:
                break
            chars += add
            hi += 1
        out.append((lo, hi))
        lo = hi
    return out


def pair_entries(pairs, where, salt):
    """Entries whose Chain[0] is a pair member; `where(k)` -> position key.  Each member issues three leaves, and every
    leaf also appears under the other member (same serial, same notAfter): known exactly when the issuers coincide."""
    items = []
    for p, (a, b) in enumerate(pairs):
        for m, der in enumerate((a, b)):
            for t in range(3):
                lf = leaf(salt + 10 * p + t)
                items.append((where(p, m, t), entry(TS0 + 100 * p + 10 * m + t, lf, [der], precert=(p + m + t) % 2 == 1)))
    items.sort(key=lambda x: x[0])
    return [e for _, e in items]


def collision_pairs(salt, length=700):
    return [F.colliding_pair(kind, salt + k, length + 8 * k + k % 3) for k, kind in enumerate(F.PAIR_KINDS)]


def control_of(pairs):
    """Each pair's second member replaced by an uncrafted certificate of the same length (the pre-image of the craft:
    same bytes but the free word), whose hash differs."""
    out = []
    for a, b in pairs:
        c = bytearray(b)
        j = len(b) // 8 - 2
        c[8 * j:8 * j + 8] = bytes(8)
        c = bytes(c)
        if F.chain0_hash(c) == F.chain0_hash(a):  # cannot happen for a 64-bit hash, but the check must not depend on luck
            c = c[:-1] + bytes([c[-1] ^ 1])
        out.append((a, c))
    return out


def launches(db):
    return db.frontend_profile_last()[2]


def expected_cardinalities(ora, db, odb, r_o):
    ok = r_o.path.status == 0
    for h, der in {(int(r_o.path.exp_hour[i]), r_o.issuer_der[i]) for i in np.nonzero(ok)[0]}:
        d = issuer_digest_of(ora, der)
        assert db.get_known_certificates(h, d).count() == odb.set_cardinality(h, d)


def run_collisions(eng, ora, calls, pre_register=(), max_batch_entries=0, **kw):
    """Each call's pages through one ctx (and the oracle); returns the frontend launch count of every call."""
    odb = ora.DB(b"", True)
    counts = []
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 14, max_batch_entries=max_batch_entries, **kw) as db:
        if pre_register:
            db.register_issuers(*pack(list(pre_register)))
        for k, pages in enumerate(calls):
            r_g, r_o = check(ora, db, odb, pages, what=("collision call", k))
            counts.append(launches(db))
            expected_cardinalities(ora, db, odb, r_o)
        assert {k: v for k, v in db.issuer_counts().items() if v} == odb.issuer_counts()
    return counts


def check_pair_outcomes(ora, eng, pairs, pages):
    """Dense indices by kind: different SPKIs differ, the same SPKI shares one, the unparseable member is ISSUER_BAD."""
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 14) as db:
        r = db.store_raw_entries(*pages, NOW_NS)
    text, lo, ll, xo, xl = pages
    r_o = ora.raw_process(ora.DB(b"", True), text, lo, ll, xo, xl, NOW_NS)
    idx = {}
    for i, der in enumerate(r_o.issuer_der):
        if der is not None:
            idx.setdefault(der, set()).add(int(r.issuer[i]))
    assert all(len(v) == 1 for v in idx.values())
    for kind, (a, b) in zip(F.PAIR_KINDS, pairs):
        ia, ib = next(iter(idx[a])), next(iter(idx[b]))
        if kind == F.OTHER_SPKI:
            assert ia != ib and 0xFFFFFFFE not in (ia, ib)
        elif kind == F.SAME_SPKI:
            assert ia == ib != 0xFFFFFFFE
        else:
            assert ia != 0xFFFFFFFE and ib == 0xFFFFFFFE


def test_collisions_inside_one_chunk(eng, ora):
    pairs = collision_pairs(1)
    pages = raw_pages(pair_entries(pairs, lambda p, m, t: (t, p, m), 50_000))
    ctrl = raw_pages(pair_entries(control_of(pairs), lambda p, m, t: (t, p, m), 50_000))
    assert np.array_equal(pages[2], ctrl[2]) and np.array_equal(pages[4], ctrl[4])
    check_pair_outcomes(ora, eng, pairs, pages)
    got, want = run_collisions(eng, ora, [pages]), run_collisions(eng, ora, [ctrl])
    # one chunk holding unseen colliding pairs: the byte compare sends the second member into one more round
    assert got[0] == want[0] + 1, (got, want)
    assert want[0] == FE_LAUNCHES_OUTSIDE_ROUNDS + 2


def test_collisions_across_chunks(eng, ora, monkeypatch):
    """A small character budget: the members of each pair in different chunks of one call.  The second member meets its
    partner in the mirror, fails the byte compare and is registered in its own chunk's first round: no extra round."""
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(1 << 16))
    pairs = collision_pairs(2, length=1200)
    ctrl = control_of(pairs)

    def spread(p, m, t):  # members far apart: each chunk holds ~20 entries
        return (m, t, p)

    fill = [entry(TS0 + k, leaf(60_000 + k), [CA0.der]) for k in range(60)]
    calls, calls_ctrl = [], []
    for ps in (pairs, ctrl):
        e = pair_entries(ps, spread, 70_000)
        (calls if ps is pairs else calls_ctrl).append(raw_pages(e[:9] + fill + e[9:]))
    layout_ = chunks_of(calls[0][2], calls[0][4], 1 << 16, 1 << 16)
    assert len(layout_) >= 3
    pos = {}
    for k, (lo, hi) in enumerate(layout_):
        for i in range(lo, hi):
            pos[i] = k
    assert all(pos[i] != pos[j] for i in range(9) for j in range(69, 78))  # no chunk holds both members of a pair
    got = run_collisions(eng, ora, calls)
    want = run_collisions(eng, ora, calls_ctrl)
    assert got == want, (got, want)


def test_collisions_across_calls_and_after_register_issuers(eng, ora):
    # across calls: first members in call 1, second members in call 2 (each call one chunk)
    pairs2 = collision_pairs(3)
    firsts = raw_pages(pair_entries([(a, a) for a, _ in pairs2], lambda p, m, t: (p, m, t), 80_000))
    seconds = raw_pages(pair_entries([(b, b) for _, b in pairs2], lambda p, m, t: (p, m, t), 80_000))
    seconds_c = raw_pages(pair_entries([(b, b) for _, b in control_of(pairs2)], lambda p, m, t: (p, m, t), 80_000))
    got = run_collisions(eng, ora, [firsts, seconds])
    want = run_collisions(eng, ora, [firsts, seconds_c])
    assert got == want and got[1] == FE_LAUNCHES_OUTSIDE_ROUNDS + 2, (got, want)

    # one member registered through the leaf API first, the other seen by the front end
    got = run_collisions(eng, ora, [seconds], pre_register=[a for a, _ in pairs2])
    want = run_collisions(eng, ora, [seconds_c], pre_register=[a for a, _ in pairs2])
    assert got == want == [FE_LAUNCHES_OUTSIDE_ROUNDS + 2], (got, want)
    # and both members in one call after the first was registered: the second is unseen, the first is not
    both = raw_pages(pair_entries(pairs2, lambda p, m, t: (t, p, m), 80_000))
    both_c = raw_pages(pair_entries(control_of(pairs2), lambda p, m, t: (t, p, m), 80_000))
    got = run_collisions(eng, ora, [both], pre_register=[a for a, _ in pairs2])
    want = run_collisions(eng, ora, [both_c], pre_register=[a for a, _ in pairs2])
    assert got == want, (got, want)


# ------------------------------------------------------------------------------------------------ 7. mirror wrap and capacity

def wrap_corpus():
    """Chain[0] DERs clustered at the top of a 64-slot mirror and of the pending table (hash low 16 bits 0xffff), more
    at 0x0000 / 0x0001 where the wrapped chains land, lengths of every residue mod 8 -- at x509 and precert framings
    with pre_certificates of varying length (Chain[0] at every alignment) -- and chains whose second certificate is a
    blob of >= 65536 bytes, so that the byte after Chain[0] is not zero."""
    ders = F.clustered(10, 0xFFFF, 520, salt=1)
    ders += F.clustered(4, 0x0000, 521, salt=2) + F.clustered(4, 0x0001, 522, salt=3, same_spki=False)
    ders += [F.clustered(1, 0xFFC0 + r, 523 + r, salt=4 + r)[0] for r in range(5)]  # lengths 523..527, mirror slot 0 + r
    assert {len(d) % 8 for d in ders} == set(range(8)) and len(ders) == 23
    big = bytes([0x5A]) * 65536 + b"\x01" * (1 + len(ders))
    entries = []
    for k, der in enumerate(ders):
        for v in range(4):
            lf = leaf(90_000 + 4 * k + v, sig_len=17 + (3 * k + v) % 16)
            chain = [der] if v < 2 else [der, big[:65536 + k]]
            entries.append(entry(TS0 + 4 * k + v, lf, chain, precert=v % 2 == 1))
    return ders, entries


def test_mirror_probe_wrap_and_tail_mask(eng, ora):
    ders, entries = wrap_corpus()
    hs = [F.chain0_hash(d) for d in ders]
    assert sum(h % 64 == 63 for h in hs) == 10 and sum(h & 0xFFFF == 0xFFFF for h in hs) == 10
    pages = raw_pages(entries)
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 14, max_issuers=16) as db:
        check(ora, db, odb, pages, what="wrap")
        assert launches(db) == FE_LAUNCHES_OUTSIDE_ROUNDS + 2
        check(ora, db, odb, pages, what="wrap, all known")  # every Chain[0] now found by probing alone
        assert launches(db) == FE_LAUNCHES_OUTSIDE_ROUNDS + 1
        assert {k: v for k, v in db.issuer_counts().items() if v} == odb.issuer_counts()


def test_mirror_capacity_is_two_ders_per_max_issuer(eng, ora):
    """max_issuers = 16: 64 mirror slots, 32 distinct Chain[0] DERs.  One key, so the registry holds one issuer."""
    ders = F.clustered(33, 0x1234, 600, salt=9)
    es = [entry(TS0 + k, leaf(95_000 + k), [d]) for k, d in enumerate(ders)]
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 12, max_issuers=16) as db:
        with pytest.raises(eng.CtmrError) as e:
            db.store_raw_entries(*raw_pages(es), NOW_NS)
        assert e.value.code == -5
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 12, max_issuers=16) as db:
        dense = db.register_issuers(*pack(ders[:32]))
        assert len(set(dense.tolist())) == 1
        with pytest.raises(eng.CtmrError) as e:
            db.store_raw_entries(*raw_pages(es[32:]), NOW_NS)
        assert e.value.code == -5
        # ... and stays one: the DER that did not fit is not remembered as registered
        with pytest.raises(eng.CtmrError) as e:
            db.store_raw_entries(*raw_pages(es[32:]), NOW_NS)
        assert e.value.code == -5
        with pytest.raises(eng.CtmrError) as e:
            db.register_issuers(*pack(ders[32:]))
        assert e.value.code == -5
        # the batch error left the ctx usable: the 32 registered DERs still resolve
        check(ora, db, odb, raw_pages(es[:32]), what="after the capacity error")
        assert launches(db) == FE_LAUNCHES_OUTSIDE_ROUNDS + 1


# ------------------------------------------------------------------------------------------------ 8. group front end

def test_group_front_end_matches_single_ctx(eng, ora):
    """The framing fuzz and the collision pages through GpuCertGroup([0, 0, 0]) (three shards, three mirrors, one
    registry): identical to one ctx and to the oracle."""
    pairs = collision_pairs(4)
    calls = [raw_pages(framing_corpus(1200, seed=7)),
             raw_pages(pair_entries(pairs, lambda p, m, t: (t, p, m), 110_000)),
             raw_pages(pair_entries(pairs + collision_pairs(5), lambda p, m, t: (m, t, p), 120_000))]
    odb = ora.DB(b"", True)
    single = []
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16, max_batch_entries=64) as db:
        for pages in calls:
            single.append(db.store_raw_entries(*pages, NOW_NS))
    with eng.GpuCertGroup([0, 0, 0], log_expired_entries=True, table_capacity=1 << 16, max_batch_entries=64) as g:
        for k, pages in enumerate(calls):
            r_g, r_o = check(ora, g, odb, pages, what=("group", k))
            same_results(r_g, single[k], ("group vs single", k))
            expected_cardinalities(ora, g, odb, r_o)
        assert {k: v for k, v in g.issuer_counts().items() if v} == odb.issuer_counts()
