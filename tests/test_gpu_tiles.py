"""static-ct-api data tiles on the GPU (ctmr_process_tiles, include/ctmr_frontend.h) against the test oracle
(tests/tiles_oracle.py: the tile rules, then the get-entries oracle on the equivalent entries): bit-exact on every
output.  Marked gpu."""
import hashlib
import struct

import numpy as np
import pytest

import tiles_oracle as to
from conftest import NOW_NS, README_FILTER

pytestmark = pytest.mark.gpu

TS0 = 1_690_000_000_000
PATH_FIELDS = ("status", "exp_hour", "serial_off", "serial_len", "was_unknown", "first_issuer_hour")
META_FIELDS = ("issuer_name_off", "issuer_name_len", "crldp_off", "crldp_len", "first_issuer_dn", "first_crldp")


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


class Corpus:
    """Synthetic tiles: x509 and precert entries, chains of 0-3 fingerprints, duplicates, an unparseable Chain[0]."""

    def __init__(self, ora, widths, seed=7, first_tile=0, tile_numbers=None, **cfg_kw):
        from ct_mapreduce_b200 import frontend as fe
        n = sum(widths)
        cfg = ora.synth_cfg(n, dup_mode=1, **cfg_kw)
        blob, offs, idx = ora.synth_corpus(cfg, 0, n)
        iblob, ioffs = ora.synth_issuers(cfg)
        self.issuers = [iblob[int(ioffs[k]):int(ioffs[k + 1])].tobytes() for k in range(ioffs.size - 1)]
        bad = bytearray(self.issuers[0]); bad[6] ^= 0xFF
        self.bad_issuer = bytes(bad)
        self.certs = self.issuers + [self.bad_issuer]
        self.fp = [hashlib.sha256(d).digest() for d in self.certs]
        self.by_fp = dict(zip(self.fp, self.certs))
        rng = np.random.default_rng(seed)
        kinds = rng.integers(0, 1000, n)
        self.leaves, self.tile_leaves = [], []
        self.index = list(tile_numbers) if tile_numbers is not None else list(range(first_tile, first_tile + len(widths)))
        i = 0
        for t, w in enumerate(widths):
            tl = []
            for j in range(w):
                leaf, k, kind = blob[int(offs[i]):int(offs[i + 1])].tobytes(), int(idx[i]), int(kinds[i])
                first = len(self.certs) - 1 if kind % 53 == 7 else k
                chain = [self.fp[first]] + [self.fp[(k + m) % len(self.issuers)] for m in range(1, kind % 3 + 1)]
                chain = chain[:kind % 4]
                ext = fe.leaf_index_extension(256 * self.index[t] + j) + (b"\x05\x00\x02ab" if kind % 7 == 0 else b"")
                if kind % 3 == 0:
                    tl.append(fe.tile_leaf_precert(TS0 + i, self.fp[k], fe.tbs_of(leaf), leaf, chain, ext))
                else:
                    tl.append(fe.tile_leaf_x509(TS0 + i, leaf, chain, ext))
                self.leaves.append(leaf)
                i += 1
            self.tile_leaves.append(tl)
        self.widths = list(widths)
        self.pack()

    def pack(self, tiles=None, gap=b"\x00" * 5):
        """tiles (bytes) back to back with a few bytes between them, as an HTTP client might leave them"""
        tiles = tiles if tiles is not None else [b"".join(t) for t in self.tile_leaves]
        data, off, ln = bytearray(), [], []
        for t in tiles:
            data += gap
            off.append(len(data)); ln.append(len(t))
            data += t
        self.data = bytes(data)
        self.off, self.len = np.array(off, np.uint64), np.array(ln, np.uint32)
        self.tile_index, self.width = np.array(self.index, np.uint64), np.array(self.widths, np.uint16)

    def args(self, sl=slice(None)):
        return self.data, self.off[sl], self.len[sl], self.tile_index[sl], self.width[sl]

    def register(self, db, certs=None):
        from conftest import pack
        return db.register_chain_certs(*pack(self.certs if certs is None else certs))


def compare(ora, db, r_g, r_o, n=None, want_meta=False, want_pem=False):
    n = r_o.n_done if n is None else n
    for f in ("entry_status", "entry_type", "timestamp_ms", "leaf_index", "leaf_off", "leaf_len"):
        a, b = getattr(r_g, f)[:n], getattr(r_o, f)[:n]
        bad = np.nonzero(a != b)[0]
        assert bad.size == 0, (f, bad[:10], a[bad[:10]], b[bad[:10]])
    if r_g.leaf_hash is not None:
        assert np.array_equal(r_g.leaf_hash[:n], r_o.leaf_hash[:n])
    assert np.array_equal(r_g.tile_status[:r_o.tiles_done], r_o.tile_status[:r_o.tiles_done])
    for f in PATH_FIELDS + (META_FIELDS if want_meta else ()):
        a, b = getattr(r_g.path, f)[:n], getattr(r_o.path, f)[:n]
        if f in ("exp_hour", "serial_off", "serial_len") + META_FIELDS[:4]:
            m = r_o.path.status[:n] != 1
            a, b = a[m], b[m]
        bad = np.nonzero(a != b)[0]
        assert bad.size == 0, (f, bad[:10], a[bad[:10]], b[bad[:10]])
    assert np.array_equal(r_g.path.sha256[:n], r_o.path.sha256[:n])
    memo = {}
    for i in range(n):   # Chain[0] -> Issuer.ID for every entry whose fingerprint was looked up
        fp = r_o.chain0_fp[i]
        if fp is None:
            assert r_g.issuer[i] == 0xFFFFFFFF, i
            continue
        if fp not in memo:
            rc, c = ora.parse_cert(db_certs[fp])
            memo[fp] = None if rc else ora.issuer_id(db_certs[fp][c.spki_off:c.spki_off + c.spki_len])[0]
        if memo[fp] is None:
            assert r_g.issuer[i] == 0xFFFFFFFE, i
        else:
            assert db.issuer_digest(int(r_g.issuer[i])) == memo[fp], i
    if want_pem:
        from conftest import go_pem
        for i in range(n):
            assert r_g.path.pem_of(i) == (go_pem(r_o.leaves[i]) if r_o.path.was_unknown[i] else b""), i


db_certs = {}


def run_both(ora, db, odb, cp, sl=slice(None), known=None, **kw):
    db_certs.update(cp.by_fp)
    r_o = to.tiles_process(ora, odb, *cp.args(sl), cp.by_fp, NOW_NS, known=known)
    r_g = db.store_tiles(*cp.args(sl), NOW_NS, **kw)
    assert r_g.tiles_done == r_o.tiles_done and r_g.missing == r_o.missing
    compare(ora, db, r_g, r_o, want_meta=kw.get("want_meta", False), want_pem=kw.get("want_pem", False))
    return r_g, r_o


def test_mixed_corpus_bit_exact(eng, ora):
    cp = Corpus(ora, [256] * 11 + [100], first_tile=40)
    odb = ora.DB(README_FILTER, False)
    with eng.GpuCertDatabase(issuer_cn_filter=README_FILTER, table_capacity=1 << 16) as db:
        cp.register(db)
        r_g, r_o = run_both(ora, db, odb, cp, want_meta=True, want_pem=True, want_leaf_hash=True)
        assert r_g.tiles_done == 12 and not r_g.missing
        assert set(r_o.entry_status.tolist()) <= {0, 5} and set(r_o.path.status.tolist()) >= {0, 5, 6}
        assert {k: v for k, v in db.issuer_counts().items() if v} == odb.issuer_counts()
        assert np.array_equal(db.status_counters(), odb.filter_counters())
        fe_ms, path_ms, launches = db.frontend_profile_last()
        assert fe_ms > 0 and path_ms > 0 and launches >= 6


def test_pages_and_tiles_give_the_same_result(eng, ora):
    from ct_mapreduce_b200 import frontend as fe
    cp = Corpus(ora, [256] * 6 + [77], seed=3)
    entries = []
    for t in range(len(cp.widths)):
        entries += fe.tile_to_get_entries(b"".join(cp.tile_leaves[t]), cp.by_fp, width=cp.widths[t])
    body = fe.get_entries_body(entries)
    lo, ll, xo, xl = fe.find_entry_spans(body)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as d1, \
            eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as d2:
        r1 = d1.store_raw_entries(body, lo, ll, xo, xl, NOW_NS)
        cp.register(d2)
        r2 = d2.store_tiles(*cp.args(), NOW_NS)
        for f in PATH_FIELDS + ("sha256",):
            assert np.array_equal(getattr(r1.path, f), getattr(r2.path, f)), f
        for f in ("entry_status", "entry_type", "timestamp_ms", "leaf_len"):
            assert np.array_equal(getattr(r1, f), getattr(r2, f)), f
        c1 = {k: v for k, v in d1.issuer_counts().items() if v}
        assert c1 == {k: v for k, v in d2.issuer_counts().items() if v} and c1
        assert np.array_equal(d1.status_counters(), d2.status_counters())
        for i in np.nonzero(r1.path.status == 0)[0][:50]:
            dig = d1.issuer_digest(int(r1.issuer[i]))
            assert d2.issuer_digest(int(r2.issuer[i])) == dig
            h = int(r1.path.exp_hour[i])
            assert d1.get_known_certificates(h, dig).count() == d2.get_known_certificates(h, dig).count() > 0


def malformed(cp, t, how):
    """tile t of the corpus with one tile-level malformation"""
    tl = list(cp.tile_leaves[t])
    j = 5
    b = bytearray(tl[j])
    ts_type = struct.unpack(">H", b[8:10])[0]
    if how == "truncated":
        return b"".join(tl)[:-3]
    if how == "trailing":
        return b"".join(tl) + b"\x00"
    if how == "bad_type":
        b[8:10] = b"\x00\x02"
    elif how == "chain_not_32":   # one more byte of chain, and a chain length that is not a multiple of 32
        c = _chain_len(tl[j])
        pos = len(b) - 2 - c
        b[pos:pos + 2] = struct.pack(">H", c + 1)
        b += b"\x00"
    elif how == "zero_cert":
        b[10 + 32 * ts_type:13 + 32 * ts_type] = b"\x00\x00\x00"
    elif how == "past_end":
        b[10 + 32 * ts_type:13 + 32 * ts_type] = b"\x7f\xff\xff"
    tl[j] = bytes(b)
    return b"".join(tl)


def _chain_len(leaf):
    from ct_mapreduce_b200 import frontend as fe
    return 32 * len(fe.split_tile(leaf, 1)[0][3])


@pytest.mark.parametrize("how", ["truncated", "trailing", "width_high", "width_low", "bad_type", "chain_not_32", "zero_cert", "past_end"])
def test_tile_malformations(eng, ora, how):
    cp = Corpus(ora, [256] * 5, seed=13)
    tiles = [b"".join(t) for t in cp.tile_leaves]
    if how == "width_high":
        tiles[2] = b"".join(cp.tile_leaves[2][:200]); cp.widths[2] = 201
    elif how == "width_low":
        cp.widths[2] = 255
    else:
        tiles[2] = malformed(cp, 2, how)
    cp.pack(tiles)
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        cp.register(db)
        r_g, r_o = run_both(ora, db, odb, cp, want_leaf_hash=True)
        assert r_g.tile_status.tolist() == [0, 0, 6, 0, 0]
        e2 = slice(512, 512 + int(cp.widths[2]))
        assert set(r_g.entry_status[e2].tolist()) == {6} and set(r_g.path.status[e2].tolist()) == {1}
        assert not r_g.leaf_hash[e2].any() and (r_g.issuer[e2] == 0xFFFFFFFF).all()
        assert set(r_g.entry_status[:512].tolist()) == {0} and set(r_g.entry_status[e2.stop:].tolist()) == {0}
        # the tiles after the bad one went through: the same tiles again are all known
        r2 = db.store_tiles(*cp.args(slice(3, 5)), NOW_NS)
        assert not r2.path.was_unknown.any()


@pytest.mark.parametrize("how", ["missing", "duplicated", "wrong_length", "off_by_one", "extra_extensions"])
def test_leaf_index_cases(eng, ora, how):
    from ct_mapreduce_b200 import frontend as fe
    cp = Corpus(ora, [256] * 3, seed=17, first_tile=9)
    j = 40
    i = 256 * 1 + j
    leaf, k = cp.leaves[i], 1
    ext = {"missing": b"", "duplicated": fe.leaf_index_extension(256 * 10 + j) * 2,
           "wrong_length": b"\x00\x00\x04" + (256 * 10 + j).to_bytes(4, "big"),
           "off_by_one": fe.leaf_index_extension(256 * 10 + j + 1),
           "extra_extensions": b"\x01\x00\x00" + fe.leaf_index_extension(256 * 10 + j) + b"\xff\x00\x03abc"}[how]
    cp.tile_leaves[1][j] = fe.tile_leaf_x509(TS0 + i, leaf, [cp.fp[k]], ext)
    cp.pack()
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        cp.register(db)
        r_g, r_o = run_both(ora, db, odb, cp)
        want = 0 if how == "extra_extensions" else 7
        assert r_g.entry_status[i] == want and r_g.tile_status.tolist() == [0, 0, 0]
        assert (r_g.path.status[i] == 1) == (want == 7)


def ready_slots(db):
    """The known-certificate table as a sorted list of (lowest entry index, exp_hour, Issuer.ID digest, serial): slot
    positions and dense issuer indices depend on registration order, the entry indices must not"""
    from keymodel import decode_snapshot
    table, _ = decode_snapshot(db.snapshot())
    raw = table.view(np.uint8).reshape(-1, 64)
    out = []
    for x in raw[raw[:, 8:16].any(axis=1)]:
        first = ~int.from_bytes(x[0:8].tobytes(), "little") & (2**64 - 1)
        out.append((first, x[16:20].tobytes(), db.issuer_digest(int.from_bytes(x[20:24].tobytes(), "little")), x[24:64].tobytes()))
    return sorted(out)


def test_missing_issuers_stop_and_resume(eng, ora):
    cp = Corpus(ora, [256] * 8 + [31], seed=19)
    # issuers first met in tile 3: everything the first three tiles need is registered, nothing more
    need = set()
    r_all = to.tiles_process(ora, ora.DB(b"", True), *cp.args(), cp.by_fp, NOW_NS)
    for i in range(768):
        if r_all.chain0_fp[i] is not None:
            need.add(r_all.chain0_fp[i])
    first = [cp.by_fp[f] for f in need]
    later = [d for d in cp.certs if hashlib.sha256(d).digest() not in need]
    assert later
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db, \
            eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as one:
        cp.register(db, first)
        r_g, r_o = run_both(ora, db, odb, cp, known=need, want_leaf_hash=True)
        assert r_g.tiles_done == r_o.tiles_done >= 3 and r_g.tiles_done < 9 and r_g.missing
        # no entry of the stop tile or later reached the tables
        assert np.array_equal(db.status_counters(), odb.filter_counters())
        assert {k: v for k, v in db.issuer_counts().items() if v} == odb.issuer_counts()
        # resume: fetch + register + call again from tiles_done, until done; equals one call with everything registered
        fetched = []

        def fetch(fps):
            fetched.append(list(fps))
            return [cp.by_fp[f] for f in fps]
        cp.register(one)
        r_one = one.store_tiles(*cp.args(), NOW_NS, want_pem=True, want_leaf_hash=True)
        one_counts = {k: v for k, v in one.issuer_counts().items() if v}
        one_slots = ready_slots(one)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db2:
        cp.register(db2, first)
        r_res = db2.store_tiles(*cp.args(), NOW_NS, want_pem=True, want_leaf_hash=True, fetch=fetch)
        assert r_res.tiles_done == 9 and len(fetched) >= 1 and fetched[0] == r_g.missing
        for f in PATH_FIELDS + ("sha256",):
            assert np.array_equal(getattr(r_res.path, f), getattr(r_one.path, f)), f
        for f in ("entry_status", "timestamp_ms", "leaf_index", "leaf_off", "leaf_len", "leaf_hash", "tile_status", "pem", "pem_off"):
            a, b = getattr(r_res, f, None), getattr(r_one, f, None)
            if a is None:
                a, b = getattr(r_res.path, f), getattr(r_one.path, f)
            assert np.array_equal(a, b), f
        assert {k: v for k, v in db2.issuer_counts().items() if v} == one_counts
        assert ready_slots(db2) == one_slots


def test_unparseable_chain0(eng, ora):
    cp = Corpus(ora, [256] * 4, seed=23)
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        dense, fps = cp.register(db)
        assert dense[-1] == 0xFFFFFFFE and fps.tobytes() == b"".join(cp.fp)
        r_g, r_o = run_both(ora, db, odb, cp)
        assert (r_g.path.status == ora.ST_ISSUER_PARSE_ERR).any()


def test_chunk_boundaries_and_oversized_tile(eng, ora, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(3 << 20))   # 1.5 MB of tiles per chunk: several chunks per call
    cp = Corpus(ora, [256] * 12 + [9], seed=29)
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16, max_batch_entries=700) as db:
        cp.register(db)
        for sl in (slice(0, 1), slice(1, 6), slice(6, 13)):
            run_both(ora, db, odb, cp, sl, want_pem=True, want_leaf_hash=True)
        # tiles scattered over the buffer (packed on the host)
        cp2 = Corpus(ora, [256] * 4, seed=31, tile_numbers=[5, 6, 7, 8])
        cp2.pack([b"".join(t) for t in cp2.tile_leaves], gap=b"\x00" * 2_500_000)
        with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16, max_batch_entries=600) as db2:
            cp2.register(db2)
            run_both(ora, db2, ora.DB(b"", True), cp2, want_leaf_hash=True)
    big = Corpus(ora, [256] * 2, seed=37, len_mode=1, len_lo=6000, len_hi=6500)   # ~1.6 MB per tile
    with eng.GpuCertDatabase(table_capacity=1 << 14) as db:
        big.register(db)
        from ct_mapreduce_b200 import capi
        with pytest.raises(capi.CtmrError) as ei:
            db.store_tiles(*big.args(), NOW_NS)
        assert ei.value.code == capi.E_BATCH_TOO_LARGE


def test_invalid_batches(eng, ora):
    from ct_mapreduce_b200 import capi
    cp = Corpus(ora, [256, 10], seed=41)
    with eng.GpuCertDatabase(table_capacity=1 << 14) as db:
        for w in (0, 257):
            with pytest.raises(capi.CtmrError) as ei:
                db.store_tiles(cp.data, cp.off, cp.len, cp.tile_index, np.array([w, 10], np.uint16), NOW_NS)
            assert ei.value.code == capi.E_INVALID
        with pytest.raises(capi.CtmrError) as ei:
            db.store_tiles(cp.data[:-1], cp.off, cp.len, cp.tile_index, cp.width, NOW_NS)
        assert ei.value.code == capi.E_INVALID


def test_mixing_entry_points_and_restore(eng, ora):
    from ct_mapreduce_b200 import frontend as fe
    cp = Corpus(ora, [256] * 6, seed=43)
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        dense, _ = cp.register(db)
        run_both(ora, db, odb, cp, slice(0, 2))
        # the same certificates through the leaf API and as get-entries pages: all known, indices continue
        blob = np.frombuffer(b"".join(cp.leaves[:100]), np.uint8)
        offs = np.zeros(101, np.uint64); offs[1:] = np.cumsum([len(x) for x in cp.leaves[:100]])
        r1 = db.store_batch(blob, offs, None, None, None, NOW_NS)
        ent = fe.tile_to_get_entries(b"".join(cp.tile_leaves[2]), cp.by_fp)
        body = fe.get_entries_body(ent)
        r2 = db.store_raw_entries(body, *fe.find_entry_spans(body), NOW_NS)
        r3 = db.store_tiles(*cp.args(slice(2, 3)), NOW_NS)
        assert not r3.path.was_unknown.any() and np.array_equal(r2.path.status, r3.path.status)
        snap = db.snapshot()
        r4 = db.store_tiles(*cp.args(slice(3, 6)), NOW_NS)
        db.restore(snap)
        r5 = db.store_tiles(*cp.args(slice(3, 6)), NOW_NS)
        assert r5.tiles_done == 0 and r5.missing             # the fingerprint table went with the restore
        dense2, _ = cp.register(db)
        assert np.array_equal(dense, dense2)                  # same dense indices again
        r6 = db.store_tiles(*cp.args(slice(3, 6)), NOW_NS)
        for f in PATH_FIELDS:
            assert np.array_equal(getattr(r4.path, f), getattr(r6.path, f)), f
        del r1


def _group_case(eng, ora, devices, want_pem=True):
    cp = Corpus(ora, [256] * 9 + [50], seed=47)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        cp.register(db)
        want = db.store_tiles(*cp.args(), NOW_NS, want_pem=True, want_leaf_hash=True)
        wc = {k: v for k, v in db.issuer_counts().items() if v}
    with eng.GpuCertGroup(devices, log_expired_entries=True, table_capacity=1 << 15, max_batch_entries=600) as g:
        # first only some issuers: the stop lands inside a member's window and the resume completes it
        some = cp.certs[: len(cp.certs) // 2]
        cp.register(g, some)
        got = g.store_tiles(*cp.args(), NOW_NS, want_pem=want_pem, want_leaf_hash=True,
                            fetch=lambda fps: [cp.by_fp[f] for f in fps])
        assert got.tiles_done == 10
        for f in PATH_FIELDS + ("sha256",) + (("pem", "pem_off") if want_pem else ()):
            assert np.array_equal(getattr(got.path, f), getattr(want.path, f)), f
        for f in ("entry_status", "leaf_hash", "leaf_off", "tile_status"):
            assert np.array_equal(getattr(got, f), getattr(want, f)), f
        assert {k: v for k, v in g.issuer_counts().items() if v} == wc


def test_group_of_three_shards_on_one_gpu(eng, ora):
    _group_case(eng, ora, [0, 0, 0])


def test_group_of_three_shards_without_pem(eng, ora):
    """without PEM the members' back halves run on one thread each"""
    _group_case(eng, ora, [0, 0, 0], want_pem=False)


def _one_ctx_and_group_of_one(eng, calls):
    """calls(db) -> results, on one ctx and on GpuCertGroup([0]); returns both, each with the known-certificate table"""
    out = []
    for make in (eng.GpuCertDatabase, lambda **kw: eng.GpuCertGroup([0], **kw)):
        with make(log_expired_entries=True, table_capacity=1 << 16) as db:
            out.append((calls(db), ready_slots(getattr(db, "members", [db])[0])))
    return out


def _same_calls(a, b, fields):
    for k, (x, y) in enumerate(zip(a, b)):
        for f in PATH_FIELDS + ("sha256", "pem", "pem_off"):
            assert np.array_equal(getattr(x.path, f), getattr(y.path, f)), (k, f)
        for f in fields:
            assert np.array_equal(getattr(x, f), getattr(y, f)), (k, f)


def test_group_of_one_pages(eng, ora):
    """A group of one runs get-entries pages as one ctx does.  Two calls, the second holding new pages and then the
    first call's again: every output and the table slot by slot (lowest entry index included) are one ctx's, and the
    second call finds the first call's certificates known."""
    from ct_mapreduce_b200 import frontend as fe
    cp = Corpus(ora, [256] * 6, seed=61)
    ents = [fe.tile_to_get_entries(b"".join(t), cp.by_fp) for t in cp.tile_leaves]
    bodies = [fe.get_entries_body(sum(ents[:3], [])), fe.get_entries_body(sum(ents[3:] + ents[:3], []))]

    def calls(db):
        rs = [db.store_raw_entries(body, *fe.find_entry_spans(body), NOW_NS, want_pem=True) for body in bodies]
        assert rs[0].path.was_unknown.any() and not rs[1].path.was_unknown[768:].any()
        for r in rs:  # dense indices follow the order in which the GPU meets new issuers: their digests are compared
            r.issuer = [db.issuer_digest(int(i)) if i < 0xFFFFFFFE else int(i) for i in r.issuer]
        return rs
    (one, one_slots), (grp, grp_slots) = _one_ctx_and_group_of_one(eng, calls)
    _same_calls(one, grp, ("entry_status", "entry_type", "timestamp_ms", "leaf_src", "leaf_off", "leaf_len"))
    assert [r.issuer for r in one] == [r.issuer for r in grp]
    assert one_slots == grp_slots


def test_group_of_one_tiles_stop_and_resume(eng, ora):
    """A group of one runs tiles as one ctx does.  A call that stops at an unregistered Chain[0], the call that resumes
    from tiles_done after the registration, and the first call's tiles again: every output and the table slot by slot
    are one ctx's, and the later calls find the first call's certificates known."""
    cp = Corpus(ora, [256] * 8 + [31], seed=19)
    r_all = to.tiles_process(ora, ora.DB(b"", True), *cp.args(), cp.by_fp, NOW_NS)
    first = [cp.by_fp[f] for f in {r_all.chain0_fp[i] for i in range(768)} - {None}]

    def calls(db):
        cp.register(db, first)
        r1 = db.store_tiles(*cp.args(), NOW_NS, want_pem=True, want_leaf_hash=True)
        k = r1.tiles_done
        assert 3 <= k < 9 and r1.missing
        cp.register(db)
        r2 = db.store_tiles(*cp.args(slice(k, None)), NOW_NS, want_pem=True, want_leaf_hash=True)
        r3 = db.store_tiles(*cp.args(slice(0, k)), NOW_NS, want_pem=True, want_leaf_hash=True)
        assert r2.tiles_done == 9 - k and r3.tiles_done == k and not r3.path.was_unknown.any()
        return r1, r2, r3
    (one, one_slots), (grp, grp_slots) = _one_ctx_and_group_of_one(eng, calls)
    assert [r.missing for r in one] == [r.missing for r in grp]
    _same_calls(one, grp, ("entry_status", "entry_type", "timestamp_ms", "issuer", "leaf_index", "leaf_off", "leaf_len",
                           "leaf_hash", "tile_status"))
    assert one_slots == grp_slots


def test_group_all_gpus(eng, ora):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs several GPUs")
    _group_case(eng, ora, list(range(n)))


def test_fingerprints_that_differ_from_a_registered_one_in_one_byte(eng, ora):
    """Chain[0] fingerprints equal to a registered fingerprint in bytes 0..30, and in bytes 0..7 (the probe hash), are
    not that certificate: each stops the call at its tile and is listed as missing."""
    from ct_mapreduce_b200 import capi, frontend as fe
    cp = Corpus(ora, [256] * 4, seed=53)
    near = []
    for t, byte in ((1, 31), (2, 8)):
        j = 17
        i = 256 * t + j
        fp = bytearray(cp.fp[3]); fp[byte] ^= 0x01
        near.append(bytes(fp))
        cp.tile_leaves[t][j] = fe.tile_leaf_x509(TS0 + i, cp.leaves[i], [bytes(fp), cp.fp[4]], fe.leaf_index_extension(256 * t + j))
    cp.pack()
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        cp.register(db)
        r_g, r_o = run_both(ora, db, odb, cp)
        assert r_g.tiles_done == 1 and r_g.missing == [near[0]]
        r_g, r_o = run_both(ora, db, odb, cp, slice(2, 4))
        assert r_g.tiles_done == 0 and r_g.missing == [near[1]]
        r_g, r_o = run_both(ora, db, odb, cp, slice(3, 4))
        assert r_g.tiles_done == 1 and not r_g.missing
        # a fetch that returns a certificate whose SHA-256 is not the fingerprint asked for is an error, not a loop
        with pytest.raises(capi.CtmrError) as ei:
            db.store_tiles(*cp.args(slice(1, 2)), NOW_NS, fetch=lambda fps: [cp.certs[3] for _ in fps])
        assert ei.value.code == capi.E_UNKNOWN_ISSUER


def test_split_is_timed_on_its_own(eng, ora):
    cp = Corpus(ora, [256] * 3, seed=59)
    with eng.GpuCertDatabase(table_capacity=1 << 14) as db:
        cp.register(db)
        db.store_tiles(*cp.args(), NOW_NS)
        fe_ms, _, _ = db.frontend_profile_last()
        assert 0 < db.tiles_profile_last() <= fe_ms
