"""The log's Merkle tree folded on the GPU (ctmr_process_raw_tree, ctmr_process_tiles_tree) against the hashlib model
(tests/merkle_model.py).  Every case also runs the same batch through the plain call on a twin ctx and requires every
other output to be bit-identical, PEM included: the tree changes nothing else.  Marked gpu."""
import base64
import ctypes as C
import hashlib

import numpy as np
import pytest

import merkle_model as mm
from conftest import NOW_NS

pytestmark = pytest.mark.gpu

RAW_FIELDS = ("entry_status", "entry_type", "timestamp_ms", "issuer", "leaf_src", "leaf_off", "leaf_len")
TILE_FIELDS = ("entry_status", "entry_type", "timestamp_ms", "issuer", "leaf_index", "leaf_off", "leaf_len", "tile_status")
PATH_FIELDS = ("status", "sha256", "exp_hour", "serial_off", "serial_len", "was_unknown", "first_issuer_hour", "issuer_name_off",
               "issuer_name_len", "crldp_off", "crldp_len", "first_issuer_dn", "first_crldp", "pem", "pem_off")


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def new_db(eng, **kw):
    kw.setdefault("table_capacity", 1 << 20)
    return eng.GpuCertDatabase(log_expired_entries=True, **kw)


def issuer_ids(db, idx):
    """dense issuer indices -> Issuer.ID digests: the order in which a ctx meets new issuers is not fixed, so two ctxs
    may number the same issuers differently"""
    memo = {}
    return [int(i) if int(i) >= 0xFFFFFFFE else memo.setdefault(int(i), db.issuer_digest(int(i))) for i in idx]


def same(a, b, fields, db, twin):
    for f in fields:
        x, y = getattr(a, f), getattr(b, f)
        if f == "issuer":
            assert issuer_ids(db, x) == issuer_ids(twin, y), f
            continue
        assert (x is None) == (y is None) and (x is None or np.array_equal(x, y)), f
    for f in PATH_FIELDS:
        x, y = getattr(a.path, f), getattr(b.path, f)
        assert (x is None) == (y is None) and (x is None or np.array_equal(x, y)), f


# ---------------------------------------------------------------------------------------------------------------- pages
class Pages:
    """get-entries pages from libctmr's host generator; leaf_input strings can be replaced (appended to the text)"""

    def __init__(self, n):
        from ct_mapreduce_b200 import capi
        cfg = capi.synth_cfg(n)
        L = capi.load()
        need = L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, 1000, None, 0, None, None, None, None)
        self.text = np.zeros(need, np.uint8)
        self.lo, self.ll = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
        self.xo, self.xl = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
        assert L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, 1000, capi.ptr(self.text), need, capi.ptr(self.lo), capi.ptr(self.ll),
                                           capi.ptr(self.xo), capi.ptr(self.xl)) == need
        self.extra = bytearray()

    def leaf(self, i):
        a = int(self.lo[i])
        return base64.b64decode(self.text[a:a + int(self.ll[i])].tobytes(), validate=True)

    def hashes(self, lo, hi):
        return [mm.leaf_hash(self.leaf(i)) for i in range(lo, hi)]

    def replace(self, i, b64: bytes):
        self.lo[i], self.ll[i] = self.text.size + len(self.extra), len(b64)
        self.extra += b64

    def args(self, lo, hi):
        text = np.concatenate([self.text, np.frombuffer(bytes(self.extra), np.uint8)]) if self.extra else self.text
        return text, self.lo[lo:hi], self.ll[lo:hi], self.xo[lo:hi], self.xl[lo:hi]


@pytest.fixture(scope="module")
def pages():
    return Pages(4099)


@pytest.fixture(scope="module")
def pair(eng):
    db, twin = new_db(eng), new_db(eng)
    yield db, twin
    db.close()
    twin.close()


def random_tree(eng, size, rng):
    """a tree of `size` leaves whose edge rows are random (the fold does not care what they hold); clear rows junk too"""
    edge = np.frombuffer(rng.bytes(64 * 32), np.uint8).reshape(64, 32).copy()
    return eng.LogTree(size, edge), {k: edge[k].tobytes() for k in range(64) if (size >> k) & 1}


def expect(tree, e, size, hashes):
    e2, s2 = mm.extend(e, size, hashes)
    assert tree.size == s2
    assert tree.edge.tobytes() == mm.edge_rows(e2, s2)
    assert tree.root == mm.root(e2, s2)
    return e2, s2


def raw_both(db, twin, args, tree):
    r = db.store_raw_entries(*args, NOW_NS, want_meta=True, want_pem=True, tree=tree)
    p = twin.store_raw_entries(*args, NOW_NS, want_meta=True, want_pem=True)
    same(r, p, RAW_FIELDS, db, twin)
    assert p.tree is None
    return r


@pytest.mark.parametrize("start", [0, 1, 255, 256, 257, 2**32 - 1, 2**40 + 12345, 2**63 - 5])
def test_pages_from_any_start(eng, pages, pair, start):
    rng = np.random.default_rng(start % 1000003)
    for n in (1, 2, 3, 255, 256, 257, 1000, 4099):
        tree, e = random_tree(eng, start, rng)
        r = raw_both(*pair, pages.args(0, n), tree)
        expect(r.tree, e, start, pages.hashes(0, n))


def test_pages_empty_batch_gives_the_root(eng, pair):
    db, _ = pair
    z = np.zeros(0, np.uint64), np.zeros(0, np.uint32)
    r = db.store_raw_entries(b"x", z[0], z[1], z[0], z[1], NOW_NS, tree=eng.LogTree())
    assert r.tree.size == 0 and r.tree.root == hashlib.sha256(b"").digest() and not r.tree.edge.any()
    hashes = [mm.leaf_hash(bytes([i])) for i in range(11)]
    e = mm.edge(hashes, 11)
    t = eng.LogTree(11, np.frombuffer(mm.edge_rows(e, 11), np.uint8).reshape(64, 32).copy())
    assert db.store_raw_entries(b"x", z[0], z[1], z[0], z[1], NOW_NS, tree=t).tree.root == mm.mth_hashes(hashes)


def test_pages_several_chunks_per_call(eng, pages, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(1 << 16))   # ~8 entries per chunk
    rng = np.random.default_rng(5)
    with new_db(eng, max_batch_entries=600) as db, new_db(eng, max_batch_entries=600) as twin:
        for start, lo, hi in ((12345, 0, 300), (12645, 300, 1301)):
            tree, e = random_tree(eng, start, rng)
            r = raw_both(db, twin, pages.args(lo, hi), tree)
            expect(r.tree, e, start, pages.hashes(lo, hi))


@pytest.mark.parametrize("k", [0, 1, 150, 299])
def test_pages_fold_stops_before_bad_base64(eng, pair, k):
    from ct_mapreduce_b200 import capi
    pg = Pages(300)
    j = 20  # a leaf_input that is base64 but not a MerkleTreeLeaf: BAD_LEAF, and it still folds
    junk = b"\x07not a MerkleTreeLeaf"
    pg.replace(j, base64.b64encode(junk))
    pg.replace(k, base64.b64encode(pg.leaf(k))[:-4] + b"!AAA")
    rng = np.random.default_rng(k)
    tree, e = random_tree(eng, 1001, rng)
    r = raw_both(*pair, pg.args(0, 300), tree)
    assert r.entry_status[k] == capi.FE_BAD_BASE64
    if k != j:
        assert r.entry_status[j] == capi.FE_BAD_LEAF
    hashes = [mm.leaf_hash(junk) if i == j else mm.leaf_hash(pg.leaf(i)) for i in range(k)]
    expect(r.tree, e, 1001, hashes)
    assert r.tree.size == 1001 + k


def test_pages_three_calls_carry_the_tree(eng, pages, pair):
    cuts = (0, 333, 700, 1000)
    leaves = [pages.leaf(i) for i in range(1000)]

    def run(pg):
        tree = eng.LogTree()
        for a, b in zip(cuts, cuts[1:]):
            tree = raw_both(*pair, pg.args(a, b), tree).tree
            assert tree.size == b
        return tree.root

    assert run(pages) == mm.mth(leaves)
    changed = Pages(1000)
    leaf = bytearray(changed.leaf(500))
    leaf[len(leaf) // 2] ^= 0x20
    changed.replace(500, base64.b64encode(bytes(leaf)))
    leaves[500] = bytes(leaf)
    got = run(changed)
    assert got != mm.mth([pages.leaf(i) for i in range(1000)]) and got == mm.mth(leaves)


def test_pages_quarter_million_entries(eng):
    n = 1 << 18
    pg = Pages(n)
    with new_db(eng, table_capacity=1 << 21) as db, new_db(eng, table_capacity=1 << 21) as twin:
        r = raw_both(db, twin, pg.args(0, n), eng.LogTree())
    assert r.tree.size == n
    hashes = pg.hashes(0, n)
    assert r.tree.root == mm.mth_hashes(hashes)
    assert r.tree.edge.tobytes() == mm.edge_rows(mm.edge(hashes, n), n)


# ---------------------------------------------------------------------------------------------------------------- tiles
class Tiles:
    """consecutive data tiles first .. first + len(widths) - 1 from libctmr's host generator; a width below 256 is the
    tile's first W TileLeafs"""

    def __init__(self, first, widths, gap=b"\x00" * 3):
        from ct_mapreduce_b200 import capi, engine, frontend as fe
        nt = len(widths)
        cfg = capi.synth_cfg(256 * (first + nt))
        iblob, ioffs = engine.synth_issuers(cfg)
        self.certs = [iblob[int(ioffs[k]):int(ioffs[k + 1])].tobytes() for k in range(cfg.n_issuers)]
        self.by_fp = {hashlib.sha256(d).digest(): d for d in self.certs}
        fps = np.frombuffer(b"".join(hashlib.sha256(d).digest() for d in self.certs), np.uint8).copy()
        L = capi.load()
        need = L.ctmr_synth_tiles_host(C.byref(cfg), first, nt, capi.ptr(fps), None, 0, None, None)
        buf = np.zeros(need, np.uint8)
        off, ln = np.zeros(nt, np.uint64), np.zeros(nt, np.uint32)
        assert L.ctmr_synth_tiles_host(C.byref(cfg), first, nt, capi.ptr(fps), capi.ptr(buf), need, capi.ptr(off), capi.ptr(ln)) == need
        self.tiles, self.te, self.chain0 = [], [], []
        for t, w in enumerate(widths):
            tile = buf[int(off[t]):int(off[t] + ln[t])].tobytes()
            parts = fe.split_tile(tile, 256)[:w]
            self.chain0.append({chain[0] for _, _, _, chain in parts if chain})
            enc = b""
            for te, etype, pre, chain in parts:
                enc += te + ((len(pre).to_bytes(3, "big") + pre) if etype == 1 else b"") + (32 * len(chain)).to_bytes(2, "big") + b"".join(chain)
            self.tiles.append(enc)
            self.te += [te for te, _, _, _ in parts]
        self.first, self.widths, self.gap = first, list(widths), gap
        self.pack()

    def pack(self):
        data, off, ln = bytearray(), [], []
        for t in self.tiles:
            data += self.gap
            off.append(len(data)); ln.append(len(t))
            data += t
        self.data, self.off, self.len = bytes(data), np.array(off, np.uint64), np.array(ln, np.uint32)
        self.index = np.arange(self.first, self.first + len(self.tiles), dtype=np.uint64)
        self.width = np.array(self.widths, np.uint16)

    def hashes(self, lo, hi):
        """leaf hashes of log positions [lo, hi)"""
        b = 256 * self.first
        return [mm.leaf_hash(b"\x00\x00" + te) for te in self.te[lo - b:hi - b]]

    def args(self, sl=slice(None)):
        return self.data, self.off[sl], self.len[sl], self.index[sl], self.width[sl]

    def register(self, db, certs=None):
        from conftest import pack
        db.register_chain_certs(*pack(self.certs if certs is None else certs))


@pytest.fixture(scope="module")
def tiles():
    return Tiles(40, [256] * 5 + [77])


def tiles_both(db, twin, args, tree, **kw):
    r = db.store_tiles(*args, NOW_NS, want_meta=True, want_pem=True, tree=tree, **kw)
    p = twin.store_tiles(*args, NOW_NS, want_meta=True, want_pem=True, **kw)
    same(r, p, TILE_FIELDS, db, twin)
    assert r.tiles_done == p.tiles_done and r.missing == p.missing
    return r


@pytest.mark.parametrize("skip", [0, 1, 77, 255, 256])
def test_tiles_from_the_first_tile_or_inside_it(eng, tiles, skip):
    start = 256 * 40 + skip
    rng = np.random.default_rng(skip)
    with new_db(eng) as db, new_db(eng) as twin:
        tiles.register(db)
        tiles.register(twin)
        tree, e = random_tree(eng, start, rng)
        r = tiles_both(db, twin, tiles.args(), tree, want_leaf_hash=True)
        expect(r.tree, e, start, tiles.hashes(start, 256 * 45 + 77))
        # and without asking for the leaf hashes
        tree, e = random_tree(eng, start, rng)
        r = tiles_both(db, twin, tiles.args(), tree)
        expect(r.tree, e, start, tiles.hashes(start, 256 * 45 + 77))


def test_tiles_several_chunks_per_call(eng, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(3 << 20))   # 1.5 MB of tiles per chunk
    tl = Tiles(7, [256] * 12 + [9])
    hashes = tl.hashes(256 * 7, 256 * 19 + 9)
    with new_db(eng, max_batch_entries=700) as db, new_db(eng, max_batch_entries=700) as twin:
        tl.register(db)
        tl.register(twin)
        rng = np.random.default_rng(1)
        tree, e = random_tree(eng, 256 * 7 + 3, rng)
        r = tiles_both(db, twin, tl.args(), tree, want_leaf_hash=True)
        expect(r.tree, e, 256 * 7 + 3, hashes[3:])


def test_tiles_bad_tile_stops_the_fold(eng, tiles):
    from ct_mapreduce_b200 import capi
    bad = Tiles(40, [256] * 5 + [77])
    bad.tiles[2] = bad.tiles[2] + b"\x00"   # trailing byte: the tile does not split into 256 TileLeafs
    bad.pack()
    rng = np.random.default_rng(3)
    with new_db(eng) as db, new_db(eng) as twin:
        bad.register(db)
        bad.register(twin)
        tree, e = random_tree(eng, 256 * 40 + 5, rng)
        r = tiles_both(db, twin, bad.args(), tree)
        assert r.tile_status.tolist() == [0, 0, capi.FE_BAD_TILE, 0, 0, 0] and r.tiles_done == 6
        expect(r.tree, e, 256 * 40 + 5, bad.hashes(256 * 40 + 5, 256 * 42))


def test_tiles_stop_and_resume_equals_one_call(eng, tiles):
    # exactly the Chain[0] certificates of the first two tiles: the call stops at the first tile that needs another
    some = [tiles.by_fp[fp] for fp in set().union(*tiles.chain0[:2])]
    rng = np.random.default_rng(4)
    start = 256 * 40 + 100
    tree, e = random_tree(eng, start, rng)
    fetched = []

    def fetch(fps):
        fetched.append(len(fps))
        return [tiles.by_fp[f] for f in fps]

    with new_db(eng) as db, new_db(eng) as twin, new_db(eng) as one:
        tiles.register(db, some)
        tiles.register(twin, some)
        # without fetch: the stop writes the tree of the completed tiles
        r = tiles_both(db, twin, tiles.args(), tree)
        assert 2 <= r.tiles_done < 6 and r.missing
        done = r.tiles_done
        assert r.tree.size == max(start, 256 * (40 + done))
        expect(r.tree, e, start, tiles.hashes(start, r.tree.size))
        # resume from tiles_done with that tree, fetching what is missing
        r2 = tiles_both(db, twin, tiles.args(slice(done, None)), r.tree, fetch=fetch)
        assert fetched and r2.tiles_done == 6 - done
        tiles.register(one)
        r1 = one.store_tiles(*tiles.args(), NOW_NS, tree=tree)
        assert r1.tiles_done == 6
        assert (r2.tree.size, r2.tree.edge.tobytes(), r2.tree.root) == (r1.tree.size, r1.tree.edge.tobytes(), r1.tree.root)
        expect(r1.tree, e, start, tiles.hashes(start, 256 * 45 + 77))


def test_tiles_bad_tile_before_a_stop(eng):
    """A bad tile ends the fold; a later tile stops the call on an unknown Chain[0].  The stop writes back the tree held
    at the bad tile, which is final for the batch: the resume loop finishes with the plain call, and tree and outputs
    equal one call made with every certificate registered first."""
    from ct_mapreduce_b200 import capi
    from ct_mapreduce_b200.capi import CtmrError
    tl = Tiles(40, [256] * 5 + [77])
    # the Chain[0] certificates of tiles 0 and 2 only: tile 1 is made bad, the stop comes at tile 3 or later
    some = [tl.by_fp[fp] for fp in tl.chain0[0] | tl.chain0[2]]
    tl.tiles[1] = tl.tiles[1] + b"\x00"
    tl.pack()
    start = 256 * 40 + 9
    tree, e = random_tree(eng, start, np.random.default_rng(10))
    fetched = []

    def fetch(fps):
        fetched.append(len(fps))
        return [tl.by_fp[f] for f in fps]

    with new_db(eng) as db, new_db(eng) as twin, new_db(eng) as one:
        tl.register(db, some)
        tl.register(twin, some)
        r = tiles_both(db, twin, tl.args(), tree, fetch=fetch)
        assert fetched and r.tiles_done == 6 and r.tile_status.tolist() == [0, capi.FE_BAD_TILE, 0, 0, 0, 0]
        expect(r.tree, e, start, tl.hashes(start, 256 * 41))
        tl.register(one)
        r1 = one.store_tiles(*tl.args(), NOW_NS, want_meta=True, want_pem=True, tree=tree)
        same(r, r1, TILE_FIELDS, db, one)
        assert (r.tree.size, r.tree.edge.tobytes(), r.tree.root) == (r1.tree.size, r1.tree.edge.tobytes(), r1.tree.root)

    # the library's side of it: the stop's tree is below the resume tile, so only the plain call continues
    with new_db(eng) as db, new_db(eng) as twin:
        tl.register(db, some)
        tl.register(twin, some)
        r = tiles_both(db, twin, tl.args(), tree)
        done = r.tiles_done
        assert 3 <= done < 6 and r.missing and r.tree.size == 256 * 41 < 256 * (40 + done)
        with pytest.raises(CtmrError) as ex:
            db.store_tiles(*tl.args(slice(done, None)), NOW_NS, tree=r.tree)
        assert ex.value.code == capi.E_INVALID
        tl.register(db)
        tl.register(twin)
        tiles_both(db, twin, tl.args(slice(done, None)), None)


def next_index(db):
    return int(np.frombuffer(db.snapshot()[48:56].tobytes(), np.uint64)[0])


def test_tiles_invalid_arguments(eng, tiles):
    from ct_mapreduce_b200 import capi
    from ct_mapreduce_b200.capi import CtmrError
    rng = np.random.default_rng(6)
    with new_db(eng, table_capacity=1 << 12) as db:
        tiles.register(db)
        d, off, ln, idx, w = tiles.args()
        cases = [
            ("gap", (d, off, ln, np.array([40, 41, 43, 44, 45, 46], np.uint64), w), 256 * 40),
            ("order", (d, off, ln, np.array([41, 40, 42, 43, 44, 45], np.uint64), w), 256 * 40),
            ("partial_not_last", (d, off[[5, 0]], ln[[5, 0]], idx[:2], w[[5, 0]]), 256 * 40),
            ("below", (d, off, ln, idx, w), 256 * 40 - 1),
            ("above", (d, off, ln, idx, w), 256 * 41 + 1),
            ("above_partial", (d, off[5:], ln[5:], idx[5:], w[5:]), 256 * 45 + 78),
            ("wraps", (d, off[:1], ln[:1], np.array([(1 << 56) - 1], np.uint64), w[:1]), 256 * ((1 << 56) - 1)),
        ]
        before = next_index(db)
        for name, args, size in cases:
            tree, _ = random_tree(eng, size, rng)
            keep = (tree.size, tree.edge.copy())
            ct = tree.to_c()
            o = capi.TileOut()
            b = capi.TileBatch(capi.ptr(np.frombuffer(args[0], np.uint8)), len(args[0]), capi.ptr(args[1]), capi.ptr(args[2]),
                               capi.ptr(args[3]), capi.ptr(args[4]), args[1].size, NOW_NS)
            rc = db._lib.ctmr_process_tiles_tree(db.handle, C.byref(b), C.byref(o), C.byref(ct))
            assert rc == capi.E_INVALID, name
            assert eng.LogTree.from_c(ct).size == keep[0] and bytes(ct.edge) == keep[1].tobytes(), name
            with pytest.raises(CtmrError):
                db.store_tiles(*args, NOW_NS, tree=tree)
        assert next_index(db) == before
        # the same tiles with a valid tree take their indices
        db.store_tiles(*tiles.args(), NOW_NS, tree=random_tree(eng, 256 * 40, rng)[0])
        assert next_index(db) == before + 256 * 5 + 77


def test_pages_size_must_not_wrap(eng, pages):
    from ct_mapreduce_b200.capi import CtmrError
    with new_db(eng, table_capacity=1 << 12) as db:
        tree, e = random_tree(eng, 2**64 - 3, np.random.default_rng(8))
        for n in (3, 4):
            with pytest.raises(CtmrError):
                db.store_raw_entries(*pages.args(0, n), NOW_NS, tree=tree)
        assert tree.size == 2**64 - 3
        r = db.store_raw_entries(*pages.args(0, 2), NOW_NS, tree=tree)
        expect(r.tree, e, 2**64 - 3, pages.hashes(0, 2))
        assert r.tree.size == 2**64 - 1


def test_group_refuses_a_tree(eng, pages, tiles):
    from ct_mapreduce_b200.capi import CtmrError
    with eng.GpuCertGroup([0, 0], log_expired_entries=True, table_capacity=1 << 14) as g:
        with pytest.raises(CtmrError):
            g.store_raw_entries(*pages.args(0, 4), NOW_NS, tree=eng.LogTree())
        with pytest.raises(CtmrError):
            g.store_tiles(*tiles.args(), NOW_NS, tree=eng.LogTree())
        # a member of the group is refused by the library itself
        from ct_mapreduce_b200 import capi
        m = g.members[0]
        ct = capi.Tree()
        o = capi.RawOut()
        text, lo, ll, xo, xl = pages.args(0, 1)
        b = capi.RawBatch(capi.ptr(text), text.size, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl), 1, NOW_NS)
        assert m._lib.ctmr_process_raw_tree(m.handle, C.byref(b), C.byref(o), C.byref(ct)) == capi.E_INVALID
