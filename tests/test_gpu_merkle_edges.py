"""Edges of the Merkle tree fold on the GPU (ctmr_process_raw_tree, ctmr_process_tiles_tree) that the corpus of
tests/test_gpu_merkle.py never reaches: every leaf length around the SHA-256 padding boundary, every kind of entry that
has or has no leaf, chunk and level edges, the level buffers at capacity, bad tiles at the batch's and a chunk's edges,
stops at tile 0 and twice in one fetch loop, and the launches the fold adds, against the restated fold
(tests/fold_model.py).

Every case runs the tree call on a DIRTY ctx: first it and its twin process an unrelated batch (other lengths, tree and
plain calls, bad base64), so the decoded arena, the leaf rows and both level buffers hold stale bytes.  The tree must
equal the hashlib model (size, every edge row, the root) and every other output must equal the twin's plain call.
Marked gpu."""
import base64
import contextlib

import numpy as np
import pytest

import fold_model as fm
import merkle_model as mm
from conftest import NOW_NS
from test_gpu_merkle import Pages, Tiles, expect, new_db, random_tree, raw_both, same, tiles_both, TILE_FIELDS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


# ---------------------------------------------------------------------------------------------------------- batches
class Raw:
    """a get-entries batch from entries (leaf bytes or None when leaf_input is not base64, leaf_input, extra_data)"""

    def __init__(self, entries):
        text, lo, ll, xo, xl = bytearray(b'{"entries":['), [], [], [], []
        for _, li, ed in entries:
            text += b'{"leaf_input":"'
            lo.append(len(text)); ll.append(len(li))
            text += li + b'","extra_data":"'
            xo.append(len(text)); xl.append(len(ed))
            text += ed + b'"},'
        self.entries = list(entries)
        self.text = np.frombuffer(bytes(text) + b"]}", np.uint8)
        self.lo, self.ll = np.array(lo, np.uint64), np.array(ll, np.uint32)
        self.xo, self.xl = np.array(xo, np.uint64), np.array(xl, np.uint32)

    def __len__(self):
        return len(self.entries)

    def args(self, a=0, b=None):
        b = len(self) if b is None else b
        return self.text, self.lo[a:b], self.ll[a:b], self.xo[a:b], self.xl[a:b]

    def hashes(self, a, b):
        """leaf hashes of entries [a, b) up to the first one without a leaf"""
        out = []
        for leaf, _, _ in self.entries[a:b]:
            if leaf is None:
                break
            out.append(mm.leaf_hash(leaf))
        return out


def page_entry(pg, i):
    x = int(pg.xo[i])
    return pg.leaf(i), base64.b64encode(pg.leaf(i)), pg.text[x:x + int(pg.xl[i])].tobytes()


def junk_leaf(L, rng):
    """L bytes that are not a MerkleTreeLeaf (BAD_LEAF): the second byte, MerkleLeafType, is not timestamped_entry"""
    x = bytearray(rng.bytes(L))
    if L >= 2:
        x[1] = 7
    return bytes(x)


def sloppy_b64(leaf):
    """base64 whose last quantum sets the bits that padding drops: the decoder writes nonzero bytes right behind the
    leaf in the arena, inside the granule the leaf hash reads"""
    s = bytearray(base64.b64encode(leaf))
    if len(leaf) % 3:
        k = len(s) - 1 - s.count(b"=", len(s) - 2)   # the last character that carries bits
        alpha = b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/"
        v = alpha.index(s[k]) | (0x0F if len(leaf) % 3 == 1 else 0x03)
        s[k] = alpha[v]
        assert base64.b64decode(bytes(s)) == leaf
    return bytes(s)


_SOIL = {}


def soil(eng, *dbs, tiles=False):
    """an unrelated batch through each ctx, identically: other lengths, a tree call and a plain call, bad base64"""
    if "raw" not in _SOIL:
        rng = np.random.default_rng(99)
        pg = Pages(300)
        ents = [page_entry(pg, i) for i in range(300)]
        for i in range(0, 300, 7):
            leaf = junk_leaf(int(rng.integers(2000, 9000)), rng)
            ents[i] = (leaf, base64.b64encode(leaf), b"")
        ents[150] = (None, b"!!!!" + ents[150][1][4:], ents[150][2])
        _SOIL["raw"] = Raw(ents)
    if tiles and "tiles" not in _SOIL:
        _SOIL["tiles"] = Tiles(3, [256, 256, 100])
    for db in dbs:
        db.store_raw_entries(*_SOIL["raw"].args(), NOW_NS, tree=random_tree(eng, 777, np.random.default_rng(1))[0])
        db.store_raw_entries(*_SOIL["raw"].args(), NOW_NS)
        if tiles:
            tl = _SOIL["tiles"]
            tl.register(db)
            db.store_tiles(*tl.args(), NOW_NS, want_leaf_hash=True, tree=random_tree(eng, 256 * 3 + 9, np.random.default_rng(2))[0])
            db.store_tiles(*tl.args(), NOW_NS)


@contextlib.contextmanager
def dirty_pair(eng, tiles=False, **kw):
    db, twin = new_db(eng, **kw), new_db(eng, **kw)
    try:
        soil(eng, db, twin, tiles=tiles)
        yield db, twin
    finally:
        db.close()
        twin.close()


@pytest.fixture(scope="module")
def shared(eng):
    with dirty_pair(eng) as p:
        yield p


@pytest.fixture
def pair(eng, shared):
    soil(eng, *shared)
    return shared


def launches(db):
    return db.frontend_profile_last()[2]


def run_raw(eng, pair, raw, start, rng, a=0, b=None):
    b = len(raw) if b is None else b
    tree, e = random_tree(eng, start, rng)
    r = raw_both(*pair, raw.args(a, b), tree)
    expect(r.tree, e, start, raw.hashes(a, b))
    return r


# ------------------------------------------------------------------------------------------------ 1. leaf lengths (pages)
def test_pages_every_leaf_length(eng, pair):
    from ct_mapreduce_b200 import capi
    rng = np.random.default_rng(7)
    ents = []
    for L in range(0, 301):
        leaf = junk_leaf(L, rng)
        ents.append((leaf, sloppy_b64(leaf) if L % 2 else base64.b64encode(leaf), b""))
    for base in (1024, 8192, 70 * 1024):
        for r in range(52, 69):   # L + 1 = base + r: around 55/56 and 63/64 mod 64
            leaf = junk_leaf(base + r - 1, rng)
            ents.append((leaf, base64.b64encode(leaf), b""))
    pg = Pages(40)
    ents += [page_entry(pg, i) for i in range(40)]
    raw = Raw(ents)
    for start in (0, 2**40 + 3):
        r = run_raw(eng, pair, raw, start, rng)
        assert r.tree.size == start + len(raw)
        assert (r.entry_status[:-40] == capi.FE_BAD_LEAF).all()
        assert set(r.entry_type[-40:].tolist()) == {0, 1}   # x509 and precert leaves
    for L in range(0, 131):
        leaf = junk_leaf(L, rng)
        r = raw_both(*pair, Raw([(leaf, sloppy_b64(leaf), b"")]).args(), eng.LogTree())
        assert r.tree.size == 1 and r.tree.root == mm.leaf_hash(leaf), L


# ------------------------------------------------------------------------------------ 2. which entries have a leaf (pages)
def folding_kinds(pg):
    """(entry, status) of entries that fold though the front end rejects them"""
    import struct
    from ct_mapreduce_b200 import capi
    leaf, li, ed = page_entry(pg, 1)
    assert leaf[10:12] == b"\x00\x00" and leaf[15] == 0x30   # an x509_entry
    unknown = bytearray(leaf)
    unknown[10:12] = b"\x00\x05"
    bad_cert = leaf[:15] + b"\x31" + leaf[16:]   # the certificate is a SET, not a SEQUENCE
    empty = b""
    return [
        ((leaf, li, b"!" + ed[1:]), capi.FE_BAD_BASE64),                               # extra_data alone is not base64
        ((bytes(unknown), base64.b64encode(bytes(unknown)), ed), capi.FE_UNKNOWN_TYPE),
        ((leaf, li, base64.b64encode(struct.pack(">I", 7)[1:] + b"\x00\x00")), capi.FE_BAD_EXTRA),
        ((bad_cert, base64.b64encode(bad_cert), ed), capi.FE_BAD_CERT),
        ((empty, b"", ed), capi.FE_BAD_LEAF),
    ]


def no_leaf_kinds(pg):
    """leaf_input strings that are not base64, each as (name, string)"""
    leaf = pg.leaf(2)[:60]
    good = base64.b64encode(leaf)   # 80 characters, no padding
    assert len(good) == 80
    out = []
    for c in list(range(16)) + list(range(64, 80)):   # every position mod 16 of the first and the last granule
        s = bytearray(good)
        s[c] = ord("!")
        out.append(("junk@%d" % c, bytes(s)))
    for extra in (b"A", b"AB", b"ABC"):
        out.append(("len%%4=%d" % len(extra), good + extra))
    padded = base64.b64encode(leaf[:59])
    assert padded.endswith(b"=")
    out.append(("= inside", padded[:40] + b"=" + padded[41:]))
    out.append(("= early", padded[:-4] + b"A=AA"))
    return out


def test_pages_entries_that_fold(eng, pair):
    rng = np.random.default_rng(8)
    pg = Pages(40)
    base = [page_entry(pg, i) for i in range(40)]
    for (entry, status) in folding_kinds(pg):
        for j in (0, 17, 39):
            ents = list(base)
            ents[j] = entry
            r = run_raw(eng, pair, Raw(ents), 5000 + j, rng)
            assert r.entry_status[j] == status, (status, j)
            assert r.tree.size == 5000 + j + 40


def test_pages_entries_without_a_leaf(eng, pair):
    from ct_mapreduce_b200 import capi
    rng = np.random.default_rng(9)
    pg = Pages(40)
    base = [page_entry(pg, i) for i in range(40)]
    for name, s in no_leaf_kinds(pg):
        for j in (0, 20, 39):
            ents = list(base)
            ents[j] = (None, s, base[j][2])
            r = run_raw(eng, pair, Raw(ents), 99 + j, rng)
            assert r.entry_status[j] == capi.FE_BAD_BASE64, name
            assert r.tree.size == 99 + 2 * j, name


def test_pages_two_without_a_leaf_the_lowest_wins(eng, pair):
    rng = np.random.default_rng(10)
    pg = Pages(600)
    base = [page_entry(pg, i) for i in range(600)]
    for lo_, hi_ in ((3, 4), (5, 300), (255, 256), (0, 599), (511, 512)):
        ents = list(base)
        for j in (hi_, lo_):
            ents[j] = (None, b"!" + base[j][1][1:], base[j][2])
        r = run_raw(eng, pair, Raw(ents), 2**33 + 1, rng)
        assert r.tree.size == 2**33 + 1 + lo_


# ---------------------------------------------------------------------------------------------------------- 3. chunks
def chunk_launches(first_pos, n, m, chars=None, cap_text=None):
    """the launches a tree call adds to the plain call: per chunk, raw_leaf_hash and the fold.  A chunk takes at most m
    entries and, when chars (leaf_input + extra_data characters per entry) are given, half of cap_text (Pages::fit)."""
    out, j = 0, 0
    while j < n:
        c, used = 0, 0
        while j + c < n and c < m and (chars is None or used + int(chars[j + c]) <= cap_text // 2):
            used += 0 if chars is None else int(chars[j + c])
            c += 1
        assert c
        out += 1 + fm.launches(first_pos + j, c)
        j += c
    return out


@pytest.mark.parametrize("m", [1, 2, 3, 5, 8])
def test_pages_chunks(eng, m):
    rng = np.random.default_rng(m)
    pg = Pages(40)
    base = [page_entry(pg, i) for i in range(40)]
    bad = lambda j: (None, base[j][1][:-1] + b"!", base[j][2])   # noqa: E731
    last = (39 // m) * m
    spots = [(), (0,), (m // 2,), (m - 1,), (m,), (m + m // 2,), (2 * m - 1,), (last,), ((last + 39) // 2,), (39,),
             (m + 1, last), (2 * m - 1, 39)]
    with dirty_pair(eng, max_batch_entries=m) as p:
        for start in list(range(18)) + [2**32 - 1, 2**63 - 3]:
            r = run_raw(eng, p, Raw(base), start, rng)
            assert r.tree.size == start + 40
            assert launches(p[0]) - launches(p[1]) == chunk_launches(start, 40, m)
        for spot in spots:
            ents = list(base)
            for j in spot:
                ents[j] = bad(j)
            for start in (0, 5, 2**32 - 1):
                r = run_raw(eng, p, Raw(ents), start, rng)
                assert r.tree.size == start + (min(spot) if spot else 40), spot
                assert launches(p[0]) - launches(p[1]) == chunk_launches(start, 40, m)
        # one tree carried across three calls whose chunk boundaries differ
        pg2 = Pages(100)
        raw = Raw([page_entry(pg2, i) for i in range(100)])
        tree = eng.LogTree()
        for a, b in ((0, 7), (7, 18), (18, 100)):
            tree = raw_both(*p, raw.args(a, b), tree).tree
        assert tree.size == 100 and tree.root == mm.mth([pg2.leaf(i) for i in range(100)])
        # an empty tree call launches nothing: tree_root, in tree_end, is not counted
        z = np.zeros(0, np.uint64), np.zeros(0, np.uint32)
        assert p[0].store_raw_entries(b"x", z[0], z[1], z[0], z[1], NOW_NS, tree=tree).tree.root == tree.root
        assert launches(p[0]) == 0


def test_pages_chunks_cut_by_the_text_budget(eng, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(1 << 16))
    rng = np.random.default_rng(12)
    pg = Pages(200)
    base = [page_entry(pg, i) for i in range(200)]
    with dirty_pair(eng) as p:
        for spot in ((), (0,), (13,), (77,), (150, 40), (199,)):
            ents = list(base)
            for j in spot:
                ents[j] = (None, base[j][1] + b"A", base[j][2])
            raw = Raw(ents)
            r = run_raw(eng, p, raw, 1001, rng)
            assert r.tree.size == 1001 + (min(spot) if spot else 200)
            chars = raw.ll.astype(np.int64) + raw.xl
            assert launches(p[0]) - launches(p[1]) == chunk_launches(1001, 200, 1 << 18, chars, 1 << 16)


# -------------------------------------------------------------------------------------------------------- 4. capacity
@pytest.mark.parametrize("E", [4096, 4097])
def test_pages_chunk_of_exactly_the_capacity(eng, E):
    pg = Pages(E + 1)
    raw = Raw([page_entry(pg, i) for i in range(E + 1)])
    rng = np.random.default_rng(E)
    with dirty_pair(eng, max_batch_entries=E) as p:
        for start in (2**20 + 1, 2**20, 3, 0):
            for n in (E, E + 1):
                r = run_raw(eng, p, raw, start, rng, 0, n)
                assert r.tree.size == start + n
                assert launches(p[0]) - launches(p[1]) == chunk_launches(start, n, E)


def test_pages_default_capacity_from_an_odd_start(eng):
    """2^18 entries (kStageEntries) at the default configuration, from an odd start.  The character budget cuts them
    into two uneven chunks, so this is a two-chunk fold at full scale, not a chunk of exactly the capacity: that edge,
    where the level buffers' E / 2 + 2 rows are tightest, is test_pages_chunk_of_exactly_the_capacity's."""
    n = 1 << 18
    pg = Pages(n)
    rng = np.random.default_rng(18)
    start = 2**31 + 1
    with dirty_pair(eng, table_capacity=1 << 21) as (db, twin):
        tree, e = random_tree(eng, start, rng)
        r = raw_both(db, twin, pg.args(0, n), tree)
        expect(r.tree, e, start, pg.hashes(0, n))
        # the character budget, n * 6144, cuts the batch in two
        chars = pg.ll[:n].astype(np.int64) + pg.xl[:n]
        assert launches(db) - launches(twin) == chunk_launches(start, n, n, chars, n * 6144)


# ----------------------------------------------------------------------------------------------------------- 5. tiles
def retile(tl, t, edits):
    """tile t of `tl` with TimestampedEntries replaced: edits {j: fn(te) -> te}"""
    from ct_mapreduce_b200 import frontend as fe
    parts = fe.split_tile(tl.tiles[t], tl.widths[t])
    enc = b""
    for j, (te, etype, pre, chain) in enumerate(parts):
        if j in edits:
            te = edits[j](te)
            tl.te[256 * t + j] = te
        enc += te + ((len(pre).to_bytes(3, "big") + pre) if etype == 1 else b"") + (32 * len(chain)).to_bytes(2, "big") + b"".join(chain)
    tl.tiles[t] = enc
    tl.pack()


def bad_index(te):
    return te[:-1] + bytes([te[-1] ^ 1])   # the leaf_index extension's last byte: not 256 * N + j


def bad_cert(te):
    assert te[8:10] == b"\x00\x00" and te[13] == 0x30
    return te[:13] + b"\x31" + te[14:]   # the certificate is a SET, not a SEQUENCE


def tile_launches(first_pos, n, want_leaf_hash):
    return (0 if want_leaf_hash else 1) + fm.launches(first_pos, n) if n else 0


def tiles_run(eng, p, tl, start, rng, want_leaf_hash, sl=slice(None), **kw):
    tree, e = random_tree(eng, start, rng)
    r = tiles_both(*p, tl.args(sl), tree, want_leaf_hash=want_leaf_hash, **kw)
    if want_leaf_hash:
        from ct_mapreduce_b200 import frontend as fe
        for i in np.nonzero(r.entry_status != 6)[0]:
            assert r.leaf_hash[i].tobytes() == fe.leaf_hash(tl.te[int(i)]), i
    return r, tree, e


@pytest.fixture(scope="module")
def tpair(eng):
    with dirty_pair(eng, tiles=True) as p:
        yield p


@pytest.fixture
def tp(eng, tpair):
    soil(eng, *tpair, tiles=True)
    return tpair


@pytest.mark.parametrize("want_leaf_hash", [True, False])
def test_tiles_bad_index_and_bad_cert_fold(eng, tp, want_leaf_hash):
    from ct_mapreduce_b200 import capi
    tl = Tiles(40, [256, 256, 100])
    x509 = [j for j in range(256) if tl.te[256 + j][8:10] == b"\x00\x00"]
    retile(tl, 0, {0: bad_index, 5: bad_index, 255: bad_index})
    retile(tl, 1, {x509[0]: bad_cert, x509[-1]: bad_cert})
    retile(tl, 2, {99: bad_index})
    tl.register(tp[0])
    tl.register(tp[1])
    rng = np.random.default_rng(20)
    for start in (256 * 40, 256 * 40 + 3):
        r, _, e = tiles_run(eng, tp, tl, start, rng, want_leaf_hash)
        st = r.entry_status
        assert [st[0], st[5], st[255], st[256 + x509[0]], st[256 + x509[-1]], st[611]] == \
            [capi.FE_BAD_INDEX] * 3 + [capi.FE_BAD_CERT] * 2 + [capi.FE_BAD_INDEX]
        expect(r.tree, e, start, tl.hashes(start, 256 * 42 + 100))
        assert launches(tp[0]) - launches(tp[1]) == tile_launches(256 * 40, 612, want_leaf_hash)
        assert set(r.entry_type.tolist()) == {0, 1}   # precertificate TileLeafs too
        assert len({len(te) % 64 for te in tl.te}) == 64   # TimestampedEntry lengths at every residue mod 64


@pytest.mark.parametrize("want_leaf_hash", [True, False])
def test_tiles_bad_first_tile(eng, tp, want_leaf_hash):
    from ct_mapreduce_b200 import capi
    tl = Tiles(50, [256, 256, 30])
    tl.tiles[0] += b"\x00"
    tl.pack()
    tl.register(tp[0])
    tl.register(tp[1])
    rng = np.random.default_rng(21)
    for start, end in ((256 * 50, 256 * 50), (256 * 50 + 10, 256 * 50 + 10), (256 * 50 + 255, 256 * 50 + 255),
                       (256 * 51, 256 * 52 + 30)):   # at its end, every leaf of the bad tile is already in the tree
        r, _, e = tiles_run(eng, tp, tl, start, rng, want_leaf_hash)
        assert r.tile_status.tolist() == [capi.FE_BAD_TILE, 0, 0]
        expect(r.tree, e, start, tl.hashes(start, end))
        assert r.tree.size == end


@pytest.mark.parametrize("want_leaf_hash", [True, False])
def test_tiles_bad_partial_last_tile(eng, tp, want_leaf_hash):
    tl = Tiles(60, [256, 256, 77])
    tl.tiles[2] = tl.tiles[2][:-1]
    tl.pack()
    tl.register(tp[0])
    tl.register(tp[1])
    rng = np.random.default_rng(22)
    r, _, e = tiles_run(eng, tp, tl, 256 * 60 + 1, rng, want_leaf_hash)
    assert r.tile_status.tolist() == [0, 0, 6]
    expect(r.tree, e, 256 * 60 + 1, tl.hashes(256 * 60 + 1, 256 * 62))


def tile_chunks(tl, cap_text, cap_entries=1 << 18):
    """Tiles::fit: the first tile of every chunk"""
    starts, lo = [], 0
    while lo < len(tl.tiles):
        starts.append(lo)
        hi, nbytes = lo, 0
        while hi < len(tl.tiles) and 256 * (hi + 1 - lo) <= cap_entries and nbytes + int(tl.len[hi]) <= cap_text // 2:
            nbytes += int(tl.len[hi])
            hi += 1
        assert hi > lo
        lo = hi
    return starts


@pytest.mark.parametrize("want_leaf_hash", [True, False])
def test_tiles_bad_first_tile_of_a_later_chunk(eng, monkeypatch, want_leaf_hash):
    from ct_mapreduce_b200 import capi
    cap = 3 << 20
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(cap))
    tl = Tiles(7, [256] * 9 + [40])
    starts = tile_chunks(tl, cap)
    assert len(starts) >= 3
    k = starts[1]
    tl.tiles[k] += b"\x00"
    tl.pack()
    assert tile_chunks(tl, cap) == starts
    rng = np.random.default_rng(23)
    with dirty_pair(eng, tiles=True) as p:
        tl.register(p[0])
        tl.register(p[1])
        r, _, e = tiles_run(eng, p, tl, 256 * 7 + 100, rng, want_leaf_hash)
        assert r.tile_status[k] == capi.FE_BAD_TILE and r.tile_status.sum() == capi.FE_BAD_TILE
        expect(r.tree, e, 256 * 7 + 100, tl.hashes(256 * 7 + 100, 256 * (7 + k)))
        # the chunk after the bad tile's folds nothing, but its launches are made all the same
        ent = np.concatenate([[0], np.cumsum(tl.widths)])
        want = sum(tile_launches(256 * 7 + int(ent[a]), int(ent[b] - ent[a]), want_leaf_hash)
                   for a, b in zip(starts, starts[1:] + [len(tl.tiles)]))
        assert launches(p[0]) - launches(p[1]) == want


@pytest.mark.parametrize("want_leaf_hash", [True, False])
def test_tiles_stop_at_tile_zero_then_resume(eng, want_leaf_hash):
    tl = Tiles(40, [256] * 3 + [77])
    start = 256 * 40 + 200
    rng = np.random.default_rng(24)
    fetched = ([], [])   # the fetch calls of each ctx's loop

    def fetcher(k):
        def fetch(fps):
            fetched[k].append(len(fps))
            return [tl.by_fp[f] for f in fps]
        return fetch

    with dirty_pair(eng) as p, new_db(eng) as one:   # no chain certificate registered
        tree, e = random_tree(eng, start, rng)
        # nothing is processed: no output to compare but the stop itself (the dense issuer numbering of two ctxs may
        # differ, so the untouched zeros would not compare)
        r = p[0].store_tiles(*tl.args(), NOW_NS, want_leaf_hash=want_leaf_hash, tree=tree)
        q = p[1].store_tiles(*tl.args(), NOW_NS, want_leaf_hash=want_leaf_hash)
        assert r.tiles_done == q.tiles_done == 0 and r.missing and r.missing == q.missing
        expect(r.tree, e, start, [])   # written back unchanged, with its root
        assert launches(p[0]) == launches(p[1]) + (0 if want_leaf_hash else 1)   # the stop chunk folds nothing
        kw = dict(want_meta=True, want_pem=True, want_leaf_hash=want_leaf_hash)
        r2 = p[0].store_tiles(*tl.args(), NOW_NS, tree=r.tree, fetch=fetcher(0), **kw)
        q2 = p[1].store_tiles(*tl.args(), NOW_NS, fetch=fetcher(1), **kw)
        same(r2, q2, TILE_FIELDS, *p)
        assert r2.tiles_done == q2.tiles_done == 4
        assert len(fetched[0]) >= 2 and fetched[0] == fetched[1]   # two stops or more in each ctx's fetch loop
        expect(r2.tree, e, start, tl.hashes(start, 256 * 43 + 77))
        tl.register(one)
        r1 = one.store_tiles(*tl.args(), NOW_NS, want_meta=True, want_pem=True, want_leaf_hash=want_leaf_hash, tree=tree)
        same(r2, r1, TILE_FIELDS, p[0], one)
        assert (r2.tree.size, r2.tree.edge.tobytes(), r2.tree.root) == (r1.tree.size, r1.tree.edge.tobytes(), r1.tree.root)


@pytest.mark.parametrize("want_leaf_hash", [True, False])
def test_tiles_one_tile_already_in_the_tree(eng, tp, want_leaf_hash):
    rng = np.random.default_rng(25)
    for w in (256, 77, 1):
        tl = Tiles(90, [w])
        tl.register(tp[0])
        tl.register(tp[1])
        r, _, e = tiles_run(eng, tp, tl, 256 * 90 + w, rng, want_leaf_hash)
        expect(r.tree, e, 256 * 90 + w, [])
        assert launches(tp[0]) - launches(tp[1]) == tile_launches(256 * 90, w, want_leaf_hash)


@pytest.mark.parametrize("want_leaf_hash", [True, False])
def test_tiles_partial_last_tile_widths(eng, tp, want_leaf_hash):
    rng = np.random.default_rng(26)
    for w in (1, 2, 127, 255):
        tl = Tiles(30, [256, w])
        tl.register(tp[0])
        tl.register(tp[1])
        for start in (256 * 30, 256 * 30 + 5):
            r, _, e = tiles_run(eng, tp, tl, start, rng, want_leaf_hash)
            expect(r.tree, e, start, tl.hashes(start, 256 * 31 + w))
            assert r.tree.size == 256 * 31 + w
            assert launches(tp[0]) - launches(tp[1]) == tile_launches(256 * 30, 256 + w, want_leaf_hash)
