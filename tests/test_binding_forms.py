"""Which C entry point each binding method calls, on one ctx (ctmr_*) and on a group (ctmr_group_*, or member 0 for
the issuer registry), in which order and with which scalar arguments.  No GPU: the classes are built without their
constructors over a fake library that records every call and returns 0."""
import ctypes as C

import numpy as np
import pytest

from ct_mapreduce_b200 import capi, engine

NOW_NS = 1767225600 * 10**9
DIGEST = bytes(range(32))


class FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("ctmr_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name, args))
            return 0
        return call


def _db(lib, h):
    db = object.__new__(engine.GpuCertDatabase)
    db._lib, db._h, db._owned = lib, C.c_void_p(h), False
    return db


def _ctx():
    lib = FakeLib()
    return _db(lib, 0x1000), lib, {"self": 0x1000, "registry": 0x1000}, "ctmr_"


def _group():
    lib = FakeLib()
    g = object.__new__(engine.GpuCertGroup)
    g._lib, g._h = lib, C.c_void_p(0x2000)
    g.members = [_db(lib, 0x3000), _db(lib, 0x4000)]
    return g, lib, {"self": 0x2000, "registry": 0x3000}, "ctmr_group_"


def _u8(b):
    return np.frombuffer(b, np.uint8).copy()


def _raw():
    return (b"QUFB", [0], [4], [0], [0], NOW_NS)


def _bodies():
    return (b'{"entries":[]}', [0], [14], [2], NOW_NS)


def _tiles():
    return (b"\0" * 8, [0], [8], [0], [1], NOW_NS)


def _store_batch(db):
    blob, offs = _u8(b"abcdef"), np.array([0, 2, 6], np.uint64)
    db.store_batch(blob, offs, _u8(b"xyz"), np.array([0, 3], np.uint64), np.zeros(2, np.uint32), NOW_NS)


def _with_trees(db, method, *a, **k):
    """the tree forms: tree= on one ctx, <method>_with_trees on a group"""
    return getattr(db, method + "_with_trees" if isinstance(db, engine.GpuCertGroup) else method)(*a, **k)


# (method, call, [(entry point, handle, {argument position: scalar})]): "~x" is ctmr_x on a ctx and ctmr_group_x on a
# group; handle "self" is the db's own handle, "registry" the ctx that holds the issuer registry (a group's member 0)
CASES = [
    ("store_batch", _store_batch, [("~process_batch", "self", {3: 2, 6: 1, 8: NOW_NS})]),
    ("store_raw_entries", lambda db: db.store_raw_entries(*_raw()), [("~process_raw", "self", {})]),
    ("store_raw_entries_tree", lambda db: _with_trees(db, "store_raw_entries", *_raw(), tree=engine.LogTree()),
     [("~process_raw_tree", "self", {})]),
    ("store_raw_entries_trees",
     lambda db: _with_trees(db, "store_raw_entries", *_raw(), trees=[engine.LogTree()] * 3, entry_log=[0]),
     [("~process_raw_trees", "self", {5: 3})]),
    ("store_raw_bodies", lambda db: db.store_raw_bodies(*_bodies()), [("~process_raw_bodies", "self", {})]),
    ("store_raw_bodies_tree",
     lambda db: _with_trees(db, "store_raw_bodies", *_bodies(), tree=engine.LogTree(), body_start=[0]),
     [("~process_raw_bodies_tree", "self", {})]),
    ("store_raw_bodies_trees",
     lambda db: _with_trees(db, "store_raw_bodies", *_bodies(), trees=[engine.LogTree()] * 2, body_log=[1]),
     [("~process_raw_bodies_trees", "self", {6: 2})]),
    ("store_tiles", lambda db: db.store_tiles(*_tiles()), [("~process_tiles", "self", {})]),
    ("store_tiles_tree", lambda db: _with_trees(db, "store_tiles", *_tiles(), tree=engine.LogTree()),
     [("~process_tiles_tree", "self", {})]),
    ("store_tiles_trees", lambda db: _with_trees(db, "store_tiles", *_tiles(), trees=[engine.LogTree()] * 4, tile_log=[2]),
     [("~process_tiles_trees", "self", {5: 4})]),
    ("register_chain_certs", lambda db: db.register_chain_certs(_u8(b"abcde"), np.array([0, 2, 5], np.uint64)),
     [("~register_chain_certs", "self", {3: 2})]),
    ("register_issuers", lambda db: db.register_issuers(_u8(b"abcde"), np.array([0, 1, 3, 5], np.uint64)),
     [("ctmr_register_issuers", "registry", {3: 3})]),
    ("issuer_digest", lambda db: db.issuer_digest(5), [("ctmr_issuer_digest", "registry", {1: 5})]),
    ("preload_known", lambda db: db.preload_known(7, DIGEST, [b"\x01", b"\x02\x03"]),
     [("~preload_known", "self", {1: 7, 5: 2})]),
    ("evict_expired", lambda db: db.evict_expired(123), [("~evict_expired", "self", {1: 123})]),
    ("snapshot", lambda db: db.snapshot(), [("~snapshot_size", "self", {}), ("~snapshot_save", "self", {2: 0})]),
    ("restore", lambda db: db.restore(np.zeros(9, np.uint8)), [("~snapshot_load", "self", {2: 9})]),
    ("checkpoint", lambda db: db.checkpoint(), [("~checkpoint_size", "self", {}), ("~checkpoint_save", "self", {2: 1})]),
    ("load_checkpoint", lambda db: db.load_checkpoint([np.zeros(3, np.uint8), np.zeros(4, np.uint8)]),
     [("~checkpoint_load", "self", {3: 2})]),
    ("revoked_known", lambda db: db.revoked_known([b"crl"], [DIGEST]), [("~revoked_known", "self", {})]),
    ("revoked_cascade", lambda db: db.revoked_cascade([b"crl"], [DIGEST], 99, salt=b"ab"),
     [("~revoked_cascade", "self", {2: 99, 4: 2})]),
    ("revoked_stash", lambda db: db.revoked_stash([b"crl"], [DIGEST], 99, filter=b"abc", stashes=b"de"),
     [("~revoked_stash", "self", {2: 99, 4: 3, 6: 2})]),
    ("issuer_counts", lambda db: db.issuer_counts(),
     [("ctmr_issuer_count", "registry", {}), ("~issuer_counts", "self", {})]),
    ("status_counters", lambda db: db.status_counters(), [("~status_counters", "self", {})]),
    ("table_stats", lambda db: db.table_stats(), [("~table_stats", "self", {})]),
    ("set_cardinality", lambda db: db.get_known_certificates(-5, DIGEST).count(),
     [("~set_cardinality", "self", {1: -5})]),
]


@pytest.mark.parametrize("form", [_ctx, _group], ids=["ctx", "group"])
@pytest.mark.parametrize("method,call,want", CASES, ids=[c[0] for c in CASES])
def test_entry_points(form, method, call, want):
    db, lib, handles, prefix = form()
    call(db)
    got = [(name, args[0].value if isinstance(args[0], C.c_void_p) else args[0], args) for name, args in lib.calls]
    assert [(n, h) for n, h, _ in got] == [(n.replace("~", prefix), handles[h]) for n, h, _ in want]
    for (name, _, args), (_, _, scalars) in zip(got, want):
        for pos, value in scalars.items():
            assert args[pos] == value, (name, pos)


def test_set_cardinality_digest():
    for form in (_ctx, _group):
        db, lib, _, _ = form()
        db.get_known_certificates(3, DIGEST).count()
        assert bytes(lib.calls[0][1][2]) == DIGEST


def test_group_reset():
    g, lib, handles, _ = _group()
    g.reset()
    assert [(n, a[0].value) for n, a in lib.calls] == [("ctmr_group_reset", handles["self"])]


@pytest.mark.parametrize("method", ["map_device", "reduce_device", "process_device", "read_histogram_device", "profile_last",
                                    "sha256_ceiling", "reset_device", "check_device", "peer_export", "peer_attach",
                                    "peer_barrier_device", "peer_allreduce_histogram_device", "frontend_profile_last",
                                    "tiles_profile_last"])
def test_group_refuses_single_ctx_calls(method):
    g, lib, _, _ = _group()
    with pytest.raises(capi.CtmrError):
        getattr(g, method)(None, None)
    assert lib.calls == []


@pytest.mark.parametrize("method,kw", [("store_raw_entries", {"tree": engine.LogTree()}),
                                       ("store_tiles", {"trees": [engine.LogTree()]}),
                                       ("store_raw_bodies", {"body_start": [0]})])
def test_group_refuses_tree_arguments(method, kw):
    g, lib, _, _ = _group()
    with pytest.raises(capi.CtmrError):
        getattr(g, method)(None, **kw)
    assert lib.calls == []
