"""Host-side mirror of the reference interface for the CT map/reduce path, over the C ABI.

The reference is Go (no toolchain in this image), so this module plays the part the Go shim plays
in production (INTEGRATION.md): it packs batches, calls libctmr through the very same C entry
points, and exposes the results under the reference's names:

    GpuCertDatabase.store_batch        <- insertCTWorker loop body + FilesystemDatabase.Store
                                          (cmd/ct-fetch/ct-fetch.go:191-245, storage/filesystemdatabase.go:158-211)
    GpuCertDatabase.get_known_certificates(exp_hour, issuer).count()
                                       <- KnownCertificates.Count (storage/knowncertificates.go:57-63)
    GpuCertDatabase.issuer_counts      <- the per-issuer sum of cmd/storage-statistics/storage-statistics.go:44-53
    GpuCertDatabase.status_counters    <- metrics certIsFilteredOut.{CA,expired,cn-filtered}, insertCTWorker.Inserted
    GpuCertDatabase.revoked_known      <- the join CRLite makes of an issuer's CRLs (crl::<issuer>) with its
                                          serials::<expDate>::<issuer> sets (storage/knowncertificates.go:28-55)
    GpuCertDatabase.revoked_cascade    <- CRLite's filter cascade of the covered issuers' revoked and valid known
                                          certificates, built on the GPU next to the table
    GpuCertDatabase.revoked_stash      <- CRLite's stash: the revoked known certificates a published filter and the
                                          stashes since it miss
    GpuCertDatabase.revoked_verify     <- filter-cascade's verify(include, exclude) of a published filter and its
                                          stashes, with the table's revoked and valid known certificates

All arithmetic happens in the CUDA kernels; nothing here parses, hashes or de-duplicates.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import hashlib
from dataclasses import dataclass

import numpy as np

from . import capi
from .capi import CtmrError


@dataclass
class BatchResult:
    """Per-entry outputs of one batch (numpy arrays in host memory)."""
    status: np.ndarray
    sha256: np.ndarray | None
    exp_hour: np.ndarray
    serial_off: np.ndarray
    serial_len: np.ndarray
    was_unknown: np.ndarray
    first_issuer_hour: np.ndarray
    # IssuerMetadata string reducers (only filled by store_batch(..., want_meta=True))
    issuer_name_off: np.ndarray | None = None
    issuer_name_len: np.ndarray | None = None
    crldp_off: np.ndarray | None = None
    crldp_len: np.ndarray | None = None
    first_issuer_dn: np.ndarray | None = None
    first_crldp: np.ndarray | None = None
    # PEM of the new certificates (want_pem=True): texts back to back, entry i = pem[pem_off[i]:pem_off[i+1]]
    pem: np.ndarray | None = None
    pem_off: np.ndarray | None = None

    def pem_of(self, i: int) -> bytes:
        return self.pem[int(self.pem_off[i]):int(self.pem_off[i + 1])].tobytes()


class KnownCertificatesView:
    """Read side of storage.KnownCertificates for one (expDate, issuer) (knowncertificates.go:57-63), on a ctx or a
    group."""

    def __init__(self, db: "GpuCertDatabase", exp_hour: int, issuer_digest: bytes):
        self._db, self.exp_hour, self.issuer_digest = db, int(exp_hour), bytes(issuer_digest)

    def count(self) -> int:
        out = C.c_uint64(0)
        d = (C.c_uint8 * 32).from_buffer_copy(self.issuer_digest)
        self._db._check(self._db._c("set_cardinality")(self._db._h, self.exp_hour, d, C.byref(out)))
        return out.value


@dataclass
class LogTree:
    """The RFC 6962 Merkle tree over the first `size` entries of one log, held as its right edge (ctmr_tree): edge[k] is
    the root of a complete subtree of 2^k leaves for every bit k set in size.  Pass it as tree= to store_raw_entries /
    store_tiles; the result's .tree is the tree after the batch, and .root is what the log's signed tree head of that
    size must carry."""
    size: int = 0
    edge: np.ndarray | None = None   # [64][32] uint8
    root: bytes = b""

    def to_c(self) -> "capi.Tree":
        t = capi.Tree()
        t.size = int(self.size)
        if self.edge is not None:
            C.memmove(t.edge, np.ascontiguousarray(self.edge, np.uint8).tobytes(), 64 * 32)
        return t

    @classmethod
    def from_c(cls, t: "capi.Tree") -> "LogTree":
        return cls(int(t.size), np.frombuffer(bytes(t.edge), np.uint8).reshape(64, 32).copy(), bytes(t.root))


def _trees_to_c(trees):
    """[LogTree] -> a ctmr_tree array"""
    arr = (capi.Tree * max(len(trees), 1))()
    for d, t in enumerate(trees):
        arr[d] = t.to_c()
    return arr


def _log_ids(log, n: int, what: str) -> np.ndarray:
    log = np.ascontiguousarray(log, np.uint32)
    if log.shape != (n,):
        raise CtmrError(capi.E_INVALID, f"{what} must hold one log id per {'entry' if what == 'entry_log' else 'tile'}")
    return log


def _tree_args(tree, trees, log, name):
    if tree is not None and trees is not None:
        raise CtmrError(capi.E_INVALID, "pass tree= (one log) or trees= (one per log), not both")
    if trees is None and log is not None:
        raise CtmrError(capi.E_INVALID, f"{name} goes with trees=")
    if trees is not None and log is None:
        raise CtmrError(capi.E_INVALID, f"trees= needs {name}")


def _pack(ders):
    offsets = np.zeros(len(ders) + 1, np.uint64)
    offsets[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
    return np.frombuffer(b"".join(ders) or b"\0", np.uint8).copy(), offsets


def _config(table_capacity: int, issuer_cn_filter: bytes | str, log_expired_entries: bool, flags: int, max_issuers: int,
            max_batch_entries: int, max_batch_bytes: int, pair_capacity_log2: int, meta_capacity_log2: int,
            max_round_entries: int = 0, device: int = 0) -> "capi.Config":
    """ctmr_config of a ctx or a group (whose create sets each member's device)"""
    if isinstance(issuer_cn_filter, str):
        issuer_cn_filter = issuer_cn_filter.encode()
    cfg = capi.Config()
    cfg.struct_size = C.sizeof(capi.Config)
    cfg.device = device
    cfg.table_capacity, cfg.max_batch_entries, cfg.max_batch_bytes = table_capacity, max_batch_entries, max_batch_bytes
    cfg.max_issuers, cfg.pair_capacity_log2, cfg.meta_capacity_log2 = max_issuers, pair_capacity_log2, meta_capacity_log2
    cfg.max_round_entries = max_round_entries
    cfg.issuer_cn_filter = bytes(issuer_cn_filter)
    cfg.issuer_cn_filter_len = len(issuer_cn_filter)
    cfg.log_expired_entries, cfg.flags = int(bool(log_expired_entries)), flags
    return cfg


def _at(a, e0: int = 0, per: int = 1):
    """address of row e0 of a (rows of `per` elements), or None"""
    return None if a is None else capi.ptr(a) + e0 * per * a.itemsize


def _path_out(p: BatchResult, want_sha: bool, want_meta: bool, e0: int = 0) -> "capi.Out":
    """ctmr_out over p's arrays from entry e0 on: sha256 with want_sha, the string-identity arrays with want_meta"""
    meta = [_at(p.issuer_name_off, e0), _at(p.issuer_name_len, e0), _at(p.crldp_off, e0), _at(p.crldp_len, e0),
            _at(p.first_issuer_dn, e0), _at(p.first_crldp, e0)] if want_meta else [None] * 6
    return capi.Out(_at(p.status, e0), _at(p.sha256, e0, 32) if want_sha else None, _at(p.exp_hour, e0), _at(p.serial_off, e0),
                    _at(p.serial_len, e0), _at(p.was_unknown, e0), _at(p.first_issuer_hour, e0), *meta)


def _attach_pem(o: "capi.Out", res: BatchResult, n: int, der_bytes: int):
    """Room for the PEM of every certificate of the batch (the worst case: all new)."""
    res.pem = np.zeros(der_bytes // 3 * 4 + der_bytes // 48 + 64 * n + 256, np.uint8)
    res.pem_off = np.zeros(n + 1, np.uint64)
    o.pem, o.pem_cap, o.pem_off = capi.ptr(res.pem), res.pem.size, capi.ptr(res.pem_off)


class RawBatchResult:
    """Outputs of ctmr_process_raw (ctmr_raw_out): the path's outputs plus what the wire format carried."""

    def __init__(self, n: int, want_sha: bool = True, want_meta: bool = False):
        self.path = BatchResult(np.zeros(n, np.uint8), np.zeros((n, 32), np.uint8) if want_sha else None, np.zeros(n, np.int64),
                                np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint8), np.zeros(n, np.uint8))
        if want_meta:
            p = self.path
            p.issuer_name_off, p.issuer_name_len = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
            p.crldp_off, p.crldp_len = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
            p.first_issuer_dn, p.first_crldp = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        self.entry_status = np.zeros(n, np.uint8)
        self.entry_type = np.zeros(n, np.uint8)
        self.timestamp_ms = np.zeros(n, np.uint64)
        self.issuer = np.zeros(n, np.uint32)
        self.leaf_src = np.zeros(n, np.uint8)
        self.leaf_off = np.zeros(n, np.uint32)
        self.leaf_len = np.zeros(n, np.uint32)
        self.tree = None    # LogTree after the batch, when the call was given one
        self.trees = None   # [LogTree] after the batch, when the call was given trees= (one per log)


class BodiesResult(RawBatchResult):
    """Outputs of ctmr_process_raw_bodies (ctmr_body_out): per entry found, what ctmr_process_raw gives plus where its
    strings lie in the text; per body, its status and its entries."""

    def __init__(self, cap: int, n_bodies: int, want_sha: bool = True, want_meta: bool = False):
        super().__init__(cap, want_sha, want_meta)
        self.body_status = np.zeros(n_bodies, np.uint8)
        self.body_first = np.zeros(n_bodies, np.uint64)
        self.body_entries = np.zeros(n_bodies, np.uint32)
        self.leaf_input_off = np.zeros(cap, np.uint64)
        self.leaf_input_len = np.zeros(cap, np.uint32)
        self.extra_data_off = np.zeros(cap, np.uint64)
        self.extra_data_len = np.zeros(cap, np.uint32)
        self.escaped = np.zeros(cap, np.uint8)
        self.n_entries = 0

    def trim(self, n: int):
        """keeps the n entries the call wrote"""
        self.n_entries = n
        p, cap = self.path, self.leaf_input_off.shape[0]
        for obj in (self, p):
            for k, v in list(vars(obj).items()):
                if isinstance(v, np.ndarray) and not k.startswith("body_") and k not in ("pem", "pem_off") and v.shape[:1] == (cap,):
                    setattr(obj, k, v[:n])
        if p.pem_off is not None:
            p.pem_off = p.pem_off[:n + 1]


class TileBatchResult(RawBatchResult):
    """Outputs of ctmr_process_tiles (ctmr_tile_out)."""

    def __init__(self, n: int, n_tiles: int, want_sha: bool = True, want_meta: bool = False, want_leaf_hash: bool = False):
        super().__init__(n, want_sha, want_meta)
        del self.leaf_src
        self.leaf_off = np.zeros(n, np.uint64)
        self.leaf_index = np.zeros(n, np.uint64)
        self.leaf_hash = np.zeros((n, 32), np.uint8) if want_leaf_hash else None
        self.tile_status = np.zeros(n_tiles, np.uint8)
        self.tiles_done = 0
        self.missing = []   # fingerprints (bytes) of the unregistered Chain[0] certificates of tile `tiles_done`


class RevokedResult:
    """Outputs of ctmr_revoked_known (include/ctmr.h ctmr_crl_out): per CRL, and per entry of the listed CRLs.
    serial_len saturates at 255, so serial() of an entry whose serial has 256 or more octets (CTMR_RV_SERIAL_TOO_LONG,
    never joined) returns only its first 255 octets; serial_off is exact."""

    _CRL = (("crl_status", np.uint8), ("crl_flags", np.uint8), ("this_update", np.int64), ("next_update", np.int64),
            ("tbs_off", np.uint64), ("tbs_len", np.uint32), ("issuer_name_off", np.uint64), ("issuer_name_len", np.uint32),
            ("crl_first", np.uint64), ("crl_entries", np.uint32))
    _ENTRY = (("serial_off", np.uint64), ("serial_len", np.uint8), ("revoked_at", np.int64), ("reason", np.uint8),
              ("entry_status", np.uint8), ("known", np.uint8), ("known_exp_hour", np.int64), ("known_sets", np.uint32))

    def __init__(self, n_crls: int, entry_cap: int):
        for name, dt in self._CRL:
            setattr(self, name, np.zeros(n_crls, dt))
        for name, dt in self._ENTRY:
            setattr(self, name, np.zeros(max(entry_cap, 1), dt))
        self.entry_cap = entry_cap
        self.n_entries = 0

    def to_c(self) -> "capi.CrlOut":
        o = capi.CrlOut()
        for name, _ in self._CRL + self._ENTRY:
            setattr(o, name, getattr(self, name).ctypes.data)
        o.entry_cap = self.entry_cap
        return o

    def trim(self, n: int):
        for name, _ in self._ENTRY:
            setattr(self, name, getattr(self, name)[:n])
        self.n_entries = n

    def serial(self, data: np.ndarray, e: int) -> bytes:
        o = int(self.serial_off[e])
        return bytes(data[o:o + int(self.serial_len[e])])


class CascadeResult:
    """Outputs of ctmr_revoked_cascade (include/ctmr.h ctmr_cascade_out): the serialized filter cascade, each CRL's
    status, and the covered issuers, levels and key records in R (revoked) and S (valid)."""

    def __init__(self, data: bytes, crl_status: np.ndarray, o):
        self.bytes = data
        self.crl_status = crl_status
        self.issuers, self.levels, self.revoked, self.valid = int(o.issuers), int(o.levels), int(o.revoked), int(o.valid)


class StashResult:
    """Outputs of ctmr_revoked_stash (include/ctmr.h ctmr_stash_out): the serialized stash, each CRL's status, the
    covered issuers, the issuer units written, the key records in R, those the filter and the earlier stashes already
    answer, and the (issuer, serial) entries written."""

    def __init__(self, data: bytes, crl_status: np.ndarray, o):
        self.bytes = data
        self.crl_status = crl_status
        self.issuers, self.stash_issuers = int(o.issuers), int(o.stash_issuers)
        self.revoked, self.in_filter, self.in_stashes, self.serials = int(o.revoked), int(o.in_filter), int(o.in_stashes), int(o.serials)


MISS_DTYPE = np.dtype([("digest", "u1", 32), ("exp_hour", "<i8"), ("first_index", "<u8"), ("serial_len", "u1"),
                       ("serial", "u1", capi.MAX_SERIAL), ("blocked", "u1"), ("pad", "u1", 7)])   # ctmr_verify_miss


class VerifyResult:
    """Outputs of ctmr_revoked_verify (include/ctmr.h ctmr_verify_out): each CRL's status, the covered issuers, the
    filter's levels, the counts of the records first seen before covered_below (.before) and of the others (.since), each
    a dict of revoked, missed, valid and blocked, and .list, a MISS_DTYPE array of the `before` records answered wrongly
    in the header's order."""

    def __init__(self, crl_status: np.ndarray, o, lst: np.ndarray):
        self.crl_status = crl_status
        self.issuers, self.levels = int(o.issuers), int(o.levels)
        self.before, self.since = ({f: int(getattr(c, f)) for f, _ in capi.VerifyCounts._fields_} for c in (o.before, o.since))
        self.list = lst

    def entries(self) -> list:
        """the list as (digest, serial, exp_hour, first_index, blocked) tuples"""
        return [(r["digest"].tobytes(), r["serial"][:r["serial_len"]].tobytes(), int(r["exp_hour"]), int(r["first_index"]),
                 bool(r["blocked"])) for r in self.list]


def _crl_batch(crls, issuer_digests):
    """(ctmr_crl_batch, the arrays it points into) of a list of DER CRLs or (data, crl_off, crl_len)"""
    if isinstance(crls, tuple):
        data, offs, lens = (np.ascontiguousarray(a) for a in crls)
        data, offs, lens = data.astype(np.uint8, copy=False), offs.astype(np.uint64), lens.astype(np.uint64)
    else:
        data, offs, lens = pack_crls(crls)
    n = len(offs)
    dig = np.frombuffer(b"".join(bytes(d) for d in issuer_digests), np.uint8) if n else np.zeros(32, np.uint8)
    if n and dig.size != 32 * n:
        raise ValueError("one 32-byte issuer digest per CRL")
    b = capi.CrlBatch(capi.ptr(data) if data.size else None, data.size, capi.ptr(offs) if n else None,
                      capi.ptr(lens) if n else None, capi.ptr(dig) if n else None, n)
    return b, (data, offs, lens, dig)


def pack_crls(crls):
    """(data, crl_off, crl_len) of a list of DER CRLs laid back to back."""
    lens = np.array([len(c) for c in crls], np.uint64)
    offs = np.zeros(len(crls), np.uint64)
    if len(crls) > 1:
        offs[1:] = np.cumsum(lens)[:-1]
    data = np.frombuffer(b"".join(bytes(c) for c in crls), np.uint8) if crls else np.zeros(0, np.uint8)
    return data, offs, lens


class GpuCertDatabase:
    """One ctmr_ctx = one GPU's share of the known-certificate state."""

    _peers = False   # attached to peers in other processes (peer_attach): the front end is collective
    _form = "ctmr_"  # prefix of the C entry points that take this handle (a group's: ctmr_group_)

    def __init__(self, device: int = 0, table_capacity: int = 1 << 22, issuer_cn_filter: bytes | str = b"",
                 log_expired_entries: bool = False, flags: int = 0, max_issuers: int = 0, max_batch_entries: int = 0,
                 max_batch_bytes: int = 0, pair_capacity_log2: int = 0, meta_capacity_log2: int = 0, max_round_entries: int = 0,
                 _adopt=None):
        self._lib = capi.load()
        if _adopt is not None:  # a member of a GpuCertGroup: the group owns the handle
            self._h, self.device, self.flags, self._owned = _adopt, device, flags, False
            return
        self._owned = True
        cfg = _config(table_capacity, issuer_cn_filter, log_expired_entries, flags, max_issuers, max_batch_entries,
                      max_batch_bytes, pair_capacity_log2, meta_capacity_log2, max_round_entries, device)
        h = C.c_void_p()
        rc = self._lib.ctmr_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise CtmrError(rc, (self._lib.ctmr_last_error(None) or b"").decode())
        self._h = h
        self.device = device
        self.flags = flags

    # ------------------------------------------------------------------ plumbing
    def _c(self, name: str):
        """the C entry point `name` in this handle's form: ctmr_<name>, or ctmr_group_<name> on a group"""
        return getattr(self._lib, self._form + name)

    @property
    def _registry(self) -> "GpuCertDatabase":
        """the ctx whose handle reaches the issuer registry: this one (a group's member 0)"""
        return self

    def _check(self, rc: int):
        if rc != 0:
            raise CtmrError(rc, (self._c("last_error")(self._h) or b"").decode())

    def close(self):
        if getattr(self, "_h", None):
            if getattr(self, "_owned", True):
                self._lib.ctmr_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    @property
    def handle(self):
        return self._h

    # ------------------------------------------------------------------ issuers
    def register_issuers(self, issuer_blob: np.ndarray, issuer_offsets: np.ndarray) -> np.ndarray:
        """NewIssuer(x509.ParseCertificate(Chain[0])) for each certificate -> dense indices."""
        issuer_blob = np.ascontiguousarray(issuer_blob, np.uint8)
        issuer_offsets = np.ascontiguousarray(issuer_offsets, np.uint64)
        n = issuer_offsets.size - 1
        out = np.zeros(max(n, 1), np.uint32)
        reg = self._registry
        reg._check(self._lib.ctmr_register_issuers(reg._h, capi.ptr(issuer_blob), capi.ptr(issuer_offsets), n, capi.ptr(out)))
        return out[:n]

    def issuer_digest(self, dense_idx: int) -> bytes:
        d = (C.c_uint8 * 32)()
        reg = self._registry
        reg._check(self._lib.ctmr_issuer_digest(reg._h, dense_idx, d))
        return bytes(d)

    # ------------------------------------------------------------------ the hot path, host buffers
    def store_batch(self, blob, offsets, issuer_blob, issuer_offsets, issuer_idx, now_unix_ns: int,
                    want_sha: bool = True, out: BatchResult | None = None, want_meta: bool = False,
                    want_pem: bool = False) -> BatchResult:
        """One batch through ctmr_process_batch (HOST buffers in, HOST buffers out)."""
        blob = np.ascontiguousarray(blob, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        n = offsets.size - 1
        n_iss = 0
        if issuer_offsets is not None:
            issuer_blob = np.ascontiguousarray(issuer_blob, np.uint8)
            issuer_offsets = np.ascontiguousarray(issuer_offsets, np.uint64)
            n_iss = issuer_offsets.size - 1
        if issuer_idx is not None:
            issuer_idx = np.ascontiguousarray(issuer_idx, np.uint32)
        if out is None:
            out = BatchResult(np.zeros(n, np.uint8), np.zeros((n, 32), np.uint8) if want_sha else None, np.zeros(n, np.int64),
                              np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint8), np.zeros(n, np.uint8))
        if want_meta and out.first_issuer_dn is None:
            out.issuer_name_off, out.issuer_name_len = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
            out.crldp_off, out.crldp_len = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
            out.first_issuer_dn, out.first_crldp = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        o = _path_out(out, want_sha, want_meta)
        if want_pem:
            _attach_pem(o, out, n, int(blob.size))
        self._check(self._c("process_batch")(self._h, capi.ptr(blob), capi.ptr(offsets), n,
                                             capi.ptr(issuer_blob) if n_iss else None,
                                             capi.ptr(issuer_offsets) if n_iss else None, n_iss,
                                             capi.ptr(issuer_idx), now_unix_ns, C.byref(o)))
        return out

    # ------------------------------------------------------------------ CT wire-format front end (include/ctmr_frontend.h)
    def store_raw_entries(self, text, leaf_off, leaf_len, extra_off, extra_len, now_unix_ns: int, want_sha: bool = True,
                          want_meta: bool = False, want_pem: bool = False, tree: LogTree | None = None, trees=None,
                          entry_log=None) -> "RawBatchResult":
        """get-entries strings (base64 leaf_input / extra_data, spans into `text`) through ctmr_process_raw:
        what GetRawEntries' JSON decode, ct.LogEntryFromLeaf (ct-fetch.go:424,452) and insertCTWorker + Store do.
        With tree= (the log's entries before these), ctmr_process_raw_tree also folds the entries into it: r.tree.
        With trees= (one LogTree per log) and entry_log= (the log of each entry, capi.NO_TREE for none),
        ctmr_process_raw_trees folds each entry into its log's tree: r.trees.
        On a db attached to peers the call is collective; when another rank's tiles stopped (peer_frontend_stopped()),
        every rank calls again until none is left, this one with an empty batch if it has nothing to add."""
        with self._peer_refusal():
            _tree_args(tree, trees, entry_log, "entry_log")
            text = np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray, memoryview)) else np.ascontiguousarray(text, np.uint8)
            leaf_off, extra_off = np.ascontiguousarray(leaf_off, np.uint64), np.ascontiguousarray(extra_off, np.uint64)
            leaf_len, extra_len = np.ascontiguousarray(leaf_len, np.uint32), np.ascontiguousarray(extra_len, np.uint32)
            n = leaf_off.size
            log = _log_ids(entry_log, n, "entry_log") if trees is not None else None
        r = RawBatchResult(n, want_sha, want_meta)
        p = r.path
        o = capi.RawOut()
        o.path = _path_out(p, want_sha, want_meta)
        for name in ("entry_status", "entry_type", "timestamp_ms", "issuer", "leaf_src", "leaf_off", "leaf_len"):
            setattr(o, name, capi.ptr(getattr(r, name)))
        if want_pem:
            _attach_pem(o.path, p, n, (int(leaf_len.sum()) + int(extra_len.sum())) // 4 * 3)
        b = capi.RawBatch(capi.ptr(text), text.size, capi.ptr(leaf_off), capi.ptr(leaf_len), capi.ptr(extra_off), capi.ptr(extra_len),
                          n, now_unix_ns)
        if trees is not None:
            arr = _trees_to_c(trees)
            self._check(self._c("process_raw_trees")(self._h, C.byref(b), C.byref(o), capi.ptr(log) if n else None,
                                                     arr if trees else None, len(trees)))
            r.trees = [LogTree.from_c(arr[d]) for d in range(len(trees))]
            return r
        if tree is None:
            self._check(self._c("process_raw")(self._h, C.byref(b), C.byref(o)))
            return r
        ct = tree.to_c()
        self._check(self._c("process_raw_tree")(self._h, C.byref(b), C.byref(o), C.byref(ct)))
        r.tree = LogTree.from_c(ct)
        return r

    def store_raw_bodies(self, text, body_off, body_len, body_max, now_unix_ns: int, want_sha: bool = True, want_meta: bool = False,
                         want_pem: bool = False, tree: LogTree | None = None, trees=None, body_log=None,
                         body_start=None) -> "BodiesResult":
        """Whole get-entries response bodies (body b is text[body_off[b]:body_off[b] + body_len[b]], body_max[b] the entries
        requested) through ctmr_process_raw_bodies: the GPU finds the entries with encoding/json's rules, then does what
        store_raw_entries does with them.  The per-entry arrays of the result hold the n_entries entries found, in (body,
        position) order; r.body_status / r.body_first / r.body_entries say which are whose.
        With body_start= (the start of the get-entries request each body answers) and tree= (the log's entries before
        these), ctmr_process_raw_bodies_tree also folds the entries into it: r.tree.  With trees= (one LogTree per log) and
        body_log= (the log of each body, capi.NO_TREE for none), ctmr_process_raw_bodies_trees folds each body's entries
        into its log's tree: r.trees.  A body that is not OK, or a gap between a log's bodies, stops that log's fold;
        entries a body repeats below the tree's end are skipped."""
        with self._peer_refusal():
            _tree_args(tree, trees, body_log, "body_log")
            if body_start is not None and tree is None and trees is None:
                raise CtmrError(capi.E_INVALID, "body_start goes with tree= or trees=")
            text = np.frombuffer(text, np.uint8) if isinstance(text, (bytes, bytearray, memoryview)) else np.ascontiguousarray(text, np.uint8)
            body_off = np.ascontiguousarray(body_off, np.uint64)
            body_len, body_max = np.ascontiguousarray(body_len, np.uint32), np.ascontiguousarray(body_max, np.uint32)
            nb = body_off.size
            start = None if body_start is None else np.ascontiguousarray(body_start, np.uint64)
            log = None if body_log is None else np.ascontiguousarray(body_log, np.uint32)
            if (start is not None and start.shape != (nb,)) or (log is not None and log.shape != (nb,)):
                raise CtmrError(capi.E_INVALID, "body_start and body_log hold one value per body")
        cap = int(body_max.sum())
        r = BodiesResult(cap, nb, want_sha, want_meta)
        p = r.path
        o = capi.BodyOut()
        o.raw.path = _path_out(p, want_sha, want_meta)
        for name in ("entry_status", "entry_type", "timestamp_ms", "issuer", "leaf_src", "leaf_off", "leaf_len"):
            setattr(o.raw, name, capi.ptr(getattr(r, name)))
        for name in ("body_status", "body_first", "body_entries", "leaf_input_off", "leaf_input_len", "extra_data_off",
                     "extra_data_len", "escaped"):
            setattr(o, name, capi.ptr(getattr(r, name)))
        if want_pem:
            _attach_pem(o.raw.path, p, cap, int(body_len.sum()) // 4 * 3)
        b = capi.BodyBatch(capi.ptr(text), text.size, capi.ptr(body_off), capi.ptr(body_len), capi.ptr(body_max), nb, now_unix_ns)
        starts = capi.ptr(start) if start is not None and nb else None
        if trees is not None:
            arr = _trees_to_c(trees)
            self._check(self._c("process_raw_bodies_trees")(self._h, C.byref(b), C.byref(o), capi.ptr(log) if log is not None and nb else None,
                                                            starts, arr if trees else None, len(trees)))
            r.trees = [LogTree.from_c(arr[d]) for d in range(len(trees))]
        elif tree is not None:
            ct = tree.to_c()
            self._check(self._c("process_raw_bodies_tree")(self._h, C.byref(b), C.byref(o), starts, C.byref(ct)))
            r.tree = LogTree.from_c(ct)
        else:
            self._check(self._c("process_raw_bodies")(self._h, C.byref(b), C.byref(o)))
        r.trim(int(o.n_entries))
        return r

    def bodies_profile_last(self) -> float:
        """Milliseconds of the JSON kernels in the last store_raw_bodies call, part of frontend_ms."""
        a = C.c_float(0)
        self._check(self._lib.ctmr_bodies_profile_last(self._h, C.byref(a)))
        return a.value

    # ------------------------------------------------------------------ static-ct-api data tiles (include/ctmr_frontend.h)
    def register_chain_certs(self, blob, offsets):
        """Chain certificates -> (dense issuer indices, SHA-256 fingerprints [n][32]); the fingerprints become known to
        store_tiles."""
        blob = np.ascontiguousarray(blob, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        n = offsets.size - 1
        dense = np.zeros(max(n, 1), np.uint32)
        fps = np.zeros((max(n, 1), 32), np.uint8)
        self._check(self._c("register_chain_certs")(self._h, capi.ptr(blob) if blob.size else None, capi.ptr(offsets), n,
                                                    capi.ptr(dense), capi.ptr(fps)))
        return dense[:n], fps[:n]

    def store_tiles(self, data, tile_off, tile_len, tile_index, tile_width, now_unix_ns: int, want_sha: bool = True,
                    want_meta: bool = False, want_pem: bool = False, want_leaf_hash: bool = False, missing_cap: int = 256,
                    fetch=None, tree: LogTree | None = None, trees=None, tile_log=None) -> "TileBatchResult":
        """static-ct-api data tiles through ctmr_process_tiles.  Without `fetch`, a tile naming an unregistered Chain[0]
        stops the call: the result has tiles_done < n_tiles and the missing fingerprints.  With fetch(fingerprints) ->
        DERs, those certificates are registered and the call resumes from there until every tile is done.  With tree= (the
        log's entries before these; consecutive tiles of that log), ctmr_process_tiles_tree also folds the entries into
        it and every resumed call carries it on: r.tree.  With trees= (one LogTree per log) and tile_log= (the log of each
        tile, capi.NO_TREE for none), ctmr_process_tiles_trees folds each tile into its log's tree: r.trees; a resumed
        call carries the trees on, and passes as NO_TREE the rest of a log whose fold a bad tile stopped.
        On a db attached to peers every call is collective: with fetch, this rank keeps calling while any rank stopped
        (peer_frontend_stopped()), with an empty batch once its own tiles are done or its own call failed."""
        with self._peer_refusal():
            _tree_args(tree, trees, tile_log, "tile_log")
            data = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.ascontiguousarray(data, np.uint8)
            tile_off, tile_index = np.ascontiguousarray(tile_off, np.uint64), np.ascontiguousarray(tile_index, np.uint64)
            tile_len, tile_width = np.ascontiguousarray(tile_len, np.uint32), np.ascontiguousarray(tile_width, np.uint16)
            nt = tile_off.size
            if trees is not None:
                tlog = _log_ids(tile_log, nt, "tile_log").copy()
        ent = np.zeros(nt + 1, np.int64)
        ent[1:] = np.cumsum(tile_width.astype(np.int64))
        n = int(ent[-1])
        r = TileBatchResult(n, nt, want_sha, want_meta, want_leaf_hash)
        p = r.path
        if want_pem:
            _attach_pem(capi.Out(), p, n, int(tile_len.astype(np.int64).sum()))
        miss = np.zeros((max(missing_cap, 1), 32), np.uint8)
        ct = tree.to_c() if tree is not None else None
        if trees is not None:
            arr = _trees_to_c(trees)
        t0, pem_base = 0, 0
        while True:
            e0 = int(ent[t0])
            o = capi.TileOut()
            o.path = _path_out(p, want_sha, want_meta, e0)
            if want_pem:
                o.path.pem, o.path.pem_cap, o.path.pem_off = capi.ptr(p.pem) + pem_base, p.pem.size - pem_base, _at(p.pem_off, e0)
            for name in ("entry_status", "entry_type", "timestamp_ms", "issuer", "leaf_index", "leaf_off", "leaf_len"):
                setattr(o, name, _at(getattr(r, name), e0))
            o.leaf_hash = _at(r.leaf_hash, e0, 32)
            o.tile_status = capi.ptr(r.tile_status) + t0
            o.missing_fp, o.missing_cap = capi.ptr(miss), missing_cap
            b = capi.TileBatch(capi.ptr(data), data.size, capi.ptr(tile_off) + 8 * t0, capi.ptr(tile_len) + 4 * t0,
                               capi.ptr(tile_index) + 8 * t0, capi.ptr(tile_width) + 2 * t0, nt - t0, now_unix_ns)
            if ct is not None and 0 < t0 < nt and ct.size < 256 * int(tile_index[t0]):
                ct = None  # a bad tile among the completed tiles stopped the fold: r.tree is final, the rest runs plain
            if trees is not None:
                if t0 > 0:  # a log whose tree stopped below its first tile of the rest: a bad tile stopped its fold
                    for d in range(len(trees)):
                        rest = np.flatnonzero(tlog[t0:] == d)
                        if rest.size and arr[d].size < 256 * int(tile_index[t0 + rest[0]]):
                            tlog[t0 + rest] = capi.NO_TREE
                rc = self._c("process_tiles_trees")(self._h, C.byref(b), C.byref(o), capi.ptr(tlog) + 4 * t0 if nt else None,
                                                    arr if trees else None, len(trees))
                if rc in (0, capi.E_UNKNOWN_ISSUER):
                    r.trees = [LogTree.from_c(arr[d]) for d in range(len(trees))]
            elif ct is None:
                rc = self._c("process_tiles")(self._h, C.byref(b), C.byref(o))
            else:  # written back on success and at the stop: the resumed call continues this tree
                rc = self._c("process_tiles_tree")(self._h, C.byref(b), C.byref(o), C.byref(ct))
                if rc in (0, capi.E_UNKNOWN_ISSUER):
                    r.tree = LogTree.from_c(ct)
            done = int(o.tiles_done)
            if want_pem:
                e1 = int(ent[t0 + done])
                p.pem_off[e0:e1 + 1] += pem_base
                pem_base = int(p.pem_off[e1])
            t0 += done
            r.tiles_done = t0
            r.missing = [miss[k].tobytes() for k in range(o.n_missing)] if rc == capi.E_UNKNOWN_ISSUER else []
            if rc != capi.E_UNKNOWN_ISSUER:
                if rc and fetch is not None:   # the others' resumed calls wait for this rank too
                    err = CtmrError(rc, (self._c("last_error")(self._h) or b"").decode())
                    self._join_resumes()
                    raise err
                self._check(rc)
                if fetch is None or not self._peers or not self.peer_frontend_stopped():
                    return r
                continue   # another rank stopped: this rank joins its resumed call with what it has left (nothing)
            if fetch is None:
                return r
            with self._peer_refusal():   # a rank that gives up here still meets the others' resumed call
                ders = [bytes(d) for d in fetch(r.missing)]
                # a log that serves the wrong bytes at issuer/<hex> would otherwise stop at this tile for ever
                got = [hashlib.sha256(d).digest() for d in ders]
                if set(got) != set(r.missing):
                    raise CtmrError(capi.E_UNKNOWN_ISSUER, "fetch returned certificates whose SHA-256 does not match the missing "
                                    "fingerprints of tile %d" % t0)
                self.register_chain_certs(*_pack(ders))


    def tiles_profile_last(self) -> float:
        """Milliseconds of tile_split (the serial per-tile walk) in the last store_tiles call, part of frontend_ms."""
        a = C.c_float(0)
        self._check(self._lib.ctmr_tiles_profile_last(self._h, C.byref(a)))
        return a.value

    def frontend_profile_last(self):
        """(frontend_ms, path_ms, frontend_launches) of the last store_raw_entries call (CUDA events inside the library)."""
        a, b, k = C.c_float(0), C.c_float(0), C.c_uint64(0)
        self._check(self._lib.ctmr_frontend_profile_last(self._h, C.byref(a), C.byref(b), C.byref(k)))
        return a.value, b.value, k.value

    # ------------------------------------------------------------------ device-resident variants (torch tensors / raw pointers)
    def map_device(self, batch: capi.DevBatch, out: capi.DevOut, stream=None):
        self._check(self._lib.ctmr_map_device(self._h, C.byref(batch), C.byref(out), stream))

    def reduce_device(self, keys, m: int, was_unknown, first_issuer_hour, stream=None):
        self._check(self._lib.ctmr_reduce_device(self._h, capi.ptr(keys), m, capi.ptr(was_unknown),
                                                 capi.ptr(first_issuer_hour), stream))

    def process_device(self, batch: capi.DevBatch, out: capi.DevOut, stream=None):
        self._check(self._lib.ctmr_process_device(self._h, C.byref(batch), C.byref(out), stream))

    def read_histogram_device(self, counts_dst, n_slots: int, status_dst=None, stream=None):
        self._check(self._lib.ctmr_read_histogram_device(self._h, capi.ptr(counts_dst), n_slots, capi.ptr(status_dst), stream))

    def profile_last(self):
        """(map_ms, total_ms) of the last process_device call, from the library's own CUDA events."""
        m, t = C.c_float(0), C.c_float(0)
        self._check(self._lib.ctmr_profile_last(self._h, C.byref(m), C.byref(t)))
        return m.value, t.value

    def sha256_ceiling(self, iters=2000, rolled=True, ctas_per_sm=2):
        """Register-only SHA-256 rate on this GPU: (GB/s of message bytes, ms)."""
        ms, blocks = C.c_float(0), C.c_uint64(0)
        self._check(self._lib.ctmr_sha256_ceiling_device(self._h, iters, int(rolled), ctas_per_sm, C.byref(ms), C.byref(blocks)))
        return blocks.value * 64 / (ms.value / 1e3) / 1e9, ms.value

    def reset_device(self, stream=None):
        self._check(self._lib.ctmr_reset_device(self._h, stream))

    def check_device(self, stream=None):
        self._check(self._lib.ctmr_check_device(self._h, stream))

    # ------------------------------------------------------------------ one process per GPU: peers over CUDA IPC (ctmr_peer_*)
    def peer_export(self, world: int) -> bytes:
        h = (C.c_uint8 * capi.PEER_HANDLE_BYTES)()
        self._check(self._lib.ctmr_peer_export(self._h, world, h))
        return bytes(h)

    def peer_attach(self, rank: int, world: int, handles: list):
        """handles[r] = rank r's peer_export().  Afterwards process_device / store_batch / reset_device and the front end
        (store_raw_entries, store_tiles, with or without trees), checkpoint / load_checkpoint and revoked_known are
        collective."""
        buf = (C.c_uint8 * (capi.PEER_HANDLE_BYTES * world)).from_buffer_copy(b"".join(handles))
        self._check(self._lib.ctmr_peer_attach(self._h, rank, world, buf))
        self._peers = world > 1

    def peer_frontend_stopped(self) -> int:
        """Ranks that stopped at an unknown Chain[0] fingerprint in the last collective store_raw_entries / store_tiles
        call: a resume loop calls again on every rank while this is non-zero."""
        n = C.c_uint32(0)
        self._check(self._lib.ctmr_peer_frontend_stopped(self._h, C.byref(n)))
        return n.value

    def next_index(self) -> int:
        """The global index the next host-buffer or front-end call on this ctx starts at (ctmr_next_index)."""
        n = C.c_uint64(0)
        self._check(self._lib.ctmr_next_index(self._h, C.byref(n)))
        return n.value

    @contextlib.contextmanager
    def _peer_refusal(self, call=None):
        """On a db attached to peers the front end and revoked_known are collective: a rank that gives up on a call
        before making it (an argument its binding refuses, a failed fetch) still makes it with no batch, so that the other
        ranks return CTMR_E_PEER_FAILED instead of waiting at a barrier.  `call` makes that call (default: the front
        end's ctmr_process_raw)."""
        try:
            yield
        except Exception:
            if self._peers:
                if call is None:
                    self._lib.ctmr_process_raw(self._h, None, None)
                else:
                    call()
            raise

    def _join_resumes(self):
        """A rank whose own collective call failed joins, with an empty batch, the calls that resume other ranks' stops."""
        while self._peers and self.peer_frontend_stopped():
            if self._lib.ctmr_process_tiles(self._h, C.byref(capi.TileBatch()), C.byref(capi.TileOut())) != 0:
                return

    def peer_barrier_device(self, stream=None):
        self._check(self._lib.ctmr_peer_barrier_device(self._h, stream))

    def peer_allreduce_histogram_device(self, counts_dst, n_slots: int, status_dst=None, stream=None):
        self._check(self._lib.ctmr_peer_allreduce_histogram_device(self._h, capi.ptr(counts_dst), n_slots, capi.ptr(status_dst), stream))

    # ------------------------------------------------------------------ warm start / checkpoint (SURVEY §8(f)-4)
    def preload_known(self, exp_hour: int, issuer_digest: bytes, serials):
        """Seed one "serials::<expDate>::<issuer>" set (e.g. KnownCertificates.Known() read back from Redis)."""
        serials = [bytes(x) for x in serials]
        blob, offs = _pack(serials)
        d = (C.c_uint8 * 32).from_buffer_copy(issuer_digest)
        self._check(self._c("preload_known")(self._h, exp_hour, d, capi.ptr(blob), capi.ptr(offs), len(serials)))

    def snapshot(self) -> np.ndarray:
        need = C.c_uint64(0)
        self._check(self._c("snapshot_size")(self._h, C.byref(need)))
        buf = np.empty(need.value, np.uint8)
        wrote = C.c_uint64(0)
        self._check(self._c("snapshot_save")(self._h, capi.ptr(buf), buf.size, C.byref(wrote)))
        return buf[:wrote.value]

    def restore(self, snap: np.ndarray):
        snap = np.ascontiguousarray(snap, np.uint8)
        self._check(self._c("snapshot_load")(self._h, capi.ptr(snap), snap.size))

    def revoked_known(self, crls, issuer_digests, entry_cap: int | None = None) -> RevokedResult:
        """Which revoked serials of these CRLs are known certificates (ctmr_revoked_known).  `crls`: a list of DER CRLs,
        or (data, crl_off, crl_len); `issuer_digests`: per CRL the 32-byte Issuer.ID() digest whose crl:: set named it.
        Read-only.  entry_cap defaults to the bound that always suffices (total bytes // 18).  An empty list of CRLs
        (and of digests) returns an empty result.
        On a db attached to peers the call is collective: every rank calls it with its own CRLs (an empty list will do)
        and gets the answers for its own CRLs against every rank's shard.  A rank whose arguments are refused here
        still makes the call, with no batch, so that the other ranks return CTMR_E_PEER_FAILED, and then raises."""
        with self._peer_refusal(lambda: self._c("revoked_known")(self._h, None, None)):
            b, keep = _crl_batch(crls, issuer_digests)
            lens = keep[2]
            cap = int(lens.sum()) // capi.CRL_MIN_ENTRY if entry_cap is None else int(entry_cap)
            res = RevokedResult(int(b.n_crls), cap)
            o = res.to_c()
        rc = self._c("revoked_known")(self._h, C.byref(b), C.byref(o))
        res.n_entries = int(o.n_entries)
        try:
            self._check(rc)
        except CtmrError as e:
            e.n_entries = res.n_entries  # CTMR_E_BATCH_TOO_LARGE: the entry_cap that suffices
            raise
        res.trim(int(o.n_entries))
        return res

    _cascade_bytes = 0   # size of the last cascade this db built: the next call's first buffer holds twice that

    def revoked_cascade(self, crls, issuer_digests, now_unix_sec: int, salt: bytes = b"", cap: int | None = None) -> CascadeResult:
        """CRLite's filter cascade (ctmr_revoked_cascade): it includes the live known certificates of the covered issuers
        that these CRLs revoke and excludes every other live known certificate of those issuers.  An issuer is covered
        when it is registered and every one of its CRLs here parses (CRL_OK).  `crls` and `issuer_digests` as for
        revoked_known; `salt`: at most 32 bytes.  Read-only.  Returns .bytes (the serialized cascade), .crl_status,
        .issuers, .levels, .revoked and .valid.
        The output buffer holds `cap` bytes; by default 16 MiB, or twice the last cascade this db built if that is more.
        A cascade larger than the buffer is built twice: the first build only reports its size (the library writes
        nothing else when the buffer is too small), the second fills a buffer of that size.
        On a db attached to peers the call is collective: every rank calls it with its own CRLs (an empty list will do) and
        the same now_unix_sec and salt, and every rank gets the cascade of every rank's shard and every rank's CRLs, as
        one db holding all the shards would build it from the ranks' CRLs in rank order; .crl_status covers the rank's own
        CRLs.  A buffer too small on any rank is too small on every rank, so every rank builds it the second time together.
        A rank whose arguments are refused here still makes the call, with no batch, so that the other ranks return
        CTMR_E_PEER_FAILED, and then raises."""
        fn = self._c("revoked_cascade")
        with self._peer_refusal(lambda: fn(self._h, None, 0, None, 0, None)):
            b, keep = _crl_batch(crls, issuer_digests)
            salt = bytes(salt)
            sbuf = (C.c_uint8 * max(len(salt), 1)).from_buffer_copy(salt or b"\0")
            status = np.zeros(max(int(b.n_crls), 1), np.uint8)
            size = int(cap) if cap is not None else max(16 << 20, 2 * self._cascade_bytes)
            buf = np.empty(max(size, 1), np.uint8)
            o = capi.CascadeOut(capi.ptr(buf), size, 0, capi.ptr(status))
            now_unix_sec = int(now_unix_sec)
        rc = fn(self._h, C.byref(b), now_unix_sec, sbuf, len(salt), C.byref(o))
        if rc == capi.E_BATCH_TOO_LARGE and o.bytes:  # larger than the buffer: again into one of the size it reported
            buf = np.empty(int(o.bytes), np.uint8)
            o = capi.CascadeOut(capi.ptr(buf), buf.size, 0, capi.ptr(status))
            rc = fn(self._h, C.byref(b), now_unix_sec, sbuf, len(salt), C.byref(o))
        self._check(rc)
        self._cascade_bytes = int(o.bytes)
        return CascadeResult(buf[:o.bytes].tobytes(), status[:b.n_crls].copy(), o)

    _stash_bytes = 0   # size of the last stash this db computed: the next call's first buffer holds twice that

    def revoked_stash(self, crls, issuer_digests, now_unix_sec: int, filter: bytes, stashes: bytes = b"",
                      cap: int | None = None) -> StashResult:
        """CRLite's next stash (ctmr_revoked_stash): every (issuer, serial) of the cascade's revoked set R for these CRLs
        and now_unix_sec that the published `filter` answers "not revoked" and that none of `stashes` (every stash
        published since the filter, back to back) lists.  `crls` and `issuer_digests` as for revoked_cascade.  Read-only.
        Returns .bytes (the serialized stash), .crl_status, .issuers, .stash_issuers, .revoked, .in_filter, .in_stashes
        and .serials.  The output buffer holds `cap` bytes; by default 1 MiB, or twice the last stash this db computed if
        that is more.  A larger stash is computed twice: the first call only reports its size.  Not on a db attached to
        peers (CTMR_E_INVALID on every rank)."""
        fn = self._c("revoked_stash")
        b, keep = _crl_batch(crls, issuer_digests)
        filter, stashes = bytes(filter), bytes(stashes)
        fbuf = (C.c_uint8 * max(len(filter), 1)).from_buffer_copy(filter or b"\0")
        sbuf = (C.c_uint8 * max(len(stashes), 1)).from_buffer_copy(stashes or b"\0")
        status = np.zeros(max(int(b.n_crls), 1), np.uint8)
        size = int(cap) if cap is not None else max(1 << 20, 2 * self._stash_bytes)
        buf = np.empty(max(size, 1), np.uint8)
        o = capi.StashOut(capi.ptr(buf), size, 0, capi.ptr(status))
        now_unix_sec = int(now_unix_sec)
        rc = fn(self._h, C.byref(b), now_unix_sec, fbuf, len(filter), sbuf, len(stashes), C.byref(o))
        if rc == capi.E_BATCH_TOO_LARGE and o.bytes:  # larger than the buffer: again into one of the size it reported
            buf = np.empty(int(o.bytes), np.uint8)
            o = capi.StashOut(capi.ptr(buf), buf.size, 0, capi.ptr(status))
            rc = fn(self._h, C.byref(b), now_unix_sec, fbuf, len(filter), sbuf, len(stashes), C.byref(o))
        self._check(rc)
        self._stash_bytes = int(o.bytes)
        return StashResult(buf[:o.bytes].tobytes(), status[:b.n_crls].copy(), o)

    _verify_records = 0   # records the last verify of this db listed: the next call's first list holds twice that

    def revoked_verify(self, crls, issuer_digests, now_unix_sec: int, filter: bytes, stashes: bytes = b"",
                       covered_below: int = 2**64 - 1, cap: int | None = None) -> VerifyResult:
        """A published `filter`, with `stashes` (every stash published since it, back to back), checked against the table
        (ctmr_revoked_verify): every live known certificate of the covered issuers, revoked by these CRLs or not, is queried,
        and counted in .before when it was first seen at a global index below covered_below (ctmr_next_index when the
        filter was built), in .since otherwise.  `crls` and `issuer_digests` as for revoked_cascade.  Read-only.  The list
        holds `cap` records; by default 4096, or twice the last list this db returned if that is more.  A longer list is
        computed twice: the first call only reports its length.
        On a db attached to peers the call is collective: every rank calls it with its own CRLs (an empty list will do) and
        the same now_unix_sec, filter, stashes and covered_below, and every rank gets the same counts and list.  A rank
        whose arguments are refused here still makes the call, with no batch, so that the other ranks return
        CTMR_E_PEER_FAILED, and then raises."""
        fn = self._c("revoked_verify")
        with self._peer_refusal(lambda: fn(self._h, None, 0, None, 0, None, 0, 0, None)):
            b, keep = _crl_batch(crls, issuer_digests)
            filter, stashes = bytes(filter), bytes(stashes)
            fbuf = (C.c_uint8 * max(len(filter), 1)).from_buffer_copy(filter or b"\0")
            sbuf = (C.c_uint8 * max(len(stashes), 1)).from_buffer_copy(stashes or b"\0")
            status = np.zeros(max(int(b.n_crls), 1), np.uint8)
            size = int(cap) if cap is not None else max(4096, 2 * self._verify_records)
            now_unix_sec, covered_below = int(now_unix_sec), int(covered_below)

        def call(n):
            lst = np.zeros(max(n, 1), MISS_DTYPE)
            o = capi.VerifyOut(capi.ptr(status), 0, 0, capi.VerifyCounts(), capi.VerifyCounts(), capi.ptr(lst), n, 0)
            return fn(self._h, C.byref(b), now_unix_sec, fbuf, len(filter), sbuf, len(stashes), covered_below, C.byref(o)), o, lst

        rc, o, lst = call(size)
        if rc == capi.E_BATCH_TOO_LARGE and o.n_list:  # longer than the list: again into one of the length it reported
            rc, o, lst = call(int(o.n_list))
        self._check(rc)
        self._verify_records = int(o.n_list)
        return VerifyResult(status[:b.n_crls].copy(), o, lst[:o.n_list].copy())

    def checkpoint(self) -> np.ndarray:
        """This db's part of a portable checkpoint (ctmr_checkpoint_save): loads into any table size, group size or number
        of ranks.  On a db attached to peers it is collective, and every rank returns its own part."""
        need = C.c_uint64(0)
        self._check(self._c("checkpoint_size")(self._h, C.byref(need)))
        buf = np.empty(max(need.value, 1), np.uint8)
        wrote = C.c_uint64(0)
        self._check(self._c("checkpoint_save")(self._h, capi.ptr(buf), buf.size, C.byref(wrote)))
        return buf[:wrote.value]

    def load_checkpoint(self, parts):
        """Replace the state with a checkpoint: `parts` = every part of it (a list of arrays, any order) or its one part.
        Collective on a db attached to peers."""
        self._parts_call("checkpoint_load", parts)

    def _parts_call(self, name, parts):
        if isinstance(parts, np.ndarray):
            parts = [parts]
        parts = [np.ascontiguousarray(p, np.uint8) for p in parts]
        ptrs = (C.c_void_p * max(len(parts), 1))(*[p.ctypes.data for p in parts])
        sizes = (C.c_uint64 * max(len(parts), 1))(*[p.size for p in parts])
        self._check(self._c(name)(self._h, ptrs, sizes, len(parts)))

    def checkpoint_delta(self, since: int) -> np.ndarray:
        """This db's part of a delta checkpoint (ctmr_checkpoint_delta_save): the records first seen at or above `since`,
        the next index kept with an earlier checkpoint or delta, with the whole registry and the status counters.
        Collective on a db attached to peers."""
        need = C.c_uint64(0)
        self._check(self._c("checkpoint_delta_size")(self._h, int(since), C.byref(need)))
        buf = np.empty(max(need.value, 1), np.uint8)
        wrote = C.c_uint64(0)
        self._check(self._c("checkpoint_delta_save")(self._h, int(since), capi.ptr(buf), buf.size, C.byref(wrote)))
        return buf[:wrote.value]

    def apply_checkpoint_delta(self, parts):
        """Put a delta checkpoint on top of the state (ctmr_checkpoint_apply): `parts` = every part of it (a list of
        arrays, any order) or its one part.  The state must stand at the delta's `since`.  Collective on a db attached
        to peers."""
        self._parts_call("checkpoint_apply", parts)

    def evict_expired(self, now_unix_sec: int) -> int:
        """Apply the Redis TTLs (EXPIREAT(expDate) on every serials:: set, knowncertificates.go:98-104): sets with
        expDate <= now vanish.  Returns the number of serials dropped."""
        n = C.c_uint64(0)
        self._check(self._c("evict_expired")(self._h, int(now_unix_sec), C.byref(n)))
        return int(n.value)

    # ------------------------------------------------------------------ reducers' read side
    def get_known_certificates(self, exp_hour: int, issuer_digest: bytes) -> KnownCertificatesView:
        return KnownCertificatesView(self, exp_hour, issuer_digest)

    def issuer_counts(self) -> dict:
        """{Issuer.ID digest (32 bytes): number of unique certificates} for every registered issuer."""
        n = C.c_size_t(self._lib.ctmr_issuer_count(self._registry._h))
        cap = max(int(n.value), 1)
        dig = np.zeros((cap, 32), np.uint8)
        cnt = np.zeros(cap, np.uint64)
        self._check(self._c("issuer_counts")(self._h, capi.ptr(dig), capi.ptr(cnt), C.byref(n)))
        return {bytes(dig[i]): int(cnt[i]) for i in range(n.value)}

    def status_counters(self) -> np.ndarray:
        out = np.zeros(capi.ST_COUNT, np.uint64)
        self._check(self._c("status_counters")(self._h, capi.ptr(out)))
        return out

    def table_stats(self):
        used, cap = C.c_uint64(0), C.c_uint64(0)
        self._check(self._c("table_stats")(self._h, C.byref(used), C.byref(cap)))
        return used.value, cap.value

    def resize(self, table_capacity: int | None = None, pair_capacity_log2: int | None = None,
               meta_capacity_log2: int | None = None):
        """The known-certificate, (issuer, expDate) and string-identity tables in other sizes, rehashed on the device
        (ctmr_resize): afterwards every call answers as a db created with these capacities and loaded from a checkpoint
        taken just before; the registry, the chain certificates and the fingerprints stay.  None keeps a table's size.
        All or nothing: on failure (E_NOMEM, a *_TABLE_FULL for a target too small) the db is unchanged.  Not on a db
        exported to peers (E_INVALID on every rank, without a collective call)."""
        self._check(self._c("resize")(self._h, int(table_capacity or 0), int(pair_capacity_log2 or 0), int(meta_capacity_log2 or 0)))

    def rollback(self, next_index: int):
        """Take the state back to the start of an earlier entry-taking call (ctmr_rollback): every record first seen at or
        above `next_index` goes, the counts follow the remaining keys, the status counters are those at that call's start
        and the next index is `next_index`.  It must be the next index at the start of one of the last
        capi.ROLLBACK_MARKS batch, front-end, device or preload calls, at or above the last reset or load (E_INVALID
        otherwise, with nothing touched); the current next index does nothing.  The registry and the chain certificates
        stay; restore your trees yourself.  Collective on a db attached to peers."""
        self._check(self._c("rollback")(self._h, int(next_index)))

    def table_occupancy(self):
        """((used known, pair, meta), (capacity known, pair, meta)): live slots and slots of the three tables
        (ctmr_table_occupancy; a group's are sums over its shards)."""
        used, cap = (C.c_uint64 * 3)(), (C.c_uint64 * 3)()
        self._check(self._c("table_occupancy")(self._h, used, cap))
        return tuple(int(v) for v in used), tuple(int(v) for v in cap)


class GpuCertGroup(GpuCertDatabase):
    """Several GPUs of one box behind ONE handle (ctmr_group_*): what the Go host calls in place of the worker pool of
    StartDatabaseThreads (cmd/ct-fetch/ct-fetch.go:140-145).  Same methods, globally exact results: every set
    "serials::<expDate>::<issuer>" lives on one owner GPU and the map kernels insert into it over NVLink."""

    _form = "ctmr_group_"

    def __init__(self, devices, table_capacity: int = 1 << 22, issuer_cn_filter: bytes | str = b"", log_expired_entries: bool = False,
                 flags: int = 0, max_issuers: int = 0, max_batch_entries: int = 0, max_batch_bytes: int = 0,
                 pair_capacity_log2: int = 0, meta_capacity_log2: int = 0):
        self._lib = capi.load()
        cfg = _config(table_capacity, issuer_cn_filter, log_expired_entries, flags, max_issuers, max_batch_entries,
                      max_batch_bytes, pair_capacity_log2, meta_capacity_log2)
        devs = (C.c_int32 * len(devices))(*devices)
        h = C.c_void_p()
        rc = self._lib.ctmr_group_create(C.byref(cfg), devs, len(devices), C.byref(h))
        if rc != 0:
            raise CtmrError(rc, (self._lib.ctmr_group_last_error(None) or b"").decode())
        self._h, self._owned = h, True
        self.devices, self.device, self.flags = list(devices), devices[0], flags
        self.members = [GpuCertDatabase(device=devices[r], flags=flags, _adopt=C.c_void_p(self._lib.ctmr_group_member(h, r)))
                        for r in range(len(devices))]

    @property
    def _registry(self) -> GpuCertDatabase:
        return self.members[0]   # the registry is the group's, in member 0's memory

    def close(self):
        if getattr(self, "_h", None):
            for m in self.members:
                m._h = None
            self._lib.ctmr_group_destroy(self._h)
            self._h = None

    def store_raw_entries(self, *a, tree=None, trees=None, **k):
        if tree is not None or trees is not None:
            raise CtmrError(capi.E_INVALID, "tree= and trees= take one ctx: on a group use store_raw_entries_with_trees")
        return super().store_raw_entries(*a, **k)

    def store_tiles(self, *a, tree=None, trees=None, **k):
        if tree is not None or trees is not None:
            raise CtmrError(capi.E_INVALID, "tree= and trees= take one ctx: on a group use store_tiles_with_trees")
        return super().store_tiles(*a, **k)

    def store_raw_bodies(self, *a, tree=None, trees=None, body_log=None, body_start=None, **k):
        if tree is not None or trees is not None or body_log is not None or body_start is not None:
            raise CtmrError(capi.E_INVALID, "tree= and trees= take one ctx: on a group use store_raw_bodies_with_trees")
        return super().store_raw_bodies(*a, **k)

    def store_raw_bodies_with_trees(self, *a, tree=None, trees=None, body_log=None, body_start=None, **k):
        """store_raw_bodies with tree= or trees= / body_log=, and body_start=, on the group
        (ctmr_group_process_raw_bodies_tree(s)): the same outputs as the plain group call, and r.tree / r.trees as the
        one-ctx call gives them"""
        return GpuCertDatabase.store_raw_bodies(self, *a, tree=tree, trees=trees, body_log=body_log, body_start=body_start, **k)

    def store_raw_entries_with_trees(self, *a, tree=None, trees=None, entry_log=None, **k):
        """store_raw_entries with tree= or trees= / entry_log= on the group (ctmr_group_process_raw_tree(s)): the same
        outputs as the plain group call, and r.tree / r.trees as the one-ctx call gives them"""
        return GpuCertDatabase.store_raw_entries(self, *a, tree=tree, trees=trees, entry_log=entry_log, **k)

    def store_tiles_with_trees(self, *a, fetch=None, tree=None, trees=None, tile_log=None, **k):
        """store_tiles with tree= or trees= / tile_log= on the group (ctmr_group_process_tiles_tree(s)), with the same
        fetch-and-resume loop and per-log resume rule as GpuCertDatabase.store_tiles"""
        return GpuCertDatabase.store_tiles(self, *a, fetch=fetch, tree=tree, trees=trees, tile_log=tile_log, **k)

    def reset(self):
        self._check(self._lib.ctmr_group_reset(self._h))

    def _single_ctx_only(self, *a, **k):
        raise CtmrError(capi.E_INVALID, "this entry point takes one ctx: use group.members[r] (read side) or the group's own methods")

    # the device-resident / per-ctx entry points of the base class do not take a group handle
    map_device = reduce_device = process_device = read_histogram_device = profile_last = sha256_ceiling = _single_ctx_only
    reset_device = check_device = peer_export = peer_attach = peer_barrier_device = _single_ctx_only
    peer_allreduce_histogram_device = frontend_profile_last = tiles_profile_last = _single_ctx_only


# ---------------------------------------------------------------------- synthetic corpus (bench/test tooling)
def synth_issuers(cfg: capi.SynthCfg):
    """DER of the synthetic CA certificates (host side), (blob u8, offsets u64[n_issuers+1])."""
    L = capi.load()
    offsets = np.zeros(cfg.n_issuers + 1, np.uint64)
    total = L.ctmr_synth_issuers_host(C.byref(cfg), capi.ptr(offsets), None, 0)
    blob = np.zeros(total, np.uint8)
    L.ctmr_synth_issuers_host(C.byref(cfg), capi.ptr(offsets), capi.ptr(blob), total)
    return blob, offsets


def synth_corpus_device(cfg: capi.SynthCfg, first: int, n: int, device, want_issuer_idx=True):
    """Generate entries [first, first+n) in HBM: (blob u8, offsets i64-as-u64 [n+1], issuer_idx i32-as-u32 [n])."""
    import torch

    L = capi.load()
    dev = torch.device(device)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream or 1  # 0x1 = cudaStreamLegacy
        offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
        total = C.c_uint64(0)
        rc = L.ctmr_synth_offsets_device(C.byref(cfg), first, n, offsets.data_ptr(), C.byref(total), stream)
        if rc:
            raise CtmrError(rc, "ctmr_synth_offsets_device")
        blob = torch.empty(total.value + 64, dtype=torch.uint8, device=dev)  # readable past the end, 16-byte rounding
        idx = torch.empty(n, dtype=torch.int32, device=dev) if want_issuer_idx else None
        rc = L.ctmr_synth_write_device(C.byref(cfg), first, n, offsets.data_ptr(), blob.data_ptr(),
                                       idx.data_ptr() if idx is not None else None, stream)
        if rc:
            raise CtmrError(rc, "ctmr_synth_write_device")
        torch.cuda.synchronize(dev)
    return blob, offsets, idx, int(total.value)
