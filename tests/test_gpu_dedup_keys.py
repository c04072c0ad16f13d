"""Dedup keys: a certificate's identity in the known-certificate table is (expiry hour, issuer, serial), whichever map
kernel computed it, wherever its entries sit in a call, and however many lanes insert it at once.  Every output is
compared with the oracle, and the table itself is decoded from a snapshot and checked slot by slot (tests/keymodel.py):
tag = restated hash, body = a key some entry produced, first index = that key's lowest entry index, no hole between a
key's home slot and its slot, used slots = distinct keys, pair counts = set cardinalities."""
import numpy as np
import pytest

import der_build as D
import keymodel as K
from conftest import NOW_NS, pack

CA = D.cert(serial=b"\x7f", subject=[[D.cn(b"Dedup CA")]], extensions=[D.basic_constraints(True)])
CA2 = D.cert(serial=b"\x7e", subject=[[D.cn(b"Other CA")]], extensions=[D.basic_constraints(True)],
             spki_bits=b"\x00" + D.tlv(0x30, D.tlv(0x02, b"\x00\xc3" + b"\x22" * 15) + D.tlv(0x02, b"\x01\x00\x01")))  # Issuer.ID = SHA-256 of the SPKI
HOUR = D.exp_hour(D.unix(2030, 6, 15, 12))
POISON = D.Ext(bytes.fromhex("2b06010401d679020403"), b"\x05\x00", critical=True)  # CT precertificate poison


def short_cert(serial, not_after):
    return D.cert(serial=serial, not_after=not_after).der


def long_cert(serial, not_after):
    """The same key as short_cert, other bytes, several 128-byte chunks longer (another length bucket): a precertificate."""
    return D.cert(serial=serial, not_after=not_after, subject=[[D.cn(b"precertificate subject " * 8)]],
                  extensions=[POISON, D.crl_distribution_points(b"http://dedup.example/" + b"p" * 300)], sig_len=512).der


# ------------------------------------------------------------------------------------------------ CPU: the restatement

def test_key_model_restatement():
    a = K.key_body(-5, 3, b"\x01")
    b = K.key_body(-5, 3, b"\x01\x00")
    assert a[:3] == (0xFFFFFFFB, 3, 0x0101) and b[2] == 0x000102 and a != b   # serial_len is part of the key
    bodies = np.array([a, b, K.key_body(HOUR, 0, bytes(range(1, 40)))], np.uint32)
    assert [int(h) for h in K.key_hash_np(bodies)] == [K.key_hash(x) for x in bodies.tolist()]


# ------------------------------------------------------------------------------------------------ GPU helpers

@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


class Both:
    """One GPU database and the oracle fed the same batches; `model` follows the table."""

    def __init__(self, eng, ora, issuers=(CA,), **kw):
        self.db = eng.GpuCertDatabase(log_expired_entries=True, **kw)
        self.odb = ora.DB(b"", True)
        self.iblob, self.ioffs = pack([c.der for c in issuers])
        self.dense = self.db.register_issuers(self.iblob, self.ioffs)
        self.model = K.KeyModel()

    def store(self, ders, idx=None, want_sha=True):
        from test_gpu_parity import assert_same
        blob, offs = pack(ders)
        idx = np.zeros(len(ders), np.uint32) if idx is None else np.asarray(idx, np.uint32)
        want = self.odb.process(blob, offs, self.iblob, self.ioffs, idx, NOW_NS)
        got = self.db.store_batch(blob, offs, self.iblob, self.ioffs, idx, NOW_NS, want_sha=want_sha)
        assert_same(got, want, sha=want_sha)
        self.model.add(blob, offs, want, self.dense[idx])
        return got, want

    def check(self):
        assert {k: v for k, v in self.db.issuer_counts().items() if v} == {k: v for k, v in self.odb.issuer_counts().items() if v}
        for (hour, issuer), n in self.model.pair_counts().items():
            dig = self.db.issuer_digest(issuer)
            hour = hour - (1 << 32) if hour >= 1 << 31 else hour
            assert self.db.get_known_certificates(hour, dig).count() == self.odb.set_cardinality(hour, dig) == n
        return K.check_table(self.db.snapshot(), self.model, self.db.table_stats()[0])

    def close(self):
        self.db.close()


# ------------------------------------------------------------------------------------------------ C.1 cross-kernel identity

def _serial_corpus():
    ders = []
    for n in range(1, 40):
        ders.append(short_cert(D.serial_bytes(n, salt=n), D.NOT_AFTER + n))
        if n >= 2:
            ders.append(short_cert(D.serial_bytes(n, lead00=True, salt=n), D.NOT_AFTER + 7 * n))
    ders.append(short_cert(b"\x00", D.NOT_AFTER))
    return ders


@pytest.mark.gpu
@pytest.mark.parametrize("first_sha", (True, False), ids=("stream_then_light", "light_then_stream"))
def test_cross_kernel_key_identity(eng, ora, first_sha):
    """The same certificates through one kernel, then the other, in one database: every entry of the second batch is
    known, and nothing is counted twice."""
    ders = _serial_corpus()
    b = Both(eng, ora, table_capacity=1 << 12)
    try:
        r1, _ = b.store(ders, want_sha=first_sha)
        assert r1.was_unknown.all()
        counts = b.db.issuer_counts()
        r2, _ = b.store(ders, want_sha=not first_sha)
        assert not r2.was_unknown.any()
        assert b.db.issuer_counts() == counts
        assert b.check() == len(ders)
    finally:
        b.close()


# ------------------------------------------------------------------------------------------------ C.2 same key, other bytes

HOURS_AND_SECONDS = ((HOUR, 5, 3599), (HOUR + 1, 0, 1), (-10, 100, 3000), (-1, 0, 3599), (-400000, 59, 60))


def _pair(e):
    """Pair e: (short DER, long DER) with one key; notAfter differs inside one hour, also before 1970."""
    h, a, c = HOURS_AND_SECONDS[e % len(HOURS_AND_SECONDS)]
    s = D.serial_bytes(12, salt=1000 + e)
    return short_cert(s, h * 3600 + a), long_cert(s, h * 3600 + c)


def _near_misses():
    """Keys that must stay apart: serials 01 / 0100, one serial under two issuers, adjacent hours."""
    s = D.serial_bytes(9, salt=77)
    return [(short_cert(b"\x01", D.NOT_AFTER), 0), (short_cert(b"\x01\x00", D.NOT_AFTER), 0),
            (short_cert(s, HOUR * 3600), 0), (short_cert(s, HOUR * 3600), 1),
            (short_cert(s, HOUR * 3600 + 3600), 0), (short_cert(s, HOUR * 3600 - 1), 0)]


def _placed(n, placements):
    """n distinct fillers, then each (i, j, der_i, der_j) written at positions i and j."""
    ders = [short_cert(D.serial_bytes(6, salt=50000 + i), D.NOT_AFTER - 3600 * (i % 50)) for i in range(n)]
    for i, j, di, dj in placements:
        ders[i], ders[j] = di, dj
    return ders


def _pair_placements(edges):
    pl = []
    for e, (lo, hi) in enumerate(edges):
        short, long_ = _pair(e)
        pl.append((lo, hi, short, long_) if e % 2 else (lo, hi, long_, short))  # the longer one first, then last
    return pl


@pytest.mark.gpu
@pytest.mark.parametrize("want_sha", (True, False), ids=("stream", "light"))
def test_same_key_different_bytes(eng, ora, want_sha):
    """Precertificate / certificate pairs inside a warp, across warps and across host-pipeline stages (700 entries per
    stage), the longer one at the lower index and at the higher; near-miss keys stay distinct."""
    edges = [(3, 7), (10, 30), (40, 100), (130, 131), (690, 710), (699, 700), (1390, 1401), (2000, 2099), (2050, 2051), (2500, 2600)]
    ders = _placed(2800, _pair_placements(edges))
    nm = _near_misses()
    idx = np.zeros(len(ders) + len(nm), np.uint32)
    idx[len(ders):] = [i for _, i in nm]
    ders += [d for d, _ in nm]
    b = Both(eng, ora, issuers=(CA, CA2), table_capacity=1 << 13, max_batch_entries=700)
    try:
        got, want = b.store(ders, idx, want_sha=want_sha)
        assert (want.status == 0).all()
        for lo, hi in edges:
            assert got.was_unknown[lo] == 1 and got.was_unknown[hi] == 0, (lo, hi)
        assert got.was_unknown[len(ders) - len(nm):].all()  # no near miss collides
        b.check()
    finally:
        b.close()


@pytest.mark.gpu
def test_same_key_across_batches(eng, ora):
    pairs = [_pair(e) for e in range(len(HOURS_AND_SECONDS))]
    b = Both(eng, ora, table_capacity=1 << 12)
    try:
        r1, _ = b.store([p[1] for p in pairs] + [p[0] for p in pairs[:2]], want_sha=True)
        assert r1.was_unknown.tolist() == [1] * len(pairs) + [0, 0]
        r2, _ = b.store([p[0] for p in pairs], want_sha=False)
        assert not r2.was_unknown.any()
        b.check()
    finally:
        b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("want_sha", (True, False), ids=("stream", "light"))
def test_same_key_across_device_rounds(eng, ora, want_sha):
    """ctmr_process_device cuts n >= 2^18 entries into two rounds (131072 entries each); pairs straddle the edge."""
    import torch
    from ct_mapreduce_b200 import capi
    from test_gpu_parity import assert_same
    n, edge = 1 << 18, 1 << 17
    spans = [(edge - 1, edge), (edge - 2, edge + 5), (edge - 40, edge + 40), (edge - 700, edge + 1000), (3, n - 2)]
    ders = [b"\x30"] * n  # rejected one-byte records around the pairs (cheap for both sides)
    for lo, hi, dl, dh in _pair_placements(spans):
        ders[lo], ders[hi] = dl, dh
    for j in range(0, n, 997):  # and some distinct certificates all over the call
        if ders[j] == b"\x30":
            ders[j] = short_cert(D.serial_bytes(5, salt=j), D.NOT_AFTER)
    blob, offs = pack(ders)
    iblob, ioffs = pack([CA.der])
    idx = np.zeros(n, np.uint32)
    odb = ora.DB(b"", True)
    want = odb.process(blob, offs, iblob, ioffs, idx, NOW_NS, nthreads=8)
    dev = torch.device("cuda:0")
    dblob = torch.from_numpy(np.concatenate([blob, np.zeros(64, np.uint8)])).to(dev)
    doffs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    didx = torch.from_numpy(idx.astype(np.int32)).to(dev)
    with eng.GpuCertDatabase(table_capacity=1 << 14, log_expired_entries=True, max_issuers=16) as db:
        dense = db.register_issuers(iblob, ioffs)
        t = {k: torch.zeros((n,) + sh, dtype=dt, device=dev) for k, sh, dt in (
            ("status", (), torch.uint8), ("sha", (32,), torch.uint8), ("exp_hour", (), torch.int64),
            ("soff", (), torch.int32), ("slen", (), torch.int32), ("wu", (), torch.uint8), ("fi", (), torch.uint8))}
        bt = capi.DevBatch()
        bt.blob, bt.blob_bytes, bt.offsets, bt.n = dblob.data_ptr(), int(offs[-1]), doffs.data_ptr(), n
        bt.issuer_idx, bt.issuer_map, bt.issuer_map_len = didx.data_ptr(), None, 0
        bt.first_index, bt.now_unix_ns = 0, NOW_NS
        o = capi.DevOut(t["status"].data_ptr(), t["sha"].data_ptr() if want_sha else None, t["exp_hour"].data_ptr(),
                        t["soff"].data_ptr(), t["slen"].data_ptr(), t["wu"].data_ptr(), t["fi"].data_ptr(), None)
        db.process_device(bt, o)
        db.check_device()
        torch.cuda.synchronize()
        got = eng.BatchResult(t["status"].cpu().numpy(), t["sha"].cpu().numpy(), t["exp_hour"].cpu().numpy(),
                              t["soff"].cpu().numpy().astype(np.uint32), t["slen"].cpu().numpy().astype(np.uint32),
                              t["wu"].cpu().numpy(), t["fi"].cpu().numpy())
        assert_same(got, want, sha=want_sha)
        for lo, hi in spans:
            assert got.was_unknown[lo] == 1 and got.was_unknown[hi] == 0, (lo, hi)
        assert {k: v for k, v in db.issuer_counts().items() if v} == odb.issuer_counts()
        model = K.KeyModel()
        model.add(blob, offs, want, dense[idx], first_index=0)
        K.check_table(db.snapshot(), model, db.table_stats()[0])


# ------------------------------------------------------------------------------------------------ C.3 hot key

@pytest.mark.gpu
@pytest.mark.parametrize("want_sha", (True, False), ids=("stream", "light"))
def test_hot_key(eng, ora, want_sha):
    """One certificate 4096 times, interleaved with distinct ones: thousands of lanes find-or-insert the same slot."""
    hot = short_cert(D.serial_bytes(16, salt=4242), D.NOT_AFTER)
    ders = []
    for i in range(4096):
        ders += [short_cert(D.serial_bytes(7, salt=i), D.NOT_AFTER + (i % 3) * 3600), hot]
    b = Both(eng, ora, table_capacity=1 << 14)
    try:
        got, _ = b.store(ders, want_sha=want_sha)
        hot_at = np.arange(1, len(ders), 2)
        assert got.was_unknown[hot_at].tolist() == [1] + [0] * 4095
        assert b.check() == 4096 + 1
    finally:
        b.close()


# ------------------------------------------------------------------------------------------------ D. chosen slots

TABLE_LOG2 = 12


def _serials_with_home(hour, homes, count, seed):
    """`count` 8-octet serials whose keys (hour, dense issuer 0) have their home slot in `homes` of a 2^12 table."""
    rng = np.random.default_rng(seed)
    s = rng.integers(0, 256, size=(1 << 20, 8), dtype=np.uint64)
    s[:, 0] = (s[:, 0] & np.uint64(0x7F)) | np.uint64(1)
    bodies = np.zeros((s.shape[0], 12), np.uint64)
    bodies[:, 0] = hour & 0xFFFFFFFF
    bodies[:, 2] = np.uint64(8) | (s[:, 0] << np.uint64(8)) | (s[:, 1] << np.uint64(16)) | (s[:, 2] << np.uint64(24))
    bodies[:, 3] = s[:, 3] | (s[:, 4] << np.uint64(8)) | (s[:, 5] << np.uint64(16)) | (s[:, 6] << np.uint64(24))
    bodies[:, 4] = s[:, 7]
    home = (K.key_hash_np(bodies) >> np.uint64(7)) & np.uint64((1 << TABLE_LOG2) - 1)
    pick = np.nonzero(np.isin(home, np.array(list(homes), np.uint64)))[0][:count]
    assert pick.size == count
    out = [bytes(int(x) for x in s[i]) for i in pick]
    for ser in out[:4]:  # the vectorised hash is the scalar restatement
        assert K.home_slot(K.key_hash(K.key_body(hour, 0, ser)), (1 << TABLE_LOG2) - 1) in homes
    return out


@pytest.mark.gpu
def test_table_slot_by_slot_cluster_wrap_fill_evict_restore(eng, ora):
    """A 2^12 table: 64 keys with one home slot, keys homed on the last four slots (their chains wrap to slot 0), filled
    to 0.9.  Checked slot by slot after the inserts, after evicting half of the wrapped chain and after a restore;
    every survivor is still known, every evicted key is new again."""
    early, late = HOUR - 1000, HOUR + 1000
    cluster = [short_cert(s, HOUR * 3600) for s in _serials_with_home(HOUR, {1000}, 64, 1)]
    wrap_early = [short_cert(s, early * 3600) for s in _serials_with_home(early, {4092, 4093, 4094, 4095}, 12, 2)]
    wrap_late = [short_cert(s, late * 3600 + 59) for s in _serials_with_home(late, {4092, 4093, 4094, 4095}, 12, 3)]
    fill_n = int(0.9 * (1 << TABLE_LOG2)) - 64 - 24
    fill = [short_cert(D.serial_bytes(10, salt=90000 + i), D.NOT_AFTER + 3600 * (i % 7)) for i in range(fill_n)]
    wrap = [d for pair in zip(wrap_early, wrap_late) for d in pair]
    b = Both(eng, ora, table_capacity=1 << TABLE_LOG2, pair_capacity_log2=10)
    try:
        b.store(cluster + wrap, want_sha=True)
        b.store(fill, want_sha=False)
        assert b.check() == 64 + 24 + fill_n
        table, _ = K.decode_snapshot(b.db.snapshot())
        assert table["tag"][0] != 0 and (table["tag"][4092:] != 0).all()  # the wrapped chain reached slot 0
        # evict the early half of the wrapped chain (and whatever else expires by then)
        cut = early * 3600
        dropped = b.db.evict_expired(cut)
        assert dropped == b.odb.evict_expired(cut) > 0
        b.model.evict(cut)
        b.check()
        r, _ = b.store(wrap, want_sha=True)
        assert r.was_unknown.tolist() == [1, 0] * 12  # evicted keys are new again, survivors are still known
        b.check()
        snap = b.db.snapshot().copy()
    finally:
        b.close()
    b2 = Both(eng, ora, table_capacity=1 << TABLE_LOG2, pair_capacity_log2=10)
    try:
        b2.db.restore(snap)
        b2.odb, b2.model = b.odb, b.model
        b2.check()
        r, _ = b2.store(cluster + wrap, want_sha=False)
        assert not r.was_unknown.any()
        b2.check()
    finally:
        b2.close()
