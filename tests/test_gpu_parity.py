"""Parity tests proper: the CUDA path, called through the C ABI, against the oracle on the same
seeded inputs -- bit-exact for every output (fingerprints, membership bits, per-issuer counts).
Marked gpu: they run on the H100 box."""
import hashlib

import numpy as np
import pytest

from conftest import NOW_NS, NOW_SEC, README_FILTER, pack

pytestmark = pytest.mark.gpu

FIELDS = ("status", "exp_hour", "serial_off", "serial_len", "was_unknown", "first_issuer_hour")


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def assert_same(r_gpu, r_ora, sha=True):
    for f in FIELDS:
        a, b = getattr(r_gpu, f), getattr(r_ora, f)
        if f in ("exp_hour", "serial_off", "serial_len"):  # defined where the leaf parsed
            m = r_ora.status != 1
            a, b = a[m], b[m]
        bad = np.nonzero(a != b)[0]
        assert bad.size == 0, (f, bad[:10], a[bad[:10]], b[bad[:10]])
    if sha:
        bad = np.nonzero((r_gpu.sha256 != r_ora.sha256).any(axis=1))[0]
        assert bad.size == 0, ("sha256", bad[:10])


def run_both(eng, ora, blob, offs, iblob, ioffs, idx, now_ns=NOW_NS, flt=README_FILTER, log_expired=False, **kw):
    odb = ora.DB(flt, log_expired)
    r_ora = odb.process(blob, offs, iblob, ioffs, idx, now_ns)
    with eng.GpuCertDatabase(issuer_cn_filter=flt, log_expired_entries=log_expired, table_capacity=1 << 18, **kw) as db:
        r_gpu = db.store_batch(blob, offs, iblob, ioffs, idx, now_ns)
        counts = db.issuer_counts()
        sc = db.status_counters()
    return r_gpu, r_ora, counts, odb, sc


def test_config1_10k_uniform(eng, ora):
    """BASELINE.json configs[0]: 10k synthetic ~1.5 KB certs, full map + both reducers."""
    n = 10000
    cfg = ora.synth_cfg(n)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    r_gpu, r_ora, counts, odb, sc = run_both(eng, ora, blob, offs, iblob, ioffs, idx)
    assert_same(r_gpu, r_ora)
    oc = odb.issuer_counts()
    assert {k: v for k, v in counts.items() if v} == oc
    assert np.array_equal(sc, odb.filter_counters())
    # independent check of the fingerprints
    for i in (0, 1, 17, n - 1):
        assert r_gpu.sha256[i].tobytes() == hashlib.sha256(blob[offs[i]:offs[i + 1]].tobytes()).digest()


def test_mixed_sizes_with_duplicates(eng, ora):
    """configs[4] shape: 512 B-8 KB, every certificate twice, 256 issuers."""
    n = 12000
    cfg = ora.synth_cfg(n, len_mode=1, len_lo=512, len_hi=8192, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    r_gpu, r_ora, counts, odb, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, flt=b"")
    assert_same(r_gpu, r_ora)
    ok = r_ora.status == 0
    assert int(r_gpu.was_unknown.sum()) * 2 == int(ok.sum())  # every kept certificate has exactly one twin
    assert {k: v for k, v in counts.items() if v} == odb.issuer_counts()


def test_persistence_across_batches(eng, ora):
    """The known-certificate set outlives a batch: later batches see earlier entries (Redis set)."""
    n = 6000
    cfg = ora.synth_cfg(n, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    odb = ora.DB(README_FILTER, False)
    with eng.GpuCertDatabase(issuer_cn_filter=README_FILTER, table_capacity=1 << 16) as db:
        cuts = [0, 1000, 1001, 3500, n]
        for a, b in zip(cuts[:-1], cuts[1:]):
            sub_offs = offs[a:b + 1]
            r_o = odb.process(blob, sub_offs, iblob, ioffs, idx[a:b], NOW_NS)
            r_g = db.store_batch(blob, sub_offs, iblob, ioffs, idx[a:b], NOW_NS)
            assert_same(r_g, r_o)
        assert {k: v for k, v in db.issuer_counts().items() if v} == odb.issuer_counts()
        # KnownCertificates.Count for a few (expDate, issuer) sets
        r_all = ora.DB(README_FILTER, False).process(blob, offs, iblob, ioffs, idx, NOW_NS)
        dense = db.register_issuers(iblob, ioffs)
        for i in np.nonzero(r_all.status == 0)[0][:25]:
            dig = db.issuer_digest(int(dense[idx[i]]))
            assert db.get_known_certificates(int(r_all.exp_hour[i]), dig).count() == odb.set_cardinality(int(r_all.exp_hour[i]), dig)


def test_pipeline_sub_batches(eng, ora):
    """Force the host path through many pipeline stages; results must not depend on the staging."""
    n = 9000
    cfg = ora.synth_cfg(n, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    r_gpu, r_ora, counts, odb, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, max_batch_entries=700)
    assert_same(r_gpu, r_ora)
    r_gpu2, _, _, _, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, max_batch_entries=4096, max_batch_bytes=1 << 20)
    assert_same(r_gpu2, r_ora)


def test_reference_fixtures(eng, ora, golden):
    """The reference's embedded PEMs through the GPU path (types_test.go:21-39, filesystemdatabase_test.go:17-64)."""
    lz, ca, real = golden["kLeadingZeroes"]["der"], golden["kEmptySPKI"]["der"], golden["kRealSPKI"]["der"]
    ders = [lz, lz, ca, real, lz]
    blob, offs = pack(ders)
    iblob, ioffs = pack([ca, real])
    idx = np.array([0, 0, 0, 1, 0xFFFFFFFF], np.uint32)
    before = (golden["kLeadingZeroes"]["not_after_unix"] - 10) * 10**9
    r_gpu, r_ora, counts, odb, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, now_ns=before, flt=b"")
    assert_same(r_gpu, r_ora)
    assert list(r_gpu.status) == [0, 0, 2, 2, 5]
    for i, d in enumerate(ders):
        assert r_gpu.sha256[i].tobytes().hex() == hashlib.sha256(d).hexdigest()
    assert r_gpu.sha256[0].tobytes().hex() == golden["kLeadingZeroes"]["sha256_der"]
    s0 = int(r_gpu.serial_off[0])
    assert lz[s0:s0 + int(r_gpu.serial_len[0])].hex() == "00aa"  # types_test.go:93
    # Issuer.ID of the CA = golden digest (types.go:124-130)
    import base64
    (dig, cnt), = [(k, v) for k, v in counts.items() if v]
    assert base64.urlsafe_b64encode(dig).decode() == golden["kEmptySPKI"]["issuer_id_of_own_spki"] and cnt == 1


def test_filter_variants(eng, ora):
    n = 3000
    cfg = ora.synth_cfg(n)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    for flt, le in ((b"", False), (b"", True), (b"Let's Encrypt", False), (b"Let's Encrypt,ISRG", True),
                    (b"x,", False), (b" ISRG Root X1,Synth Trust Services CA 3,Let's Encrypt Authority X12", False),
                    (b",", False), (b"Z" * 100, False)):
        r_gpu, r_ora, _, _, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, flt=flt, log_expired=le)
        assert_same(r_gpu, r_ora, sha=False)
    # now with a fractional part: NotAfter.Before(now) strictness
    r_gpu, r_ora, _, _, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, now_ns=NOW_NS + 1, flt=b"")
    assert_same(r_gpu, r_ora, sha=False)


def _mutations(der, rng, count=60, span=420):
    out = [der[:-1], der + b"\x00", der[:len(der) // 2], b"", b"\x30", b"\x30\x80", b"\x30\x84\xff\xff\xff\xff", der[:4]]
    for _ in range(count):
        b = bytearray(der)
        for _ in range(rng.integers(1, 4)):
            b[rng.integers(0, min(len(b), span))] = rng.integers(0, 256)
        out.append(bytes(b))
    return out


def test_malformed_inputs_are_safe_and_agree(eng, ora, golden):
    """Truncated / corrupted DER: never a crash, status agrees with the oracle, the fingerprint is
    still SHA-256 of the raw bytes (edge cases: empty record, ragged sizes, 1-byte records)."""
    rng = np.random.default_rng(7)
    cfg = ora.synth_cfg(64)
    blob0, offs0, _ = ora.synth_corpus(cfg, 0, 8)
    ders = []
    for i in range(8):
        ders += _mutations(blob0[offs0[i]:offs0[i + 1]].tobytes(), rng)
    ders += _mutations(golden["kRealSPKI"]["der"], rng)
    blob, offs = pack(ders)
    iblob, ioffs = ora.synth_issuers(cfg)
    bad_issuer = iblob[ioffs[3]:ioffs[4]].tobytes()[:-7]
    iblob2, ioffs2 = pack([iblob[ioffs[0]:ioffs[1]].tobytes(), bad_issuer])
    idx = (np.arange(len(ders)) % 3).astype(np.uint32)
    idx[idx == 2] = 0xFFFFFFFF
    r_gpu, r_ora, _, _, _ = run_both(eng, ora, blob, offs, iblob2, ioffs2, idx, flt=b"", log_expired=True)
    assert_same(r_gpu, r_ora)
    assert set(np.unique(r_gpu.status)) >= {0, 1, 5, 6}
    for i, d in enumerate(ders):
        assert r_gpu.sha256[i].tobytes() == hashlib.sha256(d).digest(), i


def test_padding_boundaries_every_length(eng, ora):
    """Fingerprint of records of every length 0..300 at every 16-byte misalignment (SHA-256 padding
    edges at 55/56/63/64 and the 256-byte streaming chunk edge)."""
    rng = np.random.default_rng(3)
    ders = [rng.integers(0, 256, size=L, dtype=np.uint8).tobytes() for L in range(0, 301)]
    ders += [rng.integers(0, 256, size=L, dtype=np.uint8).tobytes() for L in (511, 512, 513, 767, 768, 1023, 1024, 1025, 4095, 4096, 8191, 8192, 20000)]
    blob, offs = pack(ders)
    with eng.GpuCertDatabase(table_capacity=1 << 12) as db:
        r = db.store_batch(blob, offs, None, None, None, NOW_NS)
    assert (r.status == 1).all()
    for i, d in enumerate(ders):
        assert r.sha256[i].tobytes() == hashlib.sha256(d).digest(), len(d)


def test_empty_batch_and_no_issuers(eng, ora):
    with eng.GpuCertDatabase(table_capacity=1 << 12) as db:
        r = db.store_batch(np.zeros(0, np.uint8), np.zeros(1, np.uint64), None, None, None, NOW_NS)
        assert r.status.size == 0
        cfg = ora.synth_cfg(100)
        blob, offs, idx = ora.synth_corpus(cfg, 0, 100)
        r = db.store_batch(blob, offs, None, None, None, NOW_NS)  # no chain at all
        exp = ora.DB(b"", False).process(blob, offs, np.zeros(0, np.uint8), np.zeros(1, np.uint64),
                                         np.full(100, 0xFFFFFFFF, np.uint32), NOW_NS)
        assert np.array_equal(r.status, exp.status) and not r.was_unknown.any()


def test_table_full_is_reported(eng, ora):
    from ct_mapreduce_b200 import capi
    n = 20000
    cfg = ora.synth_cfg(n)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    with eng.GpuCertDatabase(table_capacity=4096) as db:
        with pytest.raises(capi.CtmrError) as ei:
            db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
        assert ei.value.code == capi.E_TABLE_FULL


def test_no_fingerprint_flag(eng, ora):
    from ct_mapreduce_b200 import capi
    n = 2000
    cfg = ora.synth_cfg(n, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    r_gpu, r_ora, _, _, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, flags=capi.F_NO_FINGERPRINT)
    assert_same(r_gpu, r_ora, sha=False)


def test_device_generator_matches_host_generator(eng, ora):
    """The bench corpus is generated in HBM; the CPU arm regenerates it on the host: same bytes."""
    import torch
    from ct_mapreduce_b200 import capi
    for kw in (dict(), dict(len_mode=1, len_lo=512, len_hi=8192, dup_mode=1), dict(len_mode=1, len_lo=512, len_hi=4096, dup_mode=1)):
        n, first = 3000, 1234
        cfg_o = ora.synth_cfg(50000, **kw)
        cfg_g = capi.synth_cfg(50000, **kw)
        blob, offs, idx = ora.synth_corpus(cfg_o, first, n)
        dblob, doffs, didx, total = eng.synth_corpus_device(cfg_g, first, n, "cuda:0")
        assert total == int(offs[-1])
        assert np.array_equal(doffs.cpu().numpy().astype(np.uint64), offs)
        assert np.array_equal(didx.cpu().numpy().astype(np.uint32), idx)
        got = dblob[:total].cpu().numpy()
        bad = np.nonzero(got != blob)[0]
        assert bad.size == 0, (kw, bad[:10])
        iblob_o, ioffs_o = ora.synth_issuers(cfg_o)
        iblob_g, ioffs_g = eng.synth_issuers(cfg_g)
        assert np.array_equal(iblob_o, iblob_g) and np.array_equal(ioffs_o, ioffs_g)


def test_process_device_pipelined_sub_batches(eng, ora):
    """ctmr_process_device on a device-resident batch big enough to take the internal map/reduce
    pipeline (2 sub-batches, two streams); every output against the oracle."""
    import torch
    from ct_mapreduce_b200 import capi
    n = 300_000
    kw = dict(len_mode=1, len_lo=512, len_hi=4096, dup_mode=1)
    cfg_o, cfg_g = ora.synth_cfg(n, **kw), capi.synth_cfg(n, **kw)
    blob, offs, idx = ora.synth_corpus(cfg_o, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg_o)
    want = ora.DB(README_FILTER, False).process(blob, offs, iblob, ioffs, idx, NOW_NS, nthreads=8)
    dev = torch.device("cuda:0")
    dblob, doffs, didx, total = eng.synth_corpus_device(cfg_g, 0, n, dev)
    with eng.GpuCertDatabase(table_capacity=1 << 20, issuer_cn_filter=README_FILTER, max_issuers=1024) as db:
        dense = db.register_issuers(iblob, ioffs)
        assert (dense == np.arange(cfg_g.n_issuers)).all()
        t = {k: torch.empty((n,) + sh, dtype=dt, device=dev) for k, sh, dt in (
            ("status", (), torch.uint8), ("sha", (32,), torch.uint8), ("exp_hour", (), torch.int64),
            ("soff", (), torch.int32), ("slen", (), torch.int32), ("wu", (), torch.uint8), ("fi", (), torch.uint8))}
        b = capi.DevBatch()
        b.blob, b.blob_bytes, b.offsets, b.n = dblob.data_ptr(), total, doffs.data_ptr(), n
        b.issuer_idx, b.issuer_map, b.issuer_map_len = didx.data_ptr(), None, 0
        b.first_index, b.now_unix_ns = 0, NOW_NS
        o = capi.DevOut(t["status"].data_ptr(), t["sha"].data_ptr(), t["exp_hour"].data_ptr(), t["soff"].data_ptr(),
                        t["slen"].data_ptr(), t["wu"].data_ptr(), t["fi"].data_ptr(), None)
        db.process_device(b, o)
        db.check_device()
        torch.cuda.synchronize()
        map_ms, total_ms = db.profile_last()
        assert 0 < map_ms <= total_ms * 1.01
        counts = db.issuer_counts()
    got = eng.BatchResult(t["status"].cpu().numpy(), t["sha"].cpu().numpy(), t["exp_hour"].cpu().numpy(),
                          t["soff"].cpu().numpy().astype(np.uint32), t["slen"].cpu().numpy().astype(np.uint32),
                          t["wu"].cpu().numpy(), t["fi"].cpu().numpy())
    assert_same(got, want)
    assert sum(counts.values()) == int(want.was_unknown.sum())


def _two_halves(ora, n=8000):
    cfg = ora.synth_cfg(n, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    odb = ora.DB(README_FILTER, False)
    h = n // 2
    ra = odb.process(blob, offs[:h + 1], iblob, ioffs, idx[:h], NOW_NS)
    rb = odb.process(blob, offs[h:], iblob, ioffs, idx[h:], NOW_NS)
    return cfg, blob, offs, idx, iblob, ioffs, h, ra, rb, odb


def test_warm_start_from_existing_sets(eng, ora):
    """SURVEY §8(f)-4: a fresh ctx seeded from the Redis sets an earlier run left behind answers the
    second half of the log exactly as the uninterrupted reference would."""
    cfg, blob, offs, idx, iblob, ioffs, h, ra, rb, odb = _two_halves(ora)
    digests = {}
    for k in range(cfg.n_issuers):
        der = iblob[ioffs[k]:ioffs[k + 1]].tobytes()
        rc, c = ora.parse_cert(der)
        digests[k] = ora.issuer_id(der[c.spki_off:c.spki_off + c.spki_len])[0]
    sets = {}  # what Redis holds after the first half: (hour, issuer) -> serials
    for i in np.nonzero(ra.was_unknown)[0]:
        a = int(offs[i]) + int(ra.serial_off[i])
        sets.setdefault((int(ra.exp_hour[i]), digests[int(idx[i])]), []).append(blob[a:a + int(ra.serial_len[i])].tobytes())
    with eng.GpuCertDatabase(issuer_cn_filter=README_FILTER, table_capacity=1 << 16) as db:
        for (hour, dig), serials in sets.items():
            db.preload_known(hour, dig, serials)
        rg = db.store_batch(blob, offs[h:], iblob, ioffs, idx[h:], NOW_NS)
        assert_same(rg, rb)
        assert {k: v for k, v in db.issuer_counts().items() if v} == odb.issuer_counts()
        (hour, dig), serials = next(iter(sets.items()))
        assert db.get_known_certificates(hour, dig).count() == odb.set_cardinality(hour, dig)


def test_snapshot_and_restore(eng, ora):
    """Checkpoint the derived device state after the first half, restore it into a new ctx, continue."""
    cfg, blob, offs, idx, iblob, ioffs, h, ra, rb, odb = _two_halves(ora)
    kw = dict(issuer_cn_filter=README_FILTER, table_capacity=1 << 16, max_issuers=512, pair_capacity_log2=18)
    with eng.GpuCertDatabase(**kw) as db1:
        r1 = db1.store_batch(blob, offs[:h + 1], iblob, ioffs, idx[:h], NOW_NS)
        assert_same(r1, ra)
        snap = db1.snapshot().copy()
    with eng.GpuCertDatabase(**kw) as db2:
        db2.restore(snap)
        r2 = db2.store_batch(blob, offs[h:], iblob, ioffs, idx[h:], NOW_NS)
        assert_same(r2, rb)
        assert {k: v for k, v in db2.issuer_counts().items() if v} == odb.issuer_counts()
        assert np.array_equal(db2.status_counters(), odb.filter_counters())
    from ct_mapreduce_b200 import capi
    with eng.GpuCertDatabase(issuer_cn_filter=README_FILTER, table_capacity=1 << 15, max_issuers=512, pair_capacity_log2=18) as db3:
        with pytest.raises(capi.CtmrError):
            db3.restore(snap)  # capacities differ


def test_fuzz_whole_certificate_mutations(eng, ora):
    """Byte flips anywhere in the record (names, validity, SPKI, every extension, signature header),
    truncations and length-field edits over mixed-size certificates: status and every other output
    must still agree with the oracle, with and without the fingerprint (streaming and light kernels)."""
    from ct_mapreduce_b200 import capi
    rng = np.random.default_rng(11)
    cfg = ora.synth_cfg(256, len_mode=1, len_lo=512, len_hi=4096)
    blob0, offs0, idx0 = ora.synth_corpus(cfg, 0, 48)
    iblob, ioffs = ora.synth_issuers(cfg)
    ders, idx = [], []
    for i in range(48):
        d = blob0[offs0[i]:offs0[i + 1]].tobytes()
        muts = _mutations(d, rng, count=40, span=len(d))
        # targeted edits of DER length octets: grow / shrink the outer and TBS lengths, flip a tag
        for pos in (1, 2, 3, 5, 6, 7):
            b = bytearray(d); b[pos] = (b[pos] + int(rng.integers(1, 255))) & 0xFF; muts.append(bytes(b))
        ders += muts
        idx += [int(idx0[i])] * len(muts)
    blob, offs = pack(ders)
    idx = np.array(idx, np.uint32)
    for flags in (0, capi.F_NO_FINGERPRINT):
        r_gpu, r_ora, _, _, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, flt=README_FILTER, log_expired=False, flags=flags)
        assert_same(r_gpu, r_ora, sha=(flags == 0))
    assert 0 < int((r_ora.status == 1).sum()) < len(ders)  # both parsed and rejected records are present


def test_issuer_metadata_string_reducers(eng, ora):
    """SURVEY §8(f)-1: spans of the issuer Name and the cRLDistributionPoints value, and the
    first-seen bits that let the host run IssuerMetadata.Accumulate's string inserts only for
    candidates (storage/issuermetadata.go:92-138).  Two batches: the sets persist."""
    import warnings
    from cryptography import x509
    warnings.filterwarnings("ignore")
    n = 6000
    cfg = ora.synth_cfg(n, len_mode=1, len_lo=512, len_hi=4096, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    odb = ora.DB(README_FILTER, False)
    h = 2500
    with eng.GpuCertDatabase(issuer_cn_filter=README_FILTER, table_capacity=1 << 16) as db:
        for lo, hi in ((0, h), (h, n)):
            want = odb.process(blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi], NOW_NS)
            got = db.store_batch(blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi], NOW_NS, want_meta=True)
            assert_same(got, want)
            parsed = want.status != 1
            for f in ("issuer_name_off", "issuer_name_len", "crldp_off", "crldp_len"):
                assert np.array_equal(getattr(got, f)[parsed], getattr(want, f)[parsed]), f
            for f in ("first_issuer_dn", "first_crldp"):
                bad = np.nonzero(getattr(got, f) != getattr(want, f))[0]
                assert bad.size == 0, (f, bad[:10])
            # candidates only among new certificates, and at most a handful per issuer
            assert not (got.first_issuer_dn & ~got.was_unknown).any()
            assert int(got.first_issuer_dn.sum()) <= cfg.n_issuers and int(got.first_crldp.sum()) <= 2 * cfg.n_issuers
        # the spans are what an X.509 library calls the issuer name / the extension value
        for i in np.nonzero(got.first_issuer_dn)[0][:20]:
            e = h + int(i)
            der = blob[offs[e]:offs[e + 1]].tobytes()
            cert = x509.load_der_x509_certificate(der)
            a, l = int(got.issuer_name_off[i]), int(got.issuer_name_len[i])
            assert der[a:a + l] == cert.issuer.public_bytes()
            a, l = int(got.crldp_off[i]), int(got.crldp_len[i])
            ext = cert.extensions.get_extension_for_oid(x509.oid.ExtensionOID.CRL_DISTRIBUTION_POINTS)
            assert ext.value[0].full_name[0].value.encode() in der[a:a + l]


def test_time_encodings_on_device(eng, ora):
    """Every UTCTime / GeneralizedTime form Go accepts or rejects (tests/test_oracle_properties.py), plus
    random instants, through both map kernels: status and expiry hour must match the oracle."""
    import datetime
    from ct_mapreduce_b200 import capi
    from test_oracle_properties import _cert_with_times, _fmt_utc
    rng = np.random.default_rng(5)
    forms = [(b"300615123045Z", 0x17), (b"3006151230Z", 0x17), (b"300615123045+0130", 0x17), (b"300615123045-0800", 0x17),
             (b"20300615123045Z", 0x18), (b"300615123045+0000", 0x17), (b"301315123045Z", 0x17), (b"300632123045Z", 0x17),
             (b"300615243045Z", 0x17), (b"300615126045Z", 0x17), (b"300615123060Z", 0x17), (b"300229123045Z", 0x17),
             (b"280229123045Z", 0x17), (b"30061512304Z", 0x17), (b"300615123045", 0x17), (b"203006151230Z", 0x18),
             (b"300615123045Z", 0x18), (b"491231235959Z", 0x17), (b"500101000000Z", 0x17), (b"00010101000000Z", 0x18),
             (b"99991231235959Z", 0x18), (b"20300615123045+0530", 0x18), (b"19691231235959Z", 0x18)]
    ders = [_cert_with_times(b"900101000000Z", na, na_tag=tag) for na, tag in forms]
    for _ in range(200):
        t = datetime.datetime(1950, 1, 1) + datetime.timedelta(seconds=int(rng.integers(0, 3155000000)))
        ders.append(_cert_with_times(b"900101000000Z", _fmt_utc(t)))
    blob, offs = pack(ders)
    ca = ders[0]
    iblob, ioffs = pack([ca])
    idx = np.zeros(len(ders), np.uint32)
    for flags in (0, capi.F_NO_FINGERPRINT):
        r_gpu, r_ora, _, _, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, flt=b"", log_expired=True, flags=flags)
        assert_same(r_gpu, r_ora, sha=(flags == 0))
    assert int((r_ora.status == 0).sum()) > 200 and int((r_ora.status == 1).sum()) >= 10


def test_large_certificates_three_byte_lengths(eng, ora):
    """Certificates of 20-70 KB: DER lengths with three octets (0x83), hundreds of streaming chunks per
    lane, the top length bucket; both kernels."""
    from ct_mapreduce_b200 import capi
    n = 256
    cfg = ora.synth_cfg(n, len_mode=0, len_lo=20000, len_hi=70000, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    assert int(np.diff(offs.astype(np.int64)).max()) > 65536
    iblob, ioffs = ora.synth_issuers(cfg)
    for flags in (0, capi.F_NO_FINGERPRINT):
        r_gpu, r_ora, counts, odb, _ = run_both(eng, ora, blob, offs, iblob, ioffs, idx, flags=flags)
        assert_same(r_gpu, r_ora, sha=(flags == 0))
        assert {k: v for k, v in counts.items() if v} == odb.issuer_counts()
    assert int((r_ora.status == 0).sum()) > 20


def test_pem_of_new_certificates(eng, ora):
    """SURVEY §8(f)-3: the PEM text Store hands to StoreCertificatePEM, encoded on the device for NEW certificates only."""
    import ssl
    from conftest import go_pem
    from ct_mapreduce_b200 import capi
    n = 5000
    cfg = ora.synth_cfg(n, len_mode=1, len_lo=300, len_hi=5000, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    der = lambda i: blob[int(offs[i]):int(offs[i + 1])].tobytes()
    assert go_pem(der(0)).decode() == ssl.DER_cert_to_PEM_cert(der(0))  # the expectation itself, against an independent encoder
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16, max_batch_entries=700) as db:  # 8 pipeline slices
        r = db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS, want_pem=True)
        assert 0 < int(r.was_unknown.sum()) < n
        assert int(r.pem_off[n]) == sum(len(go_pem(der(i))) for i in np.nonzero(r.was_unknown)[0])
        for i in range(n):
            assert r.pem_of(i) == (go_pem(der(i)) if r.was_unknown[i] else b""), i
        # every length residue mod 3 and mod 48 occurs in the corpus
        lens = np.diff(offs.astype(np.int64))[r.was_unknown == 1]
        assert set((lens % 3).tolist()) == {0, 1, 2} and len(set((lens % 48).tolist())) == 48
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        out = eng.BatchResult(np.zeros(n, np.uint8), np.zeros((n, 32), np.uint8), np.zeros(n, np.int64), np.zeros(n, np.uint32),
                              np.zeros(n, np.uint32), np.zeros(n, np.uint8), np.zeros(n, np.uint8))
        out.pem, out.pem_off = np.zeros(1000, np.uint8), np.zeros(n + 1, np.uint64)
        o = capi.Out(*[capi.ptr(getattr(out, f)) for f in ("status", "sha256", "exp_hour", "serial_off", "serial_len", "was_unknown", "first_issuer_hour")],
                     *([None] * 6), capi.ptr(out.pem), out.pem.size, capi.ptr(out.pem_off))
        import ctypes as C
        rc = db._lib.ctmr_process_batch(db._h, capi.ptr(blob), capi.ptr(offs), n, capi.ptr(iblob), capi.ptr(ioffs), ioffs.size - 1,
                                        capi.ptr(idx), NOW_NS, C.byref(o))
        assert rc == capi.E_BATCH_TOO_LARGE


def test_ttl_eviction_matches_redis_expiry(eng, ora):
    """SURVEY §8(f)-4: the reference's sets carry EXPIREAT(expDate); when the TTLs fire, whole sets vanish.  The device
    state follows: evicted serials are unknown again, counts drop, slots are reclaimed, later batches agree with the oracle."""
    n = 8000
    cfg = ora.synth_cfg(n, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    odb = ora.DB(b"", True)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 15) as db:
        half = n // 2
        r_o = odb.process(blob, offs[:half + 1], iblob, ioffs, idx[:half], NOW_NS)
        r_g = db.store_batch(blob, offs[:half + 1], iblob, ioffs, idx[:half], NOW_NS)
        assert_same(r_g, r_o)
        hours = np.sort(r_o.exp_hour[r_o.status == 0])
        used0 = db.table_stats()[0]
        assert db.evict_expired(int(hours[0]) * 3600 - 1) == odb.evict_expired(int(hours[0]) * 3600 - 1) == 0   # nothing is due yet
        cut = int(hours[hours.size // 2]) * 3600          # a set expiring exactly now is gone (EXPIREAT fires at >=)
        dropped = odb.evict_expired(cut)
        assert db.evict_expired(cut) == dropped and 0 < dropped < used0
        assert db.table_stats()[0] == used0 - dropped
        assert {k: v for k, v in db.issuer_counts().items() if v} == {k: v for k, v in odb.issuer_counts().items() if v}
        # the second half repeats certificates of the first: the evicted ones are new again, the others still known
        r_o2 = odb.process(blob, offs[half:], iblob, ioffs, idx[half:], NOW_NS)
        r_g2 = db.store_batch(blob, offs[half:], iblob, ioffs, idx[half:], NOW_NS)
        assert_same(r_g2, r_o2)
        assert 0 < int(r_o2.was_unknown.sum()) < int((r_o2.status == 0).sum())
        assert {k: v for k, v in db.issuer_counts().items() if v} == {k: v for k, v in odb.issuer_counts().items() if v}
        # everything is past its TTL eventually
        assert db.evict_expired(1 << 40) == odb.evict_expired(1 << 40) > 0
        assert db.table_stats()[0] == 0 and not any(db.issuer_counts().values())


def test_long_serials_are_declined_not_misdeduplicated(eng, ora):
    """The ONE place where the product knowingly differs from the reference (VERDICT r1, weak #2): a key record holds 39
    serial octets.  The reference has no limit (storage/types.go:171-178) and the oracle follows it; the GPU path
    DECLINES longer serials -- status CTMR_ST_SERIAL_TOO_LONG, never was_unknown, never in a set -- so that the host
    routes exactly those entries to the stock per-entry Store (go/ctmr/gpudatabase.go).  Everything else is unchanged,
    in both map kernels."""
    from ct_mapreduce_b200 import capi
    from test_oracle_properties import _cert_with_times
    ders, long_ = [], []
    for rep in range(2):
        for n in (1, 20, 38, 39, 40, 41, 64, 127, 128, 300):
            ser = bytes([0x01]) + bytes([(n * 7 + 3) & 0xFF]) * (n - 1)
            ders.append(_cert_with_times(b"900101000000Z", b"300615123045Z", serial=ser))
            long_.append(n > 39)
    long_ = np.array(long_)
    blob, offs = pack(ders)
    iblob, ioffs = pack([ders[0]])
    idx = np.zeros(len(ders), np.uint32)
    want = ora.DB(b"", True).process(blob, offs, iblob, ioffs, idx, NOW_NS)
    assert (want.status == 0).all() and want.was_unknown.tolist() == [1] * 10 + [0] * 10     # the reference stores them all
    for flags in (0, capi.F_NO_FINGERPRINT):
        with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 12, flags=flags) as db:
            got = db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS, want_sha=not flags)
            sc = db.status_counters()
            counts = db.issuer_counts()
        assert (got.status[long_] == capi.ST_SERIAL_TOO_LONG).all() and (got.was_unknown[long_] == 0).all()
        assert np.array_equal(got.status[~long_], want.status[~long_])
        assert np.array_equal(got.was_unknown[~long_], want.was_unknown[~long_])
        assert np.array_equal(got.serial_len, want.serial_len) and np.array_equal(got.serial_off, want.serial_off)
        assert np.array_equal(got.exp_hour, want.exp_hour)
        assert int(sc[capi.ST_SERIAL_TOO_LONG]) == int(long_.sum()) and int(sc[capi.ST_OK]) == int((~long_).sum())
        assert sum(counts.values()) == int(want.was_unknown[~long_].sum())
        if not flags:
            assert np.array_equal(got.sha256, want.sha256)


def test_unmodelled_ctgo_cases_agree_between_oracle_and_gpu(eng, ora):
    """The inputs of tests/test_ctgo_leniencies.py (where this path knowingly differs from Go's x509): whatever the oracle
    says about them, both CUDA walkers say the same."""
    from ct_mapreduce_b200 import capi
    from test_ctgo_leniencies import CASES, cert
    ders = [c[1] for c in CASES] * 2
    blob, offs = pack(ders)
    iblob, ioffs = pack([cert()])
    idx = np.zeros(len(ders), np.uint32)
    for flags in (0, capi.F_NO_FINGERPRINT):
        r_gpu, r_ora, counts, odb, sc = run_both(eng, ora, blob, offs, iblob, ioffs, idx, flt=b"", log_expired=True, flags=flags)
        assert_same(r_gpu, r_ora, sha=not flags)
        assert np.array_equal(sc, odb.filter_counters())
