"""Exact multi-GPU parity behind the C ABI (SURVEY.md §8(e), VERDICT r1 "missing 1/3").

Two forms of the same device code:
  * ctmr_group_*  -- one process drives several shards (what the Go host calls).  `devices` may repeat a device, so
    these tests run on a 1-GPU box (three shards on cuda:0: the owner routing, the peer-addressed tables, the event
    fan-in and the group registry are all exercised; only the wire is missing) and on real peers when there are >= 2 GPUs.
  * ctmr_peer_*   -- one process per GPU, tables attached over CUDA IPC, barriers in peer memory.  Run with two
    processes on one GPU (gloo plumbing) and, with >= 2 GPUs, one process per GPU (NCCL plumbing).
Every comparison is against the oracle run SEQUENTIALLY over the same entries in the order the group defines.
"""

import numpy as np
import pytest

from conftest import NOW_NS, NOW_SEC, README_FILTER, go_pem
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

FIELDS = ("status", "was_unknown", "first_issuer_hour")
META = ("first_issuer_dn", "first_crldp")


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def _device_sets():
    import torch
    sets = [[0, 0, 0]]
    if torch.cuda.device_count() >= 2:
        sets.append(list(range(min(torch.cuda.device_count(), 8))))
    return sets


def _check_fields(got, want, n, fields, parsed_only=()):
    for f in fields:
        a, b = getattr(got, f), getattr(want, f)
        bad = np.nonzero((a != b).reshape(n, -1).any(axis=1))[0]
        assert bad.size == 0, (f, bad.size, bad[:12])
    for f in parsed_only:
        m = want.status != 1
        assert np.array_equal(getattr(got, f)[m], getattr(want, f)[m]), f


@pytest.mark.parametrize("shards", ["one_gpu_three_shards", "all_gpus"])
def test_group_matches_sequential_oracle(eng, ora, shards):
    """configs[4]-shaped corpus (mixed sizes, 50 % duplicates whose twins land in other rounds and on other shards),
    three calls on a group with tiny rounds: every output of every entry, the summed per-issuer counts, the status
    counters and the cardinality of EVERY set equal the sequential oracle's."""
    sets = _device_sets()
    if shards == "all_gpus" and len(sets) < 2:
        pytest.skip("needs >= 2 GPUs")
    devices = sets[0] if shards == "one_gpu_three_shards" else sets[1]
    n = 30000
    cfg = ora.synth_cfg(n, len_mode=1, len_lo=512, len_hi=4096, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    odb = ora.DB(README_FILTER, False)
    cuts = [0, 9000, 9001, 21000, n]
    with eng.GpuCertGroup(devices, table_capacity=1 << 16, issuer_cn_filter=README_FILTER, max_issuers=1024,
                          max_batch_entries=1024, pair_capacity_log2=16) as g:
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            want = odb.process(blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi], NOW_NS)
            got = g.store_batch(blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi], NOW_NS, want_meta=True)
            _check_fields(got, want, hi - lo, FIELDS + ("sha256",) + META, parsed_only=("exp_hour", "serial_off", "serial_len"))
        oc = odb.issuer_counts()
        assert {k: v for k, v in g.issuer_counts().items() if v} == oc
        assert np.array_equal(g.status_counters(), odb.filter_counters())
        used, cap = g.table_stats()
        assert used == sum(oc.values()) and cap == len(devices) * (1 << 16)
        # every shard holds a share (the owner hash spreads the sets)
        per = [m.table_stats()[0] for m in g.members]
        assert all(p > 0 for p in per) and sum(per) == used
        # KnownCertificates.Count() of every set the oracle knows, asked the way storage-statistics does (per set)
        want_all = odb.process(blob, offs, iblob, ioffs, idx, NOW_NS)  # (a second pass: everything known, counts unchanged)
        assert int(want_all.was_unknown.sum()) == 0
        ok = want_all.status == 0
        sets_seen = {(int(h), int(i)) for h, i in zip(want_all.exp_hour[ok], idx[ok])}
        dense = g.register_issuers(iblob, ioffs)
        digests = {i: g.issuer_digest(int(dense[i])) for i in {s[1] for s in sets_seen}}
        assert len(sets_seen) > 1000
        for h, i in sets_seen:
            assert g.get_known_certificates(h, digests[i]).count() == odb.set_cardinality(h, digests[i]), (h, i)
        assert g.get_known_certificates(1, digests[min(digests)]).count() == 0


def test_group_twins_on_different_shards_lower_index_wins(eng, ora):
    """Hand-placed twins: the same certificate at positions that fall into different shards of the same round and into
    different rounds.  Exactly the first occurrence is unknown, whichever shard inserts first."""
    n = 6000
    cfg = ora.synth_cfg(n)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    base = np.arange(n)
    order = np.concatenate([base, base[::-1], base[::7]])  # every certificate at least twice, far apart and adjacent
    ders = [blob[offs[i]:offs[i + 1]].tobytes() for i in order]
    o2 = np.zeros(len(ders) + 1, np.uint64)
    o2[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
    b2 = np.frombuffer(b"".join(ders), np.uint8)
    i2 = idx[order]
    want = ora.DB(b"", True).process(b2, o2, iblob, ioffs, i2, NOW_NS)
    for devices in _device_sets():
        with eng.GpuCertGroup(devices, table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=512) as g:
            got = g.store_batch(b2, o2, iblob, ioffs, i2, NOW_NS)
        _check_fields(got, want, len(ders), FIELDS + ("sha256",))
        first_seen = np.zeros(n, bool)
        for pos, e in enumerate(order):
            if want.status[pos] == 0:
                assert got.was_unknown[pos] == (0 if first_seen[e] else 1)
                first_seen[e] = True


def test_group_pem_preload_evict(eng, ora):
    """The (f) rows through the group: PEM of the new certificates in entry order, warm start from existing sets (owner
    shards receive the preloaded serials), TTL eviction on every shard."""
    n = 5000
    cfg = ora.synth_cfg(n, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    odb = ora.DB(b"", True)
    want = odb.process(blob, offs, iblob, ioffs, idx, NOW_NS)
    with eng.GpuCertGroup([0, 0], table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=700) as g:
        got = g.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS, want_pem=True)
        _check_fields(got, want, n, FIELDS)
        for i in list(np.nonzero(got.was_unknown)[0][:40]) + list(np.nonzero(got.was_unknown == 0)[0][:10]):
            der = blob[offs[i]:offs[i + 1]].tobytes()
            assert got.pem_of(i) == (go_pem(der) if got.was_unknown[i] else b"")
        # Redis TTLs: an hour in the future half of the corpus has expired
        cut = NOW_SEC + 200 * 86400
        assert g.evict_expired(cut) == odb.evict_expired(cut) > 0
        assert {k: v for k, v in g.issuer_counts().items() if v} == {k: v for k, v in odb.issuer_counts().items() if v}
        want2 = odb.process(blob, offs, iblob, ioffs, idx, NOW_NS)
        got2 = g.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
        assert np.array_equal(got2.was_unknown, want2.was_unknown) and 0 < int(got2.was_unknown.sum()) < int(got.was_unknown.sum())
    # warm start: seed a fresh group with some sets of the finished run, then replay
    ok = want.status == 0
    seed_sets = {}
    for i in np.nonzero(ok & (want.was_unknown == 1))[0][:1500]:
        ser = blob[offs[i] + want.serial_off[i]: offs[i] + want.serial_off[i] + want.serial_len[i]].tobytes()
        seed_sets.setdefault((int(want.exp_hour[i]), int(idx[i])), []).append(ser)
    with eng.GpuCertGroup([0, 0, 0], table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=600) as g:
        dense = g.register_issuers(iblob, ioffs)
        for (h, k), serials in seed_sets.items():
            g.preload_known(h, g.issuer_digest(int(dense[k])), serials)
        got3 = g.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
        seeded = {(h, k, s) for (h, k), ss in seed_sets.items() for s in ss}
        for i in np.nonzero(ok)[0]:
            ser = blob[offs[i] + want.serial_off[i]: offs[i] + want.serial_off[i] + want.serial_len[i]].tobytes()
            if (int(want.exp_hour[i]), int(idx[i]), ser) in seeded:
                assert got3.was_unknown[i] == 0
            else:
                assert got3.was_unknown[i] == want.was_unknown[i]
        # the seeded serials count as members of their sets, the rest is added by the replay: the same unique total
        assert sum(g.issuer_counts().values()) == int(want.was_unknown.sum())


def test_group_issuer_registry_is_order_independent(eng, ora):
    """ADVICE r1 (medium): dense issuer indices must not depend on which shard met an issuer first.  The registry lives
    on the device of shard 0 and is shared: registering through different members, in different orders, yields one index
    per issuer, and results do not change."""
    n = 4000
    cfg = ora.synth_cfg(n)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    want = ora.DB(b"", True).process(blob, offs, iblob, ioffs, idx, NOW_NS)
    ni = ioffs.size - 1
    with eng.GpuCertGroup([0, 0], table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=500) as g:
        rev = np.arange(ni)[::-1]
        ders = [iblob[ioffs[k]:ioffs[k + 1]].tobytes() for k in rev]
        ro = np.zeros(ni + 1, np.uint64)
        ro[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
        rb = np.frombuffer(b"".join(ders), np.uint8)
        a = g.members[1].register_issuers(rb[: int(ro[ni // 2])], ro[: ni // 2 + 1])        # half, reversed, through shard 1
        b = g.members[0].register_issuers(iblob, ioffs)                                      # all, in order, through shard 0
        c = g.members[1].register_issuers(iblob, ioffs)
        assert np.array_equal(b, c) and sorted(b.tolist()) == list(range(ni))
        assert np.array_equal(a, b[rev[: ni // 2]])
        assert g.members[0].issuer_digest(int(b[3])) == g.members[1].issuer_digest(int(b[3]))
        got = g.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
        _check_fields(got, want, n, FIELDS)


def test_group_snapshot_and_restore(eng, ora):
    """Checkpoint / resume of the multi-shard form (SURVEY.md §8(f)): every shard's tables + the one issuer registry +
    the group's next index, restored into a NEW group of the same shape; the second half then behaves as if the first
    had run there.  A group of another size (the owner of a set would change) and a member ctx are refused."""
    from ct_mapreduce_b200 import capi
    n = 12000
    cfg = ora.synth_cfg(n, len_mode=1, len_lo=512, len_hi=4096, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    h = n // 2
    odb = ora.DB(README_FILTER, False)
    wa = odb.process(blob, offs[:h + 1], iblob, ioffs, idx[:h], NOW_NS)
    wb = odb.process(blob, offs[h:], iblob, ioffs, idx[h:], NOW_NS)
    kw = dict(table_capacity=1 << 15, issuer_cn_filter=README_FILTER, max_issuers=1024, max_batch_entries=1024, pair_capacity_log2=15)
    for devices in _device_sets():
        with eng.GpuCertGroup(devices, **kw) as g1:
            # register in reverse first: the restored registry must reproduce THESE indices, not first-seen order
            ni = ioffs.size - 1
            ders = [iblob[ioffs[k]:ioffs[k + 1]].tobytes() for k in range(ni)][::-1]
            ro = np.zeros(ni + 1, np.uint64)
            ro[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
            g1.register_issuers(np.frombuffer(b"".join(ders), np.uint8), ro)
            dense1 = g1.register_issuers(iblob, ioffs)
            ga = g1.store_batch(blob, offs[:h + 1], iblob, ioffs, idx[:h], NOW_NS, want_meta=True)
            _check_fields(ga, wa, h, FIELDS + META)
            snap = g1.snapshot().copy()
            with pytest.raises(capi.CtmrError):
                g1.members[0].snapshot()          # a shard alone is not a consistent checkpoint
        with eng.GpuCertGroup(devices, **kw) as g2:
            g2.restore(snap)
            assert np.array_equal(g2.register_issuers(iblob, ioffs), dense1)
            gb = g2.store_batch(blob, offs[h:], iblob, ioffs, idx[h:], NOW_NS, want_meta=True)
            _check_fields(gb, wb, n - h, FIELDS + META)
            assert {k: v for k, v in g2.issuer_counts().items() if v} == odb.issuer_counts()
            assert np.array_equal(g2.status_counters(), odb.filter_counters())
            assert np.array_equal(g2.snapshot(), g2.snapshot())
        other = list(devices) + [devices[0]] if len(devices) < 8 else list(devices)[:-1]
        with eng.GpuCertGroup(other, **kw) as g3:
            with pytest.raises(capi.CtmrError):
                g3.restore(snap)
        with eng.GpuCertGroup(devices, **dict(kw, table_capacity=1 << 14)) as g4:
            with pytest.raises(capi.CtmrError):
                g4.restore(snap)
            with pytest.raises(capi.CtmrError):
                g4.restore(snap[:100])


# ------------------------------------------------------------------------------------------------ one process per GPU
def _peer_worker(rank, world, backend, same_gpu, n):
    import torch
    import torch.distributed as dist
    devno = 0 if same_gpu else rank
    torch.cuda.set_device(devno)
    dev = torch.device("cuda", devno)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi, engine, sharded
    cfg = capi.synth_cfg(world * n * 2, len_mode=1, len_lo=512, len_hi=3000, dup_mode=1)
    iblob, ioffs = engine.synth_issuers(cfg)
    db = engine.GpuCertDatabase(device=devno, table_capacity=1 << 16, issuer_cn_filter=README_FILTER, max_issuers=1024,
                                max_batch_entries=1500)
    sharded.attach_peers(db)
    # issuers registered in a rank-dependent order: the indices must agree anyway (shared device registry)
    ni = ioffs.size - 1
    perm = np.roll(np.arange(ni), 37 * rank)
    ders = [iblob[ioffs[k]:ioffs[k + 1]].tobytes() for k in perm]
    po = np.zeros(ni + 1, np.uint64)
    po[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
    dense_perm = db.register_issuers(np.frombuffer(b"".join(ders), np.uint8), po)
    dense = np.zeros(ni, np.uint32)
    dense[perm] = dense_perm
    res = {"dense": dense}
    # everything the host has to prepare happens BEFORE the collective calls (a rank waiting at a barrier spins on the GPU)
    from oracle import oracle as ora
    m = n - 400 * (world - 1 - rank)   # ragged: the ranks pass different sizes to the host-buffer call
    hb, ho, hi = ora.synth_corpus(ora.synth_cfg(world * n * 2, len_mode=1, len_lo=512, len_hi=3000, dup_mode=1), world * n + rank * n, m)
    blob, offsets, idx, total = engine.synth_corpus_device(cfg, rank * n, n, dev)
    idx_dense = torch.from_numpy(dense.astype(np.int32)).to(dev)[idx.long()]
    status = torch.empty(n, dtype=torch.uint8, device=dev)
    sha = torch.empty((n, 32), dtype=torch.uint8, device=dev)
    exp_hour = torch.empty(n, dtype=torch.int64, device=dev)
    wu = torch.empty(n, dtype=torch.uint8, device=dev)
    fi = torch.empty(n, dtype=torch.uint8, device=dev)
    counts = torch.zeros(ni, dtype=torch.int64, device=dev)
    stat = torch.zeros(capi.ST_COUNT, dtype=torch.int64, device=dev)
    torch.cuda.synchronize(dev)
    dist.barrier()
    # ---- collective HOST-buffer call on the second half of the corpus
    got = db.store_batch(hb, ho, iblob, ioffs, hi, NOW_NS, want_meta=True)
    res["host"] = (m, got.status, got.sha256, got.was_unknown, got.first_issuer_hour, got.first_issuer_dn, got.first_crldp)
    dist.barrier()
    # ---- collective device-resident call: this rank's shard = entries [rank*n, (rank+1)*n) of the corpus; its global
    # indices start above everything the host-buffer call used
    b = capi.DevBatch()
    b.blob, b.blob_bytes, b.offsets, b.n = blob.data_ptr(), total, offsets.data_ptr(), n
    b.issuer_idx, b.issuer_map, b.issuer_map_len = idx_dense.data_ptr(), None, 0
    b.first_index, b.now_unix_ns = 1 << 40, NOW_NS
    o = capi.DevOut(status.data_ptr(), sha.data_ptr(), exp_hour.data_ptr(), None, None, wu.data_ptr(), fi.data_ptr(), None)
    db.process_device(b, o)
    db.peer_allreduce_histogram_device(counts, ni, stat)
    torch.cuda.synchronize(dev)
    db.check_device()
    res["dev"] = (status.cpu().numpy(), sha.cpu().numpy(), wu.cpu().numpy(), fi.cpu().numpy(), counts.cpu().numpy(), stat.cpu().numpy())
    res["counts"] = db.issuer_counts()
    dist.barrier()
    db.close()
    dist.destroy_process_group()
    return res


@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", ["two_processes_one_gpu", "one_process_per_gpu"])
def test_peer_processes_match_sequential_oracle(ora, mode):
    import torch
    from ct_mapreduce_b200 import sharded
    if mode == "one_process_per_gpu":
        if torch.cuda.device_count() < 2:
            pytest.skip("needs >= 2 GPUs")
        world, backend, same = min(torch.cuda.device_count(), 4), "nccl", False
    else:
        world, backend, same = 2, "gloo", True
    n = 6000
    outs = run_ranks(_peer_worker, world, (backend, same, n), timeout=800)
    # the registry gave every rank the same dense index for the same issuer, whatever the registration order
    for r in range(1, world):
        assert np.array_equal(outs[0]["dense"], outs[r]["dense"])
    dense = outs[0]["dense"]
    # ---- oracle over the order the collective calls define
    cfg = ora.synth_cfg(world * n * 2, len_mode=1, len_lo=512, len_hi=3000, dup_mode=1)
    iblob, ioffs = ora.synth_issuers(cfg)
    odb = ora.DB(README_FILTER, False)
    shard = [ora.synth_corpus(cfg, r * n, n) for r in range(world)]

    def run_order(slices, shards):
        ders, idxs = [], []
        for r, lo, hi in slices:
            b, o, i = shards[r]
            ders += [b[o[j]:o[j + 1]].tobytes() for j in range(lo, hi)]
            idxs.append(i[lo:hi])
        offs = np.zeros(len(ders) + 1, np.uint64)
        offs[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
        return odb.process(np.frombuffer(b"".join(ders), np.uint8), offs, iblob, ioffs, np.concatenate(idxs), NOW_NS)

    # ---- 1. the host-buffer collective call, second half of the corpus, ragged sizes
    ms = [outs[r]["host"][0] for r in range(world)]
    shard2 = [ora.synth_corpus(cfg, world * n + r * n, ms[r]) for r in range(world)]
    slices2 = list(sharded.host_batch_order(ms, 1500))
    want2 = run_order(slices2, shard2)
    pos = 0
    for r, lo, hi in slices2:
        m, st, sha, wu, fi, fdn, fcrl = outs[r]["host"]
        k = hi - lo
        for a, bname in ((st, "status"), (sha, "sha256"), (wu, "was_unknown"), (fi, "first_issuer_hour"), (fdn, "first_issuer_dn"),
                         (fcrl, "first_crldp")):
            assert np.array_equal(a[lo:hi], getattr(want2, bname)[pos:pos + k]), (bname, r, lo)
        pos += k
    # ---- 2. the device-resident collective call over the first half (its twins are partly in the second half: known)
    slices = list(sharded.sequential_order(n, world))
    want = run_order(slices, shard)
    pos = 0
    for r, lo, hi in slices:
        st, sha, wu, fi, counts, stat = outs[r]["dev"]
        k = hi - lo
        assert np.array_equal(st[lo:hi], want.status[pos:pos + k])
        assert np.array_equal(sha[lo:hi], want.sha256[pos:pos + k])
        assert np.array_equal(wu[lo:hi], want.was_unknown[pos:pos + k]), (r, lo)
        assert np.array_equal(fi[lo:hi], want.first_issuer_hour[pos:pos + k]), (r, lo)
        pos += k
    oc = odb.issuer_counts()
    for r in range(world):
        counts, stat = outs[r]["dev"][4], outs[r]["dev"][5]
        assert int(counts.sum()) == sum(oc.values()) == int(want.was_unknown.sum()) + int(want2.was_unknown.sum())
        assert np.array_equal(stat.astype(np.uint64), odb.filter_counters())
    # cross-rank duplicates really occurred: some entry is known because of ANOTHER rank's earlier entry
    assert int(want.was_unknown.sum()) < int((want.status == 0).sum())
    # every rank counts the keys it owns: the per-rank counts sum to the oracle's
    total = {}
    for r in range(world):
        for d, v in outs[r]["counts"].items():
            total[d] = total.get(d, 0) + v
    assert {k: v for k, v in total.items() if v} == odb.issuer_counts()


@pytest.mark.parametrize("shards", ["one_gpu_three_shards", "all_gpus"])
def test_group_front_end_matches_oracle(eng, ora, monkeypatch, shards):
    """SURVEY §8(f)-2 on the group path (ctmr_group_process_raw): get-entries pages with every entry kind and malformation,
    small staging budgets (many rounds, one chunk per shard each), several calls, string identities and PEM: every output
    equals the oracle's sequential run over the same pages -- i.e. what ctmr_process_raw returns on one GPU."""
    from conftest import go_pem
    from test_gpu_frontend import check, synth_pages
    sets = _device_sets()
    if shards == "all_gpus" and len(sets) < 2:
        pytest.skip("needs >= 2 GPUs")
    devices = sets[0] if shards == "one_gpu_three_shards" else sets[1]
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(1 << 21))
    n = 9000
    text, lo, ll, xo, xl, _ = synth_pages(ora, n, seed=13, page=700, dup_mode=1)
    odb = ora.DB(README_FILTER, False)
    with eng.GpuCertGroup(devices, issuer_cn_filter=README_FILTER, table_capacity=1 << 16, max_batch_entries=600, max_issuers=1024) as g:
        cuts = [0, 2500, 2501, n]
        for a, b in zip(cuts[:-1], cuts[1:]):
            check(eng, ora, g, odb, text, lo[a:b].copy(), ll[a:b].copy(), xo[a:b].copy(), xl[a:b].copy(), want_meta=True)
        assert {k: v for k, v in g.issuer_counts().items() if v} == {k: v for k, v in odb.issuer_counts().items() if v}
        assert np.array_equal(g.status_counters(), odb.filter_counters())
        per = [m.table_stats()[0] for m in g.members]
        assert all(p > 0 for p in per)
        # a replay through the group: everything known; PEM only for new certificates (none)
        r2 = g.store_raw_entries(text, lo, ll, xo, xl, NOW_NS, want_pem=True)
        assert not r2.path.was_unknown.any() and int(r2.path.pem_off[-1]) == 0
    # PEM of the new certificates, in entry order across the shards
    odb2 = ora.DB(b"", True)
    r_o = ora.raw_process(odb2, text, lo, ll, xo, xl, NOW_NS)
    with eng.GpuCertGroup(devices, log_expired_entries=True, table_capacity=1 << 16, max_batch_entries=500) as g:
        r_g = g.store_raw_entries(text, lo, ll, xo, xl, NOW_NS, want_pem=True)
    assert np.array_equal(r_g.path.was_unknown, r_o.path.was_unknown)
    for i in range(0, n, 7):
        assert r_g.path.pem_of(i) == (go_pem(r_o.leaves[i]) if r_o.path.was_unknown[i] else b""), i
