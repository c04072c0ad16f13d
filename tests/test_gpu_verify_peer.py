"""ctmr_revoked_verify on one process per GPU: ranks (two and three on one GPU, two on two GPUs when the box has them)
store their parts of a synthetic corpus and preload serials on the sets they own, build a filter with a collective
ctmr_revoked_cascade, store more, and verify the filter in collective calls with each rank's own CRLs.  Every rank's
counts and list must equal each other's, those of one ctx loaded with every rank's checkpoint part and given the CRLs in
rank order, and verify_model's.  Also: a filter or covered_below that differs on one rank, and a list cap too small on one
rank.  Marked gpu."""
import numpy as np
import pytest

import cascade_model as cm
import crl_build as cb
import test_gpu_cascade_peer as tcp
import test_gpu_verify as tgv
import verify_model as vm
import xchg_model as XM
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

NOW, NOW_NS, HOUR, H, TAIL, KW = tcp.NOW, tcp.NOW_NS, tcp.HOUR, tcp.H, tcp.TAIL, tcp.KW
FRESH = 700   # serials each rank preloads before the filter and the CRLs revoke after it: more than one exchange slice


def _crls(world, rank, dig, known, fresh, day):
    """this rank's CRLs: day 0 revokes a third of issuer 0's and a quarter of issuer 2's corpus serials, dealt to ranks 0
    and 1; day two adds, on the last rank, every fresh serial and a fifth more of issuer 0's"""
    e = lambda s: cb.entry(s, 1767000000)  # noqa: E731
    k0, k2 = known[dig[0]], known[dig[2]]
    per = [[cb.crl(entries=[e(s) for s in k0[::3]])], [cb.crl(entries=[e(s) for s in k2[::4]])]] + [[] for _ in range(world - 2)]
    digs = [[dig[0]], [dig[2]]] + [[] for _ in range(world - 2)]
    if day == 2:
        per[-1].append(cb.crl(entries=[e(s) for s in k0[1::5] + fresh]))
        digs[-1].append(dig[0])
    return per[rank], digs[rank]


def _fresh(world):
    return [bytes([0x31, r]) + int(i).to_bytes(2, "big") for r in range(world) for i in range(FRESH)]


def _out(r):
    return dict(code=0, before=r.before, since=r.since, issuers=r.issuers, levels=r.levels, entries=r.entries(),
                crl_status=r.crl_status.tolist())


def _verify(db, *a, **k):
    from ct_mapreduce_b200 import capi
    try:
        return _out(db.revoked_verify(*a, **k))
    except capi.CtmrError as ex:
        return dict(code=ex.code)


def _worker(rank, world, same_gpu):
    import torch
    import torch.distributed as dist
    dev = 0 if same_gpu else rank
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import engine, sharded
    c = tcp.corpus(world)
    res = {}
    db = engine.GpuCertDatabase(device=dev, **KW)
    sharded.attach_peers(db)
    dense = db.register_issuers(c[3], c[4])
    dig = [db.issuer_digest(int(d)) for d in dense]
    db.store_batch(*tcp.part(c, rank * H, (rank + 1) * H), NOW_NS)
    fresh = _fresh(world)
    db.preload_known(XM.hour_for(int(dense[0]), world, rank, HOUR + 10), dig[0], fresh[rank * FRESH:(rank + 1) * FRESH])
    dist.barrier()
    known = tcp.corpus_serials(c, world, dig)
    crls0, digs0 = _crls(world, rank, dig, known, fresh, 0)
    flt = db.revoked_cascade(crls0, digs0, NOW, b"peer").bytes
    nb = db.next_index()
    db.store_batch(*tcp.part(c, world * H + rank * TAIL, world * H + (rank + 1) * TAIL), NOW_NS)
    crls, digs = _crls(world, rank, dig, known, fresh, 2)
    res["flt"], res["nb"], res["dig"] = flt, nb, dig
    res["clean"] = _verify(db, crls0, digs0, NOW, flt)
    res["day2"] = _verify(db, crls, digs, NOW, flt)
    res["day2_split"] = _verify(db, crls, digs, NOW, flt, covered_below=nb)
    other = cm.build([], [])
    res["bad_filter"] = (_verify(db, crls, digs, NOW, other if rank == 1 else flt), _verify(db, crls, digs, NOW, flt))
    res["bad_below"] = (_verify(db, crls, digs, NOW, flt, covered_below=nb if rank == 1 else nb + 1), _verify(db, crls, digs, NOW, flt))
    n = len(res["day2"].get("entries", []))
    res["short"] = _verify(db, crls, digs, NOW, flt, cap=n - 1 if rank == world - 1 else n + 10)
    res["short_code"] = _short(db, crls, digs, flt, n - 1 if rank == world - 1 else n + 10)
    res["part"] = db.checkpoint().copy()
    db.close()
    dist.barrier()
    dist.destroy_process_group()
    return res


def _short(db, crls, digs, flt, cap):
    """the C call with a list of `cap` records: (rc, n_list)"""
    import ctypes as C
    from ct_mapreduce_b200 import capi, engine
    b, keep = engine._crl_batch(crls, digs)
    lst = np.zeros(max(cap, 1), engine.MISS_DTYPE)
    fb = (C.c_uint8 * len(flt)).from_buffer_copy(flt)
    o = capi.VerifyOut(None, 0, 0, capi.VerifyCounts(), capi.VerifyCounts(), lst.ctypes.data, cap, 0)
    rc = capi.load().ctmr_revoked_verify(db.handle, C.byref(b), NOW, fb, len(flt), None, 0, 2**64 - 1, C.byref(o))
    return rc, int(o.n_list)


def _run(world, same_gpu):
    from ct_mapreduce_b200 import build, capi, engine
    build.build()
    outs = run_ranks(_worker, world, (same_gpu,), timeout=1200)
    o0 = outs[0]
    dig, flt, nb = o0["dig"], o0["flt"], o0["nb"]
    c = tcp.corpus(world)
    known = tcp.corpus_serials(c, world, dig)
    fresh = _fresh(world)
    with engine.GpuCertDatabase(device=0, **dict(KW, table_capacity=1 << 17)) as twin:
        twin.load_checkpoint([outs[r]["part"] for r in range(world)])
        records = tgv._records(twin)
        for name, day, below in (("clean", 0, vm.ALL), ("day2", 2, vm.ALL), ("day2_split", 2, nb)):
            per = [_crls(world, r, dig, known, fresh, day) for r in range(world)]
            crls = [x for p, _ in per for x in p]
            digs = [d for _, ds in per for d in ds]
            want = _verify(twin, crls, digs, NOW, flt, covered_below=below)
            assert want["code"] == 0, name
            lo = 0
            for r in range(world):
                got = outs[r][name]
                assert {k: v for k, v in got.items() if k != "crl_status"} == {k: v for k, v in want.items() if k != "crl_status"}, (name, r)
                k = len(per[r][0])
                assert got["crl_status"] == want["crl_status"][lo:lo + k], (name, r)
                lo += k
            R, S, _, _ = tgv._model(records, crls, digs, set(dig))
            counts, lst = vm.verify(R, S, flt, b"", below)
            assert (want["before"], want["since"], want["entries"]) == (counts["before"], counts["since"], lst), name
            if name == "clean":
                assert want["before"]["missed"] == want["before"]["blocked"] == 0 and want["before"]["revoked"] > 50
            if name == "day2":
                assert len(want["entries"]) > tcp.X and want["before"]["missed"] >= world * FRESH // 2
            if name == "day2_split":
                assert want["since"]["valid"] > 0 and want["entries"] == [e for e in outs[0]["day2"]["entries"] if e[3] < nb]
    n = len(o0["day2"]["entries"])
    for r in range(world):
        o = outs[r]
        for fname in ("bad_filter", "bad_below"):
            got, again = o[fname]
            assert got["code"] == (capi.E_INVALID if r == 1 else capi.E_PEER_FAILED), (fname, r, got)
            assert again == o["day2"], (fname, r)
        assert o["short"] == o["day2"], r                                    # the binding's retry, together on every rank
        assert o["short_code"] == (capi.E_BATCH_TOO_LARGE, n), r


@pytest.mark.timeout(1500)
@pytest.mark.parametrize("world,same_gpu", [(2, True), (3, True), (2, False)], ids=["two_ranks_one_gpu", "three_ranks_one_gpu", "one_rank_per_gpu"])
def test_collective_verify_equals_one_ctx(world, same_gpu):
    import torch
    if not same_gpu and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    _run(world, same_gpu)
