"""ctmr_process_raw_bodies as a collective call of one process per GPU (include/ctmr_frontend.h "one process per GPU"):
two ranks on one GPU over gloo, each pushing its own bodies through store_raw_bodies on a db attached with
sharded.attach_peers.  Every output of every entry on every rank is compared with the oracle run SEQUENTIALLY over the
order the index rule defines: entry j of rank r's chunk k takes (k * world + r) * E + j, the chunks being those the
library cuts (at most E requested entries each).  The entries each rank's bodies hold are the ones tests/bodies_oracle.py
finds; the front-end fields come from oracle.raw_process on those strings.  Covered: a rank with no bodies, twins
across ranks and rounds, PEM and string identities on one rank only, and a rank whose check fails (the other returns
CTMR_E_PEER_FAILED, nothing changes, no index is taken).  Marked gpu."""

import numpy as np
import pytest

import bodies_oracle as bo
from conftest import NOW_NS, README_FILTER
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

E = 40          # config.max_batch_entries: the front end's entry budget, so E of the index rule
PAGE = 10       # entries per synthetic body
FIELDS = ("status", "was_unknown", "first_issuer_hour", "sha256")
PARSED = ("exp_hour", "serial_off", "serial_len")
META = ("first_issuer_dn", "first_crldp")


def inputs():
    """every rank's batches, the same in the workers and in the parent: {name: (bodies, maxes)}"""
    from test_gpu_bodies import corpus, synth_bodies
    _, a = synth_bodies(120, page=PAGE, seed=31)
    _, c = synth_bodies(60, page=PAGE, seed=32)
    extra = corpus()
    extra = extra[:15] + extra[-3:-1]   # every status: OK, BAD_JSON, BAD_TYPE, TOO_MANY, REPEATED_ENTRIES
    b_bodies = [a[0], a[1].replace(b"/", b"\\/")] + [x for x, _ in extra] + a[2:7]
    b_maxes = [PAGE, PAGE] + [m for _, m in extra] + [PAGE] * 5
    return {
        "A": (a, [PAGE] * len(a)),                            # 12 bodies: three chunks of four
        "B": (b_bodies, b_maxes),                             # escapes, bad bodies, TOO_MANY, REPEATED_ENTRIES
        "C0": (c, [PAGE] * len(c)),                           # twins of C1 on the other rank, in another order
        "C1": (c[::-1], [PAGE] * len(c)),
    }


def chunks_of(maxes, counts):
    """the library's chunks (fit): at most E requested entries and E bodies each (the text budget never binds here);
    returns the entries found per chunk"""
    out, slots, got, n = [], 0, 0, 0
    for m, k in zip(maxes, counts):
        if n and (slots + m > E or n >= E):
            out.append(got)
            slots = got = n = 0
        slots += m
        got += k
        n += 1
    if n:
        out.append(got)
    return out


def _keep(r, pem):
    p = r.path
    out = {f: getattr(p, f) for f in FIELDS + PARSED + META if getattr(p, f, None) is not None}
    for f in ("entry_status", "entry_type", "timestamp_ms", "body_status", "body_entries", "body_first", "leaf_input_off",
              "leaf_input_len", "extra_data_off", "extra_data_len", "escaped"):
        out[f] = getattr(r, f)
    if pem:
        out["pem"] = [p.pem_of(i) for i in range(p.status.size)]
    return out


def _worker(rank, world):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi, engine, sharded
    inp = inputs()
    db = engine.GpuCertDatabase(device=0, table_capacity=1 << 16, issuer_cn_filter=README_FILTER, max_issuers=1024,
                                max_batch_entries=E)
    sharded.attach_peers(db)

    def bodies(k, **kw):
        bs, ms = inp[k]
        offs = np.cumsum([0] + [len(b) for b in bs[:-1]]).astype(np.uint64)
        return db.store_raw_bodies(b"".join(bs), offs, [len(b) for b in bs], ms, NOW_NS, **kw)

    def nothing():
        return db.store_raw_bodies(b"", np.zeros(0, np.uint64), [], [], NOW_NS)

    res = {("idx", 0): db.next_index()}
    dist.barrier()
    # 1. ragged: rank 0 has three chunks, rank 1 none
    r = bodies("A", want_meta=True) if rank == 0 else nothing()
    res[1] = _keep(r, False)
    res["idx", 1] = db.next_index()
    # 2. both ranks; string identities on rank 1 only, PEM on rank 0 only
    r = bodies("B", want_pem=True) if rank == 0 else bodies("A", want_meta=True)
    res[2] = _keep(r, rank == 0)
    res["idx", 2] = db.next_index()
    # 3. twins across ranks and rounds
    r = bodies("C%d" % rank)
    res[3] = _keep(r, False)
    res["idx", 3] = db.next_index()
    # 4. rank 1 passes a body outside its text: it fails, rank 0 returns CTMR_E_PEER_FAILED, nothing changes
    before = (db.table_stats(), db.status_counters().tolist(), db.issuer_counts())
    code = None
    try:
        if rank == 1:
            db.store_raw_bodies(b"{}", [1], [2], [1], NOW_NS)
        else:
            bodies("A")
    except capi.CtmrError as e:
        code = e.code
    res[4] = (code, before == (db.table_stats(), db.status_counters().tolist(), db.issuer_counts()))
    res["idx", 4] = db.next_index()
    # 5. the next good call
    r = bodies("B") if rank == 1 else nothing()
    res[5] = _keep(r, False)
    res["idx", 5] = db.next_index()
    res["counts"] = db.issuer_counts()
    dist.barrier()
    db.close()
    dist.destroy_process_group()
    return res


def _part(ora, inp, k):
    """one rank's batch as the oracle sees it: the bodies' statuses and counts, the twin strings through raw_process"""
    if k is None:
        return dict(chunks=[], leaves=[], iders=[], fe=None, sts=[], cnts=[])
    bs, ms = inp[k]
    text, lo, ll, xo, xl, sts, cnts = bo.twin_batch(bs, ms)
    r = ora.raw_process(ora.DB(README_FILTER, False), text, np.array(lo, np.uint64), np.array(ll, np.uint32),
                        np.array(xo, np.uint64), np.array(xl, np.uint32), NOW_NS)
    return dict(chunks=chunks_of(ms, cnts), leaves=list(r.leaves), iders=list(r.issuer_der), fe=r, sts=sts, cnts=cnts,
                bodies=bs, maxes=ms)


def _run_call(ora, odb, parts, world):
    """the sequential oracle over one collective call; returns per rank (result, positions) and the call's span"""
    from conftest import pack
    from ct_mapreduce_b200 import sharded
    idx, span = sharded.frontend_indices([p["chunks"] for p in parts], E)
    order = sorted((int(idx[r][j]), r, j) for r, p in enumerate(parts) for j in range(len(p["leaves"])))
    if not order:
        return [None] * world, span
    issuers, pos, iidx = [], {}, []
    for _, r, j in order:
        d = parts[r]["iders"][j]
        if d is None:
            iidx.append(0xFFFFFFFF)
            continue
        if d not in pos:
            pos[d] = len(issuers)
            issuers.append(d)
        iidx.append(pos[d])
    blob, offs = pack([parts[r]["leaves"][j] for _, r, j in order])
    ib, io = pack(issuers)
    res = odb.process(blob, offs, ib, io, np.asarray(iidx, np.uint32), NOW_NS)
    at = [np.zeros(len(p["leaves"]), np.int64) for p in parts]
    for g, (_, r, j) in enumerate(order):
        at[r][j] = g
    return [(res, at[r]) for r in range(world)], span


def _check(got, want, part, meta=False, pem=False):
    from conftest import go_pem
    assert got["body_status"].tolist() == part["sts"]
    assert got["body_entries"].tolist() == part["cnts"]
    assert got["body_first"].tolist() == np.cumsum([0] + part["cnts"])[:-1].tolist()
    n = len(part["leaves"])
    assert got["status"].size == n
    if part["fe"] is not None:
        for f in ("entry_status", "entry_type"):
            assert np.array_equal(got[f], getattr(part["fe"], f)[:n]), f
    if want is None or n == 0:
        return
    res, at = want
    for f in FIELDS + (META if meta else ()):
        a, b = got[f], getattr(res, f)[at]
        bad = np.nonzero((a != b).reshape(n, -1).any(axis=1))[0]
        assert bad.size == 0, (f, bad[:10])
    parsed = res.status[at] != 1
    for f in PARSED:
        assert np.array_equal(got[f][parsed], getattr(res, f)[at][parsed]), f
    if pem:
        for i in range(n):
            assert got["pem"][i] == (go_pem(part["leaves"][i]) if res.was_unknown[at][i] else b""), i
    k = 0   # the spans as found, in the rank's text
    offs = np.cumsum([0] + [len(b) for b in part["bodies"][:-1]])
    for body, off, mx in zip(part["bodies"], offs, part["maxes"]):
        for leaf, extra in bo.parse_body(body, mx)[1]:
            for s, o_, l_, bit in ((leaf, "leaf_input_off", "leaf_input_len", 1), (extra, "extra_data_off", "extra_data_len", 2)):
                assert (int(got[o_][k]), int(got[l_][k])) == ((0, 0) if s is None else (int(off) + s.off, s.len)), k
                assert bool(got["escaped"][k] & bit) == bool(s is not None and s.escaped), k
            k += 1


@pytest.mark.timeout(1200)
def test_collective_bodies_match_sequential_oracle(ora):
    world = 2
    outs = run_ranks(_worker, world, timeout=1100)
    from ct_mapreduce_b200 import capi
    inp = inputs()
    odb = ora.DB(README_FILTER, False)
    index = [0]

    def call(names, step, meta=(), pem=()):
        parts = [_part(ora, inp, k) for k in names]
        want, span = _run_call(ora, odb, parts, world)
        for r in range(world):
            _check(outs[r][step], want[r], parts[r], meta=r in meta, pem=r in pem)
        index[0] += span
        assert all(outs[r]["idx", step] == index[0] for r in range(world)), (step, index[0])
        return parts

    assert all(outs[r]["idx", 0] == 0 for r in range(world))
    parts = call(["A", None], 1, meta=(0,))
    assert len(parts[0]["chunks"]) == 3 and outs[1][1]["status"].size == 0
    parts = call(["B", "A"], 2, meta=(1,), pem=(0,))
    assert set(parts[0]["sts"]) >= {0, 1, 2, 3, 4} and outs[0][2]["escaped"].any()
    assert int(outs[0][1]["first_issuer_dn"].sum()) > 0
    assert "first_issuer_dn" not in outs[0][2] and "first_issuer_dn" in outs[1][2]   # A's strings were seen in call 1
    parts = call(["C0", "C1"], 3)
    wu = [outs[r][3]["was_unknown"] for r in range(world)]
    assert int(wu[0].sum()) > 0 and int(wu[1].sum()) > 0     # new certificates on both ranks: each copy's lowest index wins
    assert outs[1][4][0] == capi.E_INVALID and outs[0][4][0] == capi.E_PEER_FAILED
    assert all(outs[r][4][1] for r in range(world)) and all(outs[r]["idx", 4] == index[0] for r in range(world))
    call([None, "B"], 5)
    oc = {k: v for k, v in odb.issuer_counts().items() if v}
    total = {}
    for r in range(world):
        for d, v in outs[r]["counts"].items():
            total[d] = total.get(d, 0) + v
    assert {k: v for k, v in total.items() if v} == oc
