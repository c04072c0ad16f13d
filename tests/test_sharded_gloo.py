"""The N>1 path on CPU: world_size-2 gloo runs of what the host language owns in the multi-GPU form
(ct_mapreduce_b200/sharded.py) plus an executable model of the exchange protocol the library runs on the GPUs.

  * attach_peers: the peer handles travel once over torch.distributed, in rank order, and every rank attaches
    with its own rank / world (production: NCCL; here: gloo and a recording stand-in for the ctx).
  * the round / index arithmetic (sequential_order, host_batch_order, call_index_span): the order a collective call
    is equivalent to -- the thing the GPU parity tests and bench.py build their oracle input from.
  * the protocol itself, modelled in numpy with gloo collectives standing in for peer memory: per round, every rank
    routes the keys of its slice to owner = key_owner(exp_hour, issuer) (csrc/ctmr_device.cuh), appends them to the
    owner's per-source inbox region, [barrier], the owner inserts its inbox + its own keys and resolves
    lowest-index-wins, [barrier], the bits come back BY POSITION.  With the global index
    first_index + (round * world + rank) * E + j the result must equal the oracle run sequentially over
    sequential_order() -- and a deliberately broken variant (resolve before every rank's appends have landed) must not.
"""
import numpy as np
import pytest
import torch.distributed as dist

from conftest import NOW_NS, README_FILTER
from peer_ranks import run_ranks

M64 = (1 << 64) - 1


def mix64(z):
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def key_owner(exp_hour, issuer, world):
    """ctmr::key_owner (csrc/ctmr_device.cuh): owner of the Redis set serials::<expDate>::<issuer>."""
    return mix64(((issuer & 0xFFFFFFFF) << 32) | (exp_hour & 0xFFFFFFFF)) % world


class RecordingCtx:
    """Stand-in for engine.GpuCertDatabase in attach_peers: records what the host logic hands to the C ABI."""

    def __init__(self, rank):
        self.rank, self.attached = rank, None

    def peer_export(self, world):
        return bytes([self.rank, world]) + b"\0" * 254   # 256-byte handle, tagged with its rank

    def peer_attach(self, rank, world, handles):
        self.attached = (rank, world, [h[0] for h in handles], [h[1] for h in handles])


def _model_worker(rank, world, n, rounds, broken):
    from ct_mapreduce_b200 import sharded
    from oracle import oracle as ora
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        # ---- 1. handle exchange
        ctx = RecordingCtx(rank)
        assert sharded.attach_peers(ctx) == (rank, world)
        assert ctx.attached == (rank, world, list(range(world)), [world] * world)
        # ---- 2. the protocol over this rank's shard [rank*n, (rank+1)*n) of one corpus with cross-rank twins
        cfg = ora.synth_cfg(world * n, len_mode=1, len_lo=512, len_hi=2048, dup_mode=1)
        blob, offs, idx = ora.synth_corpus(cfg, rank * n, n)
        iblob, ioffs = ora.synth_issuers(cfg)
        mp_ = ora.DB(README_FILTER, False).process(blob, offs, iblob, ioffs, idx, NOW_NS)   # the map half's per-entry outputs
        keys = []
        for j in range(n):
            ser = blob[offs[j] + mp_.serial_off[j]: offs[j] + mp_.serial_off[j] + mp_.serial_len[j]].tobytes()
            keys.append((int(mp_.exp_hour[j]), int(idx[j]), ser) if mp_.status[j] == 0 else None)
        E = sharded.round_entries(n, rounds)
        table, pairs, counts = {}, {}, {}          # this rank's shard of the state: key -> lowest index, (issuer,hour) -> lowest NEW index
        was_unknown = np.zeros(n, np.uint8)
        first = np.zeros(n, np.uint8)
        for k in range(rounds):
            lo, hi = min(n, k * E), min(n, (k + 1) * E)
            base = (k * world + rank) * E                      # first_index = 0
            outbox = [[] for _ in range(world)]                # records for owner o: (index, key), appended in entry order
            rev = [[] for _ in range(world)]
            for j in range(lo, hi):
                if keys[j] is None:
                    continue
                o = key_owner(keys[j][0], keys[j][1], world)
                outbox[o].append((base + j - lo, keys[j]))
                rev[o].append(j)

            def insert_all(inbox):
                for src in range(world):
                    for gi, key in inbox[src]:
                        table[key] = min(table.get(key, gi), gi)

            if broken:   # resolve after the OWN appends only: a lower index from the other rank arrives too late
                own = [outbox[rank] if s == rank else [] for s in range(world)]
                insert_all(own)
            inbox = [None] * world                             # inbox[src] = what rank src appended for me
            for o in range(world):                             # "peer stores": every rank's region for owner o
                got = [None] * world
                dist.all_gather_object(got, outbox[o])
                if o == rank:
                    inbox = got
            # -- sync 1 is the gather above --
            resolved = [[] for _ in range(world)]
            if broken:
                bits_own = [(1 if table[key] == gi else 0) for gi, key in inbox[rank]]
            insert_all(inbox)
            for src in range(world):
                for pos, (gi, key) in enumerate(inbox[src]):
                    unk = 1 if table[key] == gi else 0
                    if broken and src == rank:
                        unk = bits_own[pos]
                    if unk:
                        counts[key[1]] = counts.get(key[1], 0) + 1
                        pk = (key[1], key[0])
                        pairs[pk] = min(pairs.get(pk, gi), gi)
                    resolved[src].append([unk, gi, key])
            for src in range(world):                           # first_issuer_hour after every pair insert of the round
                for rec in resolved[src]:
                    rec.append(1 if rec[0] and pairs[(rec[2][1], rec[2][0])] == rec[1] else 0)
            # -- sync 2; the source pulls its region of every owner's outbox, bits by position --
            for o in range(world):
                back = [None] * world
                dist.all_gather_object(back, [[(r[0], r[3]) for r in resolved[s]] for s in range(world)])
                mine = back[o][rank]
                assert len(mine) == len(rev[o])
                for pos, (unk, fst) in enumerate(mine):
                    was_unknown[rev[o][pos]] = unk
                    first[rev[o][pos]] = fst
        tot = [None] * world
        dist.all_gather_object(tot, counts)                    # the histogram merge: ownership is disjoint, sums are exact
        merged = {}
        for c in tot:
            for i, v in c.items():
                merged[i] = merged.get(i, 0) + v
        dist.barrier()
        return was_unknown, first, merged
    finally:
        dist.destroy_process_group()


def _run_model(ora, broken):
    from ct_mapreduce_b200 import sharded
    world, n, rounds = 2, 3000, 4
    outs = run_ranks(_model_worker, world, (n, rounds, broken), timeout=300)
    cfg = ora.synth_cfg(world * n, len_mode=1, len_lo=512, len_hi=2048, dup_mode=1)
    iblob, ioffs = ora.synth_issuers(cfg)
    shards = [ora.synth_corpus(cfg, r * n, n) for r in range(world)]
    ders, idxs = [], []
    order = list(sharded.sequential_order(n, world, rounds))
    for r, lo, hi in order:
        b, o, i = shards[r]
        ders += [b[o[j]:o[j + 1]].tobytes() for j in range(lo, hi)]
        idxs.append(i[lo:hi])
    offs = np.zeros(len(ders) + 1, np.uint64)
    offs[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
    odb = ora.DB(README_FILTER, False)
    want = odb.process(np.frombuffer(b"".join(ders), np.uint8), offs, iblob, ioffs, np.concatenate(idxs), NOW_NS)
    mism = 0
    pos = 0
    for r, lo, hi in order:
        k = hi - lo
        mism += int((outs[r][0][lo:hi] != want.was_unknown[pos:pos + k]).sum())
        mism += int((outs[r][1][lo:hi] != want.first_issuer_hour[pos:pos + k]).sum())
        pos += k
    return mism, outs, want, odb, cfg


@pytest.mark.timeout(600)
def test_exchange_protocol_equals_the_sequential_reference(ora):
    mism, outs, want, odb, cfg = _run_model(ora, broken=False)
    assert mism == 0
    assert int(want.was_unknown.sum()) < int((want.status == 0).sum())   # cross-rank twins exist: some entries are known
    # merged per-issuer histogram == the oracle's Count() sums (synthetic issuer k has digest order = index order)
    dig = {}
    from oracle import oracle
    iblob, ioffs = oracle.synth_issuers(cfg)
    oc = odb.issuer_counts()
    assert sum(outs[0][2].values()) == sum(oc.values()) == int(want.was_unknown.sum())
    assert outs[0][2] == outs[1][2]


@pytest.mark.timeout(600)
def test_resolving_before_the_barrier_is_detectably_wrong(ora):
    """The model has teeth: if an owner resolves its own keys before the other rank's appends of the round have landed,
    some later twin is reported unknown -- so a passing run above really depends on sync 1."""
    mism, *_ = _run_model(ora, broken=True)
    assert mism > 0


def test_round_arithmetic():
    from ct_mapreduce_b200 import sharded
    assert sharded.round_entries(10, 4) == 4 and sharded.round_entries(13, 4) == 4 and sharded.round_entries(1, 8) == 1
    assert sharded.round_entries(10_000_000, 8) == 1_379_311 and sharded.round_entries(9, 2) == 5
    assert sharded.call_index_span(10, 3, 4) == 3 * 4 * 4
    from ct_mapreduce_b200 import capi   # the Python restatement and the library agree (no GPU needed for this entry point)
    for n in (1, 7, 4096, 10_000_000, 125_000_001):
        assert sharded.round_entries(n) == sharded.round_entries(n, capi.peer_rounds())
    # every entry of every rank appears exactly once; rounds ascend, ranks ascend inside a round
    for n, world, rounds in ((10, 3, 4), (7, 2, 8), (64, 8, 8), (5, 1, 4)):
        seen = [np.zeros(n, int) for _ in range(world)]
        last = (-1, -1)
        e = sharded.round_entries(n, rounds)
        for r, lo, hi in sharded.sequential_order(n, world, rounds):
            assert hi > lo and hi - lo <= e and lo % e == 0 and (hi - lo == e or hi == n)
            k = lo // e
            assert (k, r) > last
            last = (k, r)
            seen[r][lo:hi] += 1
        assert all((s == 1).all() for s in seen)
        # the library's global index is strictly increasing along this order (first_index = 0)
        prev = -1
        for r, lo, hi in sharded.sequential_order(n, world, rounds):
            gi = ((lo // e) * world + r) * e
            assert gi > prev
            prev = gi + (hi - lo) - 1
    # ragged host-buffer call: every rank runs max(rounds); short ranks contribute empty rounds
    got = list(sharded.host_batch_order([5, 2, 0], 2))
    assert got == [(0, 0, 2), (1, 0, 2), (0, 2, 4), (0, 4, 5)]
