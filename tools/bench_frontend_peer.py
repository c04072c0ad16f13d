"""The get-entries front end on several GPUs, two ways, alternated in one run:

    python -m torch.distributed.run --nproc_per_node N tools/bench_frontend_peer.py [--entries 100000] [--runs 5]

  peer   every rank (one process per GPU) pushes its own synthetic pages through the collective ctmr_process_raw on a
         ctx attached with ctmr_peer_attach: each process feeds its own PCIe link from its own host memory;
  group  rank 0 pushes the same total (every rank's pages, one after the other) through ctmr_group_process_raw on an
         in-process group of the same GPUs, the other ranks idle.

Each rank synthesises --entries distinct entries (libctmr's host generator, pinned memory); the group form's batch is
the concatenation.  A run times --steps calls of each form after --warmup calls (the certificates are known after the
first call in both forms).  --same-gpu puts every rank on GPU 0, which checks the plumbing on a one-GPU box but measures
nothing about PCIe links.  The ranks meet on gloo (a CPU barrier), so an idle rank holds no GPU.  Rank 0 prints one JSON
line: per form the entries/s of each run (in total and per rank), the median, the spread, and the library's CUDA-event
split of a call (frontend_ms, path_ms: the slowest rank or member).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ct_mapreduce_b200 import capi, engine, sharded  # noqa: E402

NOW_NS = 1767225600 * 10**9


def make_pages(first, n, page=1000):
    """entries [first, first + n) of the synthetic corpus as get-entries bodies, in pinned memory"""
    cfg = capi.synth_cfg(1 << 30)
    L = capi.load()
    need = L.ctmr_synth_raw_pages_host(C.byref(cfg), first, n, page, None, 0, None, None, None, None)
    pin = capi.PinnedBuffer(need)
    lo, ll = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    xo, xl = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    got = L.ctmr_synth_raw_pages_host(C.byref(cfg), first, n, page, pin.addr, need, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl))
    assert got == need
    return pin, lo, ll, xo, xl


def gpu_info():
    """the card and its power limit, read (not set) with nvidia-smi"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=int, default=100000, help="entries per rank and call")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--same-gpu", action="store_true")
    a = ap.parse_args()
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = 0 if a.same_gpu else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(dev)
    devices = [0 if a.same_gpu else r for r in range(world)]   # one process per GPU on one box: LOCAL_RANK == rank
    n = a.entries
    kw = dict(log_expired_entries=True, table_capacity=1 << 22)
    # ---- peer form: this rank's own pages
    pages = make_pages(rank * n, n)
    pdb = engine.GpuCertDatabase(device=dev, **kw)
    sharded.attach_peers(pdb)
    # ---- group form: rank 0 holds every rank's pages, one after the other
    if rank == 0:
        parts = [pages] + [make_pages(r * n, n) for r in range(1, world)]
        text = np.concatenate([p[0].view() for p in parts])
        base = np.cumsum([0] + [p[0].nbytes for p in parts[:-1]]).astype(np.uint64)
        gpages = capi.PinnedBuffer(text.size)
        gpages.view()[:] = text
        glo = np.concatenate([p[1] + b for p, b in zip(parts, base)])
        gxo = np.concatenate([p[3] + b for p, b in zip(parts, base)])
        gll = np.concatenate([p[2] for p in parts])
        gxl = np.concatenate([p[4] for p in parts])
        group = engine.GpuCertGroup(devices, **kw)

    def peer_call():
        r = pdb.store_raw_entries(pages[0].view(), *pages[1:], NOW_NS)
        assert int((r.entry_status == 0).sum()) == n
        return pdb.frontend_profile_last()[:2]

    def group_call():
        r = group.store_raw_entries(gpages.view(), glo, gll, gxo, gxl, NOW_NS)
        assert int((r.entry_status == 0).sum()) == world * n
        prof = [m.frontend_profile_last()[:2] for m in group.members]
        return max(p[0] for p in prof), max(p[1] for p in prof)

    results = {"peer": [], "group": []}
    for run in range(a.runs):
        for form in ("peer", "group"):
            dist.barrier()
            fe_ms = path_ms = 0.0
            for it in range(a.warmup + a.steps):
                if it == a.warmup:
                    dist.barrier()
                    t0 = time.perf_counter()
                if form == "peer":
                    f, p = peer_call()
                elif rank == 0:
                    f, p = group_call()
                else:
                    f = p = 0.0
                if it >= a.warmup:
                    fe_ms, path_ms = fe_ms + f, path_ms + p
            if form == "peer":
                dist.barrier()   # the slowest rank ends the collective calls
            dt = (time.perf_counter() - t0) / a.steps
            got = [None] * world
            dist.all_gather_object(got, (dt, fe_ms / a.steps, path_ms / a.steps))
            dt = max(g[0] for g in got) if form == "peer" else got[0][0]
            prof = got if form == "peer" else got[:1]
            results[form].append({"entries_per_sec": world * n / dt, "entries_per_sec_per_rank": n / dt, "ms_per_call": dt * 1e3,
                                  "frontend_ms": max(g[1] for g in prof), "path_ms": max(g[2] for g in prof)})
    if rank == 0:
        out = {"metric": "ct_raw_entries_per_sec_multi_gpu", "unit": "entries/s", "world": world, "entries_per_rank": n,
               "same_gpu": a.same_gpu, "gpu": gpu_info(), "runs": a.runs, "steps": a.steps}
        for form, rs in results.items():
            v = [r["entries_per_sec"] for r in rs]
            out[form] = {"median_entries_per_sec": statistics.median(v), "spread": (max(v) - min(v)) / statistics.median(v),
                         "median_entries_per_sec_per_rank": statistics.median(r["entries_per_sec_per_rank"] for r in rs),
                         "median_frontend_ms": statistics.median(r["frontend_ms"] for r in rs),
                         "median_path_ms": statistics.median(r["path_ms"] for r in rs), "runs": rs}
        print(json.dumps(out))
        group.close()
    pdb.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
