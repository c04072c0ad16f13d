"""Throughput of static-ct-api data tiles (ctmr_process_tiles) against get-entries pages (ctmr_process_raw) on one GPU.

    python tools/bench_tiles.py [--tiles 800] [--steps 5] [--warmup 2]

The same synthetic entries (2/3 x509, 1/3 precert, chains of one or two certificates; tools/bench_frontend.py's corpus)
as full data tiles, written by libctmr's host generator (ctmr_synth_tiles_host) into pinned memory, and as get-entries
pages (ctmr_synth_raw_pages_host).  Times whole calls (host bytes in, host results out) on fresh contexts and prints
one JSON line: entries/s of each format, bytes per entry each sends over PCIe, and the library's CUDA-event split of a
call into front-end kernels (with tile_split's share on its own) and the map/reduce path.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ct_mapreduce_b200 import capi, engine  # noqa: E402

NOW_NS = 1767225600 * 10**9


def make_tiles(n_tiles):
    cfg = capi.synth_cfg(256 * n_tiles)
    iblob, ioffs = engine.synth_issuers(cfg)
    certs = [iblob[int(ioffs[k]):int(ioffs[k + 1])].tobytes() for k in range(cfg.n_issuers)]
    fps = np.frombuffer(b"".join(hashlib.sha256(d).digest() for d in certs), np.uint8).copy()
    L = capi.load()
    need = L.ctmr_synth_tiles_host(C.byref(cfg), 0, n_tiles, capi.ptr(fps), None, 0, None, None)
    pin = capi.PinnedBuffer(need)
    off, ln = np.zeros(n_tiles, np.uint64), np.zeros(n_tiles, np.uint32)
    assert L.ctmr_synth_tiles_host(C.byref(cfg), 0, n_tiles, capi.ptr(fps), pin.addr, need, capi.ptr(off), capi.ptr(ln)) == need
    return pin, off, ln, iblob, ioffs


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def timed(fn, db, warmup, steps):
    fe_ms = path_ms = 0.0
    for it in range(warmup + steps):
        if it == warmup:
            t0 = time.perf_counter()
        r = fn()
        if it >= warmup:
            f, p, launches = db.frontend_profile_last()
            fe_ms += f
            path_ms += p
    return (time.perf_counter() - t0) / steps, fe_ms / steps, path_ms / steps, launches, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=800)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    n = 256 * a.tiles
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from bench_frontend import make_pages
    pin, off, ln, iblob, ioffs = make_tiles(a.tiles)
    data = pin.view()
    index, width = np.arange(a.tiles, dtype=np.uint64), np.full(a.tiles, 256, np.uint16)
    ppin, lo, ll, xo, xl = make_pages(n)
    out = {"metric": "ct_tile_entries_per_sec", "unit": "entries/s", "entries": n, "steps": a.steps, "gpu": gpu_info()}
    with engine.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 22) as db:
        db.register_chain_certs(iblob, ioffs)
        dt, fe_ms, path_ms, launches, r = timed(lambda: db.store_tiles(data, off, ln, index, width, NOW_NS), db, a.warmup, a.steps)
        assert r.tiles_done == a.tiles and int((r.entry_status == 0).sum()) == n
        split_ms = db.tiles_profile_last()   # the last call's: tile_split alone (one serial walker per tile)
        out.update(tiles_split_ms=split_ms)
        out.update(value=n / dt, tiles_ms_per_call=dt * 1e3, tiles_bytes_per_entry=len(data) / n, tiles_h2d_gbs=len(data) / dt / 1e9,
                   tiles_frontend_kernels_ms=fe_ms, tiles_path_ms=path_ms, tiles_frontend_launches=launches)
    with engine.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 22) as db:
        tv = ppin.view()
        dt, fe_ms, path_ms, launches, r = timed(lambda: db.store_raw_entries(tv, lo, ll, xo, xl, NOW_NS), db, a.warmup, a.steps)
        assert int((r.entry_status == 0).sum()) == n
        chars = int(ll.sum()) + int(xl.sum())
        out.update(pages_entries_per_sec=n / dt, pages_ms_per_call=dt * 1e3, pages_bytes_per_entry=len(tv) / n,
                   pages_base64_chars_per_entry=chars / n, pages_frontend_kernels_ms=fe_ms, pages_path_ms=path_ms)
    out["tiles_over_pages"] = out["value"] / out["pages_entries_per_sec"]
    out["note"] = ("whole calls on one fresh ctx per format, pinned host bytes in, host results out; the repeated steps find "
                   "every certificate known after the first")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
