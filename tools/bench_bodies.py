"""Whole get-entries bodies (ctmr_process_raw_bodies) against precomputed spans (ctmr_process_raw) and the host scan
that finds those spans today, on one GPU.

    python tools/bench_bodies.py [--entries 204800] [--page 1000] [--steps 3] [--warmup 1] [--out DIR]

The same synthetic entries (ctmr_synth_raw_pages_host, pages of 1,000 written into pinned memory), three rows
alternated in one command, `--steps` alternations after `--warmup`:
  (a) host: a C++ restatement of go/ctmr/frontend.go RawPages.AppendLog (copy the body into pinned memory, then
      bytes.Index for each key, IndexByte for the closing quote and for a backslash), at 1 thread and at the thread
      count whose time is below row (c)'s call;
  (b) ctmr_process_raw on the spans the generator wrote (the e2e pages row of tools/bench_tiles.py);
  (c) ctmr_process_raw_bodies on the bodies.
Each db holds every entry after the first call, so the timed calls are steady state (all known).  Prints one JSON line
with medians, min and max per row, frontend_ms and json_ms, and the card's name and power limit from the same run.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ct_mapreduce_b200 import capi, engine  # noqa: E402

NOW_NS = 1767225600 * 10**9

SCAN_CPP = r"""
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>
// RawPages.AppendLog per body: copy into the pinned buffer, then the spans of each key (bytes.Index, IndexByte '"',
// IndexByte '\\' over the string); the counts must agree.  Returns the entries found, -1 on a mismatch or an escape.
static long scan_one(const uint8_t* b, size_t n) {
    static const char* keys[2] = {"\"leaf_input\":\"", "\"extra_data\":\""};
    long cnt[2] = {0, 0};
    for (int k = 0; k < 2; ++k) {
        const size_t kl = strlen(keys[k]);
        const uint8_t* p = b;
        const uint8_t* end = b + n;
        for (;;) {
            const uint8_t* m = (const uint8_t*)memmem(p, end - p, keys[k], kl);
            if (!m) break;
            const uint8_t* s = m + kl;
            const uint8_t* q = (const uint8_t*)memchr(s, '"', end - s);
            if (!q) return -1;
            if (memchr(s, '\\', q - s)) return -1;
            ++cnt[k];
            p = q;
        }
    }
    return cnt[0] == cnt[1] ? cnt[0] : -1;
}
extern "C" long scan_bodies(const uint8_t* text, const uint64_t* off, const uint32_t* len, uint64_t n, uint8_t* dst, int threads) {
    std::vector<long> found(threads, 0);
    std::vector<std::thread> th;
    for (int t = 0; t < threads; ++t)
        th.emplace_back([&, t] {
            for (uint64_t i = t; i < n; i += threads) {
                memcpy(dst + off[i], text + off[i], len[i]);
                const long c = scan_one(dst + off[i], len[i]);
                found[t] = c < 0 || found[t] < 0 ? -1 : found[t] + c;
            }
        });
    for (auto& x : th) x.join();
    long s = 0;
    for (long f : found) s = f < 0 || s < 0 ? -1 : s + f;
    return s;
}
"""


def gpu_info():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip()


def load_scan(tmp):
    src, so = os.path.join(tmp, "scan.cpp"), os.path.join(tmp, "scan.so")
    with open(src, "w") as f:
        f.write(SCAN_CPP)
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", src, "-o", so], check=True)
    L = C.CDLL(so)
    L.scan_bodies.restype = C.c_long
    L.scan_bodies.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int]
    return L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=int, default=204800)
    ap.add_argument("--page", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, page = a.entries, a.page
    L = capi.load()
    cfg = capi.synth_cfg(n)
    need = L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, page, None, 0, None, None, None, None)
    pin = capi.PinnedBuffer(need)
    lo, ll, xo, xl = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    assert L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, page, pin.addr, need, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl)) == need
    text = pin.view()
    starts = np.array([int(lo[k]) - len(b'{"entries":[{"leaf_input":"') for k in range(0, n, page)] + [need], np.uint64)
    b_off, b_len = starts[:-1].copy(), np.diff(starts).astype(np.uint32)
    b_max = np.full(b_off.size, page, np.uint32)
    dst = capi.PinnedBuffer(need)
    rows = {"a1": [], "b": [], "c": [], "b_fe": [], "c_fe": [], "c_json": []}
    with tempfile.TemporaryDirectory() as tmp:
        scan = load_scan(tmp)
        threads = [1, 2, 4, 8, 16, 32, 64]
        rows.update({"a%d" % t: [] for t in threads})
        with engine.GpuCertDatabase(table_capacity=1 << 22, log_expired_entries=True) as db_b, \
                engine.GpuCertDatabase(table_capacity=1 << 22, log_expired_entries=True) as db_c:
            for it in range(a.warmup + a.steps):
                for t in threads:
                    t0 = time.perf_counter()
                    got = scan.scan_bodies(pin.addr, capi.ptr(b_off), capi.ptr(b_len), b_off.size, dst.addr, t)
                    dt = time.perf_counter() - t0
                    assert got == n, got
                    if it >= a.warmup:
                        rows["a%d" % t].append(dt)
                t0 = time.perf_counter()
                rb = db_b.store_raw_entries(text, lo, ll, xo, xl, NOW_NS)
                dt = time.perf_counter() - t0
                fb = db_b.frontend_profile_last()[0]
                t0 = time.perf_counter()
                rc = db_c.store_raw_bodies(text, b_off, b_len, b_max, NOW_NS)
                dc = time.perf_counter() - t0
                fc, jc = db_c.frontend_profile_last()[0], db_c.bodies_profile_last()
                assert rc.n_entries == n and np.array_equal(rc.entry_status, rb.entry_status)
                assert np.array_equal(rc.path.status, rb.path.status) and np.array_equal(rc.path.sha256, rb.path.sha256)
                if it >= a.warmup:
                    rows["b"].append(dt)
                    rows["c"].append(dc)
                    rows["b_fe"].append(fb)
                    rows["c_fe"].append(fc)
                    rows["c_json"].append(jc)

    def stat(v, scale=1.0):
        return {"median": statistics.median(v) * scale, "min": min(v) * scale, "max": max(v) * scale}
    c_med = statistics.median(rows["c"])
    keep_up = next((t for t in threads if statistics.median(rows["a%d" % t]) <= c_med), None)
    res = {
        "gpu": gpu_info(), "entries": n, "page": page, "bodies": int(b_off.size), "text_bytes": int(need), "steps": a.steps,
        "a_host_scan_ms": {str(t): stat(rows["a%d" % t], 1e3) for t in threads},
        "a_threads_to_keep_up_with_c": keep_up,
        "b_process_raw_ms": stat(rows["b"], 1e3), "b_entries_per_s": n / statistics.median(rows["b"]),
        "b_frontend_ms": stat(rows["b_fe"]),
        "c_process_raw_bodies_ms": stat(rows["c"], 1e3), "c_entries_per_s": n / c_med,
        "c_frontend_ms": stat(rows["c_fe"]), "c_json_ms": stat(rows["c_json"]),
        "host_cpus": os.cpu_count(),
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_bodies.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
