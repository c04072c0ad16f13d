#!/usr/bin/env python3
"""Where K_map's time goes: the streaming map kernel timed whole and with the DER walk, the SHA-256 compression or both
compiled out, on the bench's flagship corpus (configs[1]: 10 M x ~1.5 KB certificates, the bench's seed).

    python tools/kmap_split.py [--entries N] [--steps K] [--warmup W] [--repeats R] [--build-dir DIR]

Four experiment libraries are compiled from tools/kmap_split.cu (ctmr_map.cu under a compile-time policy, the flags of
ct_mapreduce_b200/build.py) into the build directory; libctmr.so is not touched and has no such switch.

    full       the shipped kernel
    no_walk    walk_advance never called, every entry passed as parsed with a key made of its entry number (status,
               expiry hour, serial and dedup outputs are WRONG by construction; copies, hash, insert, stores as shipped)
    no_hash    the 17 loads and byte swaps of each block kept, the compression replaced by XORs (digests WRONG)
    copy_only  both

Each variant runs the map half of a bench step (the table emptied, 8 rounds, each K_map launch behind its length
ordering, on two alternating streams; no reduce half), timed with CUDA events.  The variants are run in turn, `repeats`
times over.  One JSON line: ms per step of every repeat, median and spread per variant, full - no_walk (the most any
walker work can return), the card's name, power limit and SM clock sampled during the run, registers and spills of
each variant's kernel.  Needs a GPU.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import re
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = {  # name -> (defines, what is wrong with its outputs)
    "full": ([], None),
    "no_walk": (["-DCTMR_KMAP_SKIP_WALK=1"], "no DER walk: status forced to OK, expiry hour 0, serial = entry number"),
    "no_hash": (["-DCTMR_KMAP_SKIP_HASH=1"], "no SHA-256 compression: digests are XOR folds"),
    "copy_only": (["-DCTMR_KMAP_SKIP_WALK=1", "-DCTMR_KMAP_SKIP_HASH=1"], "neither walk nor compression"),
}
ROUNDS = 8  # ctmr_process_device cuts a batch of 2^21 entries or more into 8 rounds
NOW_SEC = 1767225600
SEED = 20260922


class Args(C.Structure):
    _fields_ = [("blob", C.c_void_p), ("blob_bytes", C.c_uint64), ("offsets", C.c_void_p), ("issuer_idx", C.c_void_p),
                ("n", C.c_uint64), ("status", C.c_void_p), ("sha256", C.c_void_p), ("exp_hour", C.c_void_p),
                ("keys", C.c_void_p), ("slot_of", C.c_void_p), ("order", C.c_void_p), ("len_hist", C.c_void_p),
                ("table", C.c_void_p), ("table_slots", C.c_uint64), ("status_counts", C.c_void_p),
                ("error_flag", C.c_void_p), ("now_sec", C.c_int64), ("rounds", C.c_uint32), ("per_round", C.c_uint32),
                ("sm_count", C.c_int32)]


def build_variant(name, build_dir):
    """Compiles one experiment library; returns (path, registers, spill bytes) of its map_stream_kernel."""
    from ct_mapreduce_b200 import build
    out = os.path.join(build_dir, f"libkmap_{name}.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + VARIANTS[name][0] + \
          ["-Xptxas", "-v", os.path.join(ROOT, "tools", "kmap_split.cu"), "-o", out, "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError(f"nvcc failed building the {name} variant")
    m = re.search(r"Function properties for \S*map_stream_kernel\S*\s+\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                  r.stderr)
    spills = int(m.group(1)) + int(m.group(2))
    cuobjdump = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    usage = subprocess.run([cuobjdump, "--dump-resource-usage", out], capture_output=True, text=True, check=True).stdout
    m = re.search(r"Function \S*map_stream_kernel\S*:\s*\n\s*REG:(\d+)", usage)
    return out, int(m.group(1)), spills


class ClockSampler:
    """name, power limit and SM clock from nvidia-smi (queries only) while the variants run"""

    def __init__(self, index):
        self.rows = []
        self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,power.draw",
                                      "--format=csv,noheader,nounits", "-lms", "200", "-i", str(index)],
                                     stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        self.thread = threading.Thread(target=lambda: self.rows.extend(self.proc.stdout), daemon=True)
        self.thread.start()

    def stop(self):
        self.proc.terminate()
        self.proc.wait()
        self.thread.join(timeout=2)
        rows = [[f.strip() for f in r.split(",")] for r in self.rows]
        rows = [r for r in rows if len(r) == 5]
        sm = sorted(float(r[2]) for r in rows)
        return {"gpu": rows[0][0], "power_limit_w": float(rows[0][1]), "sm_mhz_median": sm[len(sm) // 2], "sm_mhz_min": sm[0],
                "sm_max_mhz": float(rows[0][3]), "power_w_max": max(float(r[4]) for r in rows), "samples": len(rows)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--build-dir", default=os.path.join(ROOT, "tools", "build", "kmap_split"))
    args = ap.parse_args()
    os.makedirs(args.build_dir, exist_ok=True)
    built = {name: build_variant(name, args.build_dir) for name in VARIANTS}

    import torch
    from ct_mapreduce_b200 import capi, engine
    if not torch.cuda.is_available():
        sys.exit("kmap_split needs a GPU")
    dev = torch.device("cuda", 0)
    n = args.entries
    cfg = capi.synth_cfg(n, seed=SEED, len_mode=0, len_lo=1436, len_hi=1564, dup_mode=0)
    blob, offsets, issuer_idx, total_bytes = engine.synth_corpus_device(cfg, 0, n, dev)
    slots = 1 << 20
    while slots < 2 * n:
        slots <<= 1
    buf = dict(status=torch.empty(n, dtype=torch.uint8, device=dev), sha=torch.empty((n, 32), dtype=torch.uint8, device=dev),
               exp_hour=torch.empty(n, dtype=torch.int64, device=dev), keys=torch.empty((n, 64), dtype=torch.uint8, device=dev),
               slot_of=torch.empty(n, dtype=torch.int32, device=dev), order=torch.empty(n, dtype=torch.int32, device=dev),
               len_hist=torch.zeros(ROUNDS * 256, dtype=torch.int32, device=dev),
               table=torch.empty((slots, 64), dtype=torch.uint8, device=dev),
               counts=torch.zeros(64, dtype=torch.int64, device=dev), err=torch.zeros(1, dtype=torch.int32, device=dev))
    per_round = (4 * n + 4 * ROUNDS - 4) // (4 * ROUNDS - 3) if n >= 1 << 21 else n  # device_round_entries (ctmr_api.cu)
    a = Args(blob.data_ptr(), total_bytes, offsets.data_ptr(), issuer_idx.data_ptr(), n, buf["status"].data_ptr(),
             buf["sha"].data_ptr(), buf["exp_hour"].data_ptr(), buf["keys"].data_ptr(), buf["slot_of"].data_ptr(),
             buf["order"].data_ptr(), buf["len_hist"].data_ptr(), buf["table"].data_ptr(), slots, buf["counts"].data_ptr(),
             buf["err"].data_ptr(), NOW_SEC, ROUNDS if n >= 1 << 21 else 1, per_round,
             torch.cuda.get_device_properties(dev).multi_processor_count)
    libs = {}
    for name, (path, _, _) in built.items():
        libs[name] = C.CDLL(path, mode=os.RTLD_LOCAL)
        libs[name].kmap_split_run.argtypes = [C.POINTER(Args), C.c_int, C.POINTER(C.c_float)]

    def run(name, steps):
        ms = C.c_float(0)
        rc = libs[name].kmap_split_run(C.byref(a), steps, C.byref(ms))
        if rc:
            raise RuntimeError(f"{name}: CUDA error {rc}")
        return float(ms.value)

    # the harness drives the kernel the way the library does: the shipped variant's outputs are the real ones
    run("full", 1)
    torch.cuda.synchronize(dev)
    ok_share = float((buf["status"] == 0).float().mean())  # the corpus holds some CA certificates, which are filtered out
    assert int(buf["err"].item()) == 0 and ok_share > 0.9, f"full variant: statuses {torch.bincount(buf['status'].int()).tolist()}"
    offs = offsets[:5].cpu().tolist()
    for i in range(4):
        der = blob[offs[i]:offs[i + 1]].cpu().numpy().tobytes()
        assert hashlib.sha256(der).digest() == buf["sha"][i].cpu().numpy().tobytes(), "full variant: wrong digest"

    for name in VARIANTS:
        run(name, args.warmup)
    clocks = ClockSampler(0)
    times = {name: [] for name in VARIANTS}
    for _ in range(args.repeats):
        for name in VARIANTS:
            times[name].append(round(run(name, args.steps), 4))
    clk = clocks.stop()

    def med(v):
        return sorted(v)[len(v) // 2]

    res = {"tool": "kmap_split", "entries": n, "bytes": total_bytes, "steps": args.steps, "warmup": args.warmup,
           "repeats": args.repeats, "rounds": int(a.rounds), "stored_share": round(ok_share, 4), **clk, "variants": {}}
    for name, (_, regs, spills) in built.items():
        t = times[name]
        res["variants"][name] = {"ms_per_step": t, "median_ms": med(t), "spread_ms": round(max(t) - min(t), 4),
                                 "registers": regs, "spill_bytes": spills, "outputs_wrong": VARIANTS[name][1]}
    full, nw = med(times["full"]), med(times["no_walk"])
    res["full_minus_no_walk_ms"] = round(full - nw, 4)
    res["full_minus_no_walk_share"] = round((full - nw) / full, 4)
    res["full_minus_no_hash_ms"] = round(full - med(times["no_hash"]), 4)
    res["full_gb_per_s"] = round(total_bytes / full / 1e6, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
