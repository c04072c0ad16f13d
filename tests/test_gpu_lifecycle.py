"""Who owns the library's CUDA resources, checked from outside: every device buffer, pinned host buffer, stream and event
libctmr creates is counted by an LD_PRELOAD shim of the CUDA runtime (tests/cpp/cuda_shim.cpp).

- Lifetime: every lazily built part of a ctx is reached; repeating a call leaves the live counts unchanged, and the
  number of creations a repeated call makes is what the library needs per call (EXPECTED_REPEAT); destroy leaves none.
- Injected failures: for every creation N of every kind a call makes on a fresh ctx, that creation fails.  The call must
  return an error with a message and run no kernel after the failure.  The parts a call builds on first use are built
  whole or not at all, so what the failed call leaves live is at most what a successful call leaves (a call may keep a
  part it finished before the one that failed; the bound is not the count before the call).  The same call must then
  succeed on that ctx with the outputs and the snapshot of the same call on a fresh ctx, and leave exactly what a
  successful call leaves (nothing leaked, nothing built twice); destroy must leave nothing.

Snapshots are compared by content (`canonical`): which slot of an open-addressing table a key lands in depends on the
order of concurrent inserts, and dense issuer indices on the order of concurrent registration, so two fresh ctxs give
different bytes for the same call.  Keys, pairs, string identities, histograms and counters are compared with every
issuer index replaced by its digest.

Each case runs in a child process under the shim.  The child drives libctmr through capi / engine with numpy only: torch
loads its own CUDA runtime, which the shim would not see.  Run as a script, this file is that child."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOW_NS = 1767225600 * 10**9
KINDS = ("device", "pinned", "stream", "event")

# creations of a repeated call, per kind (device, pinned, stream, event): temporaries of that call only
EXPECTED_REPEAT = {
    "batch_pem": [0, 0, 0, 0], "device_2_rounds": [0, 0, 0, 0], "device_8_rounds": [0, 0, 0, 0],
    "map_device": [0, 0, 0, 0], "reduce_device": [0, 0, 0, 0], "raw": [0, 0, 0, 0], "raw_mirror": [0, 0, 0, 0],
    "raw_tree": [0, 0, 0, 0], "chain_certs": [3, 0, 0, 0], "tiles": [0, 0, 0, 0], "tiles_tree": [0, 0, 0, 0],
    "register_issuers": [5, 0, 0, 0], "preload": [0, 0, 0, 0], "evict": [0, 0, 0, 0],
    "snapshot": [2, 0, 0, 0], "sha256_ceiling": [0, 0, 0, 2], "group": [0, 0, 0, 0],
}
CASES = sorted(EXPECTED_REPEAT)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    from ct_mapreduce_b200 import build
    build.build()
    out = tmp_path_factory.mktemp("shim") / "libcuda_shim.so"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-shared", "-fPIC", "-o", str(out),
                    os.path.join(ROOT, "tests", "cpp", "cuda_shim.cpp"), "-ldl"], check=True)
    return str(out)


def run_child(shim, *args):
    env = dict(os.environ, LD_PRELOAD=shim, CTMR_SHIM=shim, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), *args], capture_output=True, text=True, env=env,
                       cwd=ROOT, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_shim_sees_the_librarys_runtime_calls(shim):
    """libctmr links the CUDA runtime dynamically: ctmr_create's device query reaches the shim (with or without a GPU)."""
    got = run_child(shim, "device_count")
    assert got["calls"] >= 1
    assert not got["torch"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_lifetime(shim, case):
    got = run_child(shim, "life", case)
    assert not got["torch"]
    assert got["live_after_repeat"] == got["live_after_first"], "a repeated call changed the live counts"
    assert got["created_by_repeat"] == EXPECTED_REPEAT[case]
    assert got["live_after_destroy"] == got["live_before"], "resources outlived destroy"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_fresh_ctxs_agree(shim, case):
    """What the injected cases compare is reproducible: two fresh ctxs give the same outputs and snapshot content."""
    got = run_child(shim, "twice", case)
    assert got["outputs"] and got["snapshot"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_injected_failures(shim, case):
    got = run_child(shim, "inject", case)
    assert not got["torch"]
    assert sum(got["created_by_first"]) > 0
    assert got["runs"] == sum(got["created_by_first"])
    assert got["problems"] == [], got["problems"][:10]


def _mix(z):
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _rows(cols):
    """a sorted fingerprint per row: the rows as a multiset"""
    h = np.zeros(cols.shape[0], np.uint64)
    for j in range(cols.shape[1]):
        h = _mix(h ^ (cols[:, j].astype(np.uint64) + np.uint64(0x9E3779B97F4A7C15 * (j + 1) & ((1 << 64) - 1))))
    return np.sort(h)


def canonical(snap, pair_slots):
    """A ctx or group snapshot as content: next index, issuer digests, and per shard its keys, pairs, string identities,
    per-issuer counts and status counters, with issuer indices replaced by the rank of their digest."""
    from keymodel import KNOWN_SLOT, PAIR_SLOT
    s = np.ascontiguousarray(snap, np.uint8)
    hdr = s[8:56].view("<u8")
    n_iss, next_index = int(hdr[4]), int(hdr[5])
    if s[:8].tobytes() == b"CTMRGRP1":
        members, shard_bytes, table_slots, max_iss = (int(x) for x in hdr[:4])
    else:
        table_slots, pair_slots, max_iss, members = int(hdr[0]), int(hdr[1]), int(hdr[3]), 1
        shard_bytes = s.size - 56 - 32 * n_iss
    dig = s[s.size - 32 * n_iss:].reshape(n_iss, 32)
    order = sorted(range(n_iss), key=lambda i: dig[i].tobytes())
    rank = np.zeros(n_iss, np.uint64)
    rank[order] = np.arange(n_iss, dtype=np.uint64)

    def by_digest(idx):
        idx = idx.astype(np.uint64)
        known = idx < n_iss
        return np.where(known, rank[np.minimum(idx, max(n_iss - 1, 0)).astype(np.int64)] if n_iss else idx, idx + (1 << 32))

    out = [np.array([next_index, n_iss], np.uint64), np.sort(dig.view("V32").ravel()).view(np.uint8)]
    for m in range(members):
        sh = s[56 + m * shard_bytes:56 + (m + 1) * shard_bytes]
        t_end, p_end = table_slots * 64, table_slots * 64 + pair_slots * 32
        table, pairs = sh[:t_end].view(KNOWN_SLOT), sh[t_end:p_end].view(PAIR_SLOT)
        tail = sh[p_end:]
        meta, counts, status = tail[:-(8 * max_iss + 64)], tail[-(8 * max_iss + 64):-64].view("<u8"), tail[-64:]
        ready = (table["tag"] & np.uint64(3)) == np.uint64(2)
        body = table["body"][ready].astype(np.uint64)
        body[:, 1] = by_digest(body[:, 1])
        keys = np.concatenate([body, table["inv_first"][ready][:, None]], axis=1)
        pk = pairs[pairs["key"] != 0]
        k = pk["key"] - np.uint64(1)
        pcols = np.stack([k & np.uint64(0xFFFFFFFF), by_digest(k >> np.uint64(32)), pk["inv_first"], pk["count"]], axis=1)
        mrows = meta.view("<u8").reshape(-1, 4)
        per_issuer = np.zeros(n_iss, np.uint64)
        per_issuer[rank[: n_iss].astype(np.int64)] = counts[:n_iss]
        out += [_rows(keys), _rows(pcols), _rows(mrows[mrows.any(axis=1)]), per_issuer, counts[n_iss:].copy(), status.copy()]
    return out


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


# ==================================================================================================== the child
def _child(argv):
    sys.path.insert(0, ROOT)
    from ct_mapreduce_b200 import capi, engine
    from ct_mapreduce_b200.capi import CtmrError

    if argv[0] == "device_count":
        L = capi.load()
        cfg = capi.Config()
        cfg.struct_size = C.sizeof(capi.Config)
        h = C.c_void_p()
        if L.ctmr_create(C.byref(cfg), C.byref(h)) == 0:
            L.ctmr_destroy(h)
        shim = C.CDLL(os.environ["CTMR_SHIM"])
        return {"calls": shim.shim_get_device_count_calls(), "torch": "torch" in sys.modules}

    L = capi.load()
    rt = C.CDLL("libcudart.so.12")  # the runtime libctmr loaded; its own symbols, not the shim's
    shim = C.CDLL(os.environ["CTMR_SHIM"])
    shim.shim_fail_nth.argtypes = [C.c_int, C.c_long]
    shim.shim_refused_launches.restype = C.c_long

    def counts():
        live, made = (C.c_long * 4)(), (C.c_long * 4)()
        shim.shim_counts(live, made)
        return list(live), list(made)

    def dev_alloc(nbytes):
        p = C.c_void_p()
        assert rt.cudaMalloc(C.byref(p), C.c_size_t(max(nbytes, 1))) == 0
        return p.value

    def d2h(p, nbytes):
        a = np.empty(nbytes, np.uint8)
        assert rt.cudaMemcpy(a.ctypes.data_as(C.c_void_p), C.c_void_p(p), C.c_size_t(nbytes), 2) == 0
        return a

    from oracle import oracle
    n_host = 3000
    cfg = oracle.synth_cfg(n_host, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, n_host)
    iblob, ioffs = oracle.synth_issuers(cfg)
    small = dict(table_capacity=1 << 16, pair_capacity_log2=16, meta_capacity_log2=12, max_issuers=1024)
    case, mode = argv[1], argv[0]
    big = {"device_2_rounds": dict(table_capacity=1 << 20, pair_capacity_log2=20),
           "device_8_rounds": dict(table_capacity=1 << 22, pair_capacity_log2=20)}

    def make():
        return engine.GpuCertDatabase(device=0, max_batch_entries=1024, **dict(small, **big.get(case, {})))

    def pre_issuers(db):
        db.register_issuers(iblob, ioffs)

    def batch_outputs(r):
        return [r.status, r.was_unknown, r.first_issuer_hour, r.sha256]

    # -------- device-resident inputs (the test's own buffers, made before the counts are taken)
    dev = {}

    def device_inputs(n):
        if n in dev:
            return dev[n]
        scfg = capi.synth_cfg(n, dup_mode=1)
        offsets = dev_alloc((n + 1) * 8)
        total = C.c_uint64(0)
        assert L.ctmr_synth_offsets_device(C.byref(scfg), 0, n, C.c_void_p(offsets), C.byref(total), None) == 0
        dblob, didx = dev_alloc(total.value + 64), dev_alloc(4 * n)
        assert L.ctmr_synth_write_device(C.byref(scfg), 0, n, C.c_void_p(offsets), C.c_void_p(dblob), C.c_void_p(didx), None) == 0
        out = {k: dev_alloc(n * w) for k, w in (("status", 1), ("sha", 32), ("exp", 8), ("soff", 4), ("slen", 4), ("wu", 1),
                                                 ("fi", 1), ("keys", 64))}
        assert rt.cudaDeviceSynchronize() == 0
        dev[n] = (offsets, dblob, didx, total.value, out)
        return dev[n]

    def zero_outputs(n):
        for k, w in (("status", 1), ("sha", 32), ("exp", 8), ("soff", 4), ("slen", 4), ("wu", 1), ("fi", 1), ("keys", 64)):
            assert rt.cudaMemset(C.c_void_p(dev[n][4][k]), 0, C.c_size_t(n * w)) == 0

    def process_device(db, n):
        offsets, dblob, didx, total, t = device_inputs(n)
        zero_outputs(n)
        b = capi.DevBatch()
        b.blob, b.blob_bytes, b.offsets, b.n = dblob, total, offsets, n
        b.issuer_idx, b.issuer_map, b.issuer_map_len, b.first_index, b.now_unix_ns = didx, None, 0, 0, NOW_NS
        o = capi.DevOut(t["status"], t["sha"], t["exp"], t["soff"], t["slen"], t["wu"], t["fi"], None)
        db.process_device(b, o)
        assert rt.cudaDeviceSynchronize() == 0
        return [d2h(t[k], n * w) for k, w in (("status", 1), ("wu", 1), ("fi", 1), ("sha", 32))]

    def map_device(db):
        n = 4096
        offsets, dblob, didx, total, t = device_inputs(n)
        zero_outputs(n)
        b = capi.DevBatch()
        b.blob, b.blob_bytes, b.offsets, b.n = dblob, total, offsets, n
        b.issuer_idx, b.first_index, b.now_unix_ns = didx, 0, NOW_NS
        o = capi.DevOut(t["status"], t["sha"], t["exp"], t["soff"], t["slen"], None, None, t["keys"])
        db.map_device(b, o)
        assert rt.cudaDeviceSynchronize() == 0
        return [d2h(t[k], n * w) for k, w in (("status", 1), ("sha", 32), ("keys", 64))]

    def reduce_device(db):  # over the keys map_device left (pre)
        n, t = 4096, dev[4096][4]
        for k in ("wu", "fi"):
            assert rt.cudaMemset(C.c_void_p(t[k]), 0, C.c_size_t(n)) == 0
        db.reduce_device(t["keys"], n, t["wu"], t["fi"])
        assert rt.cudaDeviceSynchronize() == 0
        return [d2h(t[k], n) for k in ("wu", "fi")]

    # -------- get-entries pages and data tiles from libctmr's host generators
    def pages(n):
        pcfg = capi.synth_cfg(n)
        need = L.ctmr_synth_raw_pages_host(C.byref(pcfg), 0, n, 1000, None, 0, None, None, None, None)
        text = np.zeros(need, np.uint8)
        lo, ll, xo, xl = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(n, np.uint32)
        L.ctmr_synth_raw_pages_host(C.byref(pcfg), 0, n, 1000, capi.ptr(text), need, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl))
        return text, lo, ll, xo, xl

    def tiles(nt):
        import hashlib
        tcfg = capi.synth_cfg(256 * nt)
        tib, tio = engine.synth_issuers(tcfg)
        certs = [tib[int(tio[k]):int(tio[k + 1])].tobytes() for k in range(tcfg.n_issuers)]
        fps = np.frombuffer(b"".join(hashlib.sha256(d).digest() for d in certs), np.uint8).copy()
        need = L.ctmr_synth_tiles_host(C.byref(tcfg), 0, nt, capi.ptr(fps), None, 0, None, None)
        buf = np.zeros(need, np.uint8)
        off, ln = np.zeros(nt, np.uint64), np.zeros(nt, np.uint32)
        L.ctmr_synth_tiles_host(C.byref(tcfg), 0, nt, capi.ptr(fps), capi.ptr(buf), need, capi.ptr(off), capi.ptr(ln))
        return buf, off, ln, np.arange(nt, dtype=np.uint64), np.full(nt, 256, np.uint32), certs

    def raw_outputs(r):
        return [r.path.status, r.path.was_unknown, r.path.first_issuer_hour, r.entry_status]

    def raw(db, tree):
        r = db.store_raw_entries(*pages(1000), NOW_NS, tree=engine.LogTree() if tree else None)
        return raw_outputs(r) + ([np.frombuffer(r.tree.root, np.uint8)] if tree else [])

    def chain_certs(db):  # every Chain[0] certificate of the tiles
        certs = tiles(4)[5]
        blob = np.frombuffer(b"".join(certs), np.uint8).copy()
        offs = np.zeros(len(certs) + 1, np.uint64)
        offs[1:] = np.cumsum([len(d) for d in certs], dtype=np.uint64)
        dense, fps = db.register_chain_certs(blob, offs)
        return [fps, np.frombuffer(b"".join(db.issuer_digest(int(i)) for i in dense), np.uint8)]

    def tile_call(db, tree):  # the chain certificates are registered (pre): no stop, one chunk
        buf, off, ln, ti, tw, _ = tiles(4)
        r = db.store_tiles(buf, off, ln, ti, tw, NOW_NS, tree=engine.LogTree() if tree else None)
        return raw_outputs(r) + ([np.frombuffer(r.tree.root, np.uint8)] if tree else [])

    digest = bytes(range(32))

    def sha(db):
        db.sha256_ceiling(iters=16)
        return []

    def snapshot(db):
        s = db.snapshot()
        db.restore(s)
        return canonical(s, 1 << 16)

    holder = {}

    def pre_evict(db):  # evicts about half of what the batch stored
        r = db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
        holder.setdefault("evict_at", int(np.median(r.exp_hour[r.status == 0])) * 3600)

    def group_call(db):
        g = engine.GpuCertGroup([0, 0], max_batch_entries=512, **small)
        holder["g"] = g
        return batch_outputs(g.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS))

    def batch_pem(db):
        r = db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS, want_meta=True, want_pem=True)
        return batch_outputs(r) + [r.pem[:int(r.pem_off[-1])]]

    table = {  # case: (pre, call)
        "batch_pem": (None, batch_pem),
        "device_2_rounds": (pre_issuers, lambda db: process_device(db, 1 << 18)),
        "device_8_rounds": (pre_issuers, lambda db: process_device(db, 1 << 21)),
        "map_device": (pre_issuers, map_device),
        "reduce_device": (lambda db: (pre_issuers(db), map_device(db)), reduce_device),
        "chain_certs": (None, chain_certs),
        "raw": (None, lambda db: raw(db, False)),
        "raw_tree": (None, lambda db: raw(db, True)),
        "tiles": (chain_certs, lambda db: tile_call(db, False)),
        "tiles_tree": (chain_certs, lambda db: tile_call(db, True)),
        "register_issuers": (None, lambda db: [np.frombuffer(b"".join(db.issuer_digest(int(i)) for i in db.register_issuers(iblob, ioffs)), np.uint8)]),
        "raw_mirror": (pre_issuers, lambda db: raw(db, False)),  # the front end mirrors the issuers registered before it
        "preload": (None, lambda db: (db.preload_known(480000, digest, [b"\x01\x02", b"\x03"]), [])[1]),
        "evict": (pre_evict, lambda db: [np.array([db.evict_expired(holder["evict_at"])])]),
        "snapshot": (lambda db: db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS), snapshot),
        "sha256_ceiling": (None, sha),
        "group": (None, group_call),
    }
    pre, call = table[case]
    if case == "register_issuers" and mode == "life":  # each call registers one certificate never seen before
        seq = iter(range(len(ioffs) - 1))

        def call(db):
            k = next(seq)
            return [db.register_issuers(iblob[int(ioffs[k]):int(ioffs[k + 1])], ioffs[k:k + 2] - ioffs[k])]

    for n in ({"device_2_rounds": [1 << 18], "device_8_rounds": [1 << 21], "map_device": [4096], "reduce_device": [4096]}).get(case, []):
        device_inputs(n)

    def fresh():
        db = make()
        if pre:
            pre(db)
        return db

    def close(db):
        g = holder.pop("g", None)
        if g is not None:
            g.close()
        db.close()

    zero = counts()[0]
    if mode == "twice":  # two fresh ctxs, the same call: the results the injected cases are held to agree
        got = []
        for _ in range(2):
            db = fresh()
            got.append((call(db), canonical((holder.get("g") or db).snapshot(), 1 << 16)))
            close(db)
        return {"torch": "torch" in sys.modules, "outputs": same(got[0][0], got[1][0]), "snapshot": same(got[0][1], got[1][1])}
    db = fresh()
    before, made0 = counts()
    out1 = call(db)
    live1, made1 = counts()
    snap1 = canonical((holder.get("g") or db).snapshot(), 1 << 16)
    res = {"torch": "torch" in sys.modules, "live_before": before, "live_after_first": live1,
           "created_by_first": [b - a for a, b in zip(made0, made1)]}
    if case == "group":  # a repeated call on the same group
        holder["g"].store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
    else:
        call(db)
    live2, made2 = counts()
    res["live_after_repeat"] = live2
    res["created_by_repeat"] = [b - a for a, b in zip(made1, made2)]
    close(db)
    res["live_after_destroy"] = counts()[0]
    if mode == "life":
        res["live_before"] = zero
        return res

    # ---- injected failures: the n-th creation of each kind the first call makes
    problems, runs = [], 0
    for kind, k in enumerate(res["created_by_first"]):
        for nth in range(1, k + 1):
            runs += 1
            tag = f"{KINDS[kind]} #{nth}"
            db = fresh()
            shim.shim_fail_nth(kind, nth)
            try:
                call(db)
                problems.append(tag + ": the call succeeded")
            except CtmrError as e:
                if not str(e).strip():
                    problems.append(tag + ": no message")
            refused = shim.shim_refused_launches()
            shim.shim_fail_nth(-1, 0)
            live_f = counts()[0]
            if refused:
                problems.append(f"{tag}: {refused} kernel launches after the failure")
            if any(b > a for a, b in zip(res["live_after_first"], live_f)):
                problems.append(f"{tag}: live {live_f} after the failure, {res['live_after_first']} after a successful call")
            try:
                out = call(db)
                if counts()[0] != res["live_after_first"]:
                    problems.append(f"{tag}: live {counts()[0]} after the retry, {res['live_after_first']} after a successful call")
                if not same(out, out1):
                    problems.append(f"{tag}: the retry's outputs differ from a fresh ctx's")
                if not same(canonical((holder.get("g") or db).snapshot(), 1 << 16), snap1):
                    problems.append(f"{tag}: the snapshot after the retry differs from a fresh ctx's")
            except CtmrError as e:
                problems.append(f"{tag}: the retry failed: {e}")
            close(db)
            if counts()[0] != zero:
                problems.append(f"{tag}: live after destroy {counts()[0]}")
    res.update(runs=runs, problems=problems)
    return res


if __name__ == "__main__":
    print(json.dumps(_child(sys.argv[1:]), default=int))
