"""Ownership of what ctmr_process_raw_bodies builds (DESIGN §2), under the LD_PRELOAD shim of the CUDA runtime
(tests/cpp/cuda_shim.cpp) that tests/test_gpu_lifecycle.py uses for the other calls: a repeated call creates nothing,
destroy releases everything, and a failure injected at the n-th creation of each kind the first call makes (device
buffer, pinned buffer, stream, event) fails the call with a message, launches nothing after it, leaves no more live
than a successful call, and leaves the ctx as it was: the retry gives the outputs and the snapshot of a fresh ctx.
Each case runs in a child process under the shim; run as a script, this file is that child."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOW_NS = 1767225600 * 10**9
CASES = ["bodies", "bodies_pem"]


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


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_lifetime(shim, case):
    got = run_child(shim, "life", case)
    assert not got["torch"]
    assert got["live_after_repeat"] == got["live_after_first"], "a repeated call changed the live counts"
    assert got["created_by_repeat"] == [0, 0, 0, 0]
    assert got["live_after_destroy"] == got["live_before"], "resources outlived destroy"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_fresh_ctxs_agree(shim, case):
    """What the injected cases compare is reproducible: two fresh ctxs give the same outputs and snapshot content."""
    got = run_child(shim, "twice", case)
    assert got["outputs"] and got["snapshot"], got["differ"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_injected_failures(shim, case):
    got = run_child(shim, "inject", case)
    assert not got["torch"]
    assert sum(got["created_by_first"]) > 0
    assert got["runs"] == sum(got["created_by_first"])
    assert got["problems"] == [], got["problems"][:10]


def _child(argv):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_gpu_lifecycle as lc
    from ct_mapreduce_b200 import capi, engine
    from ct_mapreduce_b200.capi import CtmrError

    mode, case = argv
    L = capi.load()
    shim = C.CDLL(os.environ["CTMR_SHIM"])
    shim.shim_fail_nth.argtypes = [C.c_int, C.c_long]
    shim.shim_refused_launches.restype = C.c_long

    def counts():
        live, made = (C.c_long * 4)(), (C.c_long * 4)()
        shim.shim_counts(live, made)
        return list(live), list(made)

    # 1,000 synthetic entries as four bodies, one with every '/' escaped, and a few bodies that are not OK
    n, page = 1000, 250
    cfg = capi.synth_cfg(n)
    need = L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, page, None, 0, None, None, None, None)
    text = np.zeros(need, np.uint8)
    lo, ll, xo, xl = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, page, capi.ptr(text), need, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl))
    starts = [int(lo[a]) - len(b'{"entries":[{"leaf_input":"') for a in range(0, n, page)] + [need]
    bodies = [text[starts[k]:starts[k + 1]].tobytes() for k in range(len(starts) - 1)]
    bodies[1] = bodies[1].replace(b"/", b"\\/")
    bodies += [b'{"entries":[],"Entries":[]}', b"{", b"[]", b"null"]
    maxes = np.array([page] * 4 + [1, 1, 1, 0], np.uint32)
    blob = b"".join(bodies)
    offs = np.cumsum([0] + [len(b) for b in bodies[:-1]]).astype(np.uint64)
    lens = np.array([len(b) for b in bodies], np.uint32)
    pem = case == "bodies_pem"

    def call(db):
        # no string identities: the rows the front end leaves in that table differ between two fresh ctxs already with
        # ctmr_process_raw, so a snapshot comparison could not tell a failure's trace from that
        r = db.store_raw_bodies(blob, offs, lens, maxes, NOW_NS, want_pem=pem)
        out = [r.path.status, r.path.was_unknown, r.path.first_issuer_hour, r.entry_status, r.body_status, r.body_entries,
               r.leaf_input_off, r.extra_data_len, r.escaped]
        return out + ([r.path.pem[:int(r.path.pem_off[-1])]] if pem else [])

    def fresh():  # one chunk (1,003 entries requested): every creation comes before any entry reaches the path
        return engine.GpuCertDatabase(device=0, max_batch_entries=1024, table_capacity=1 << 16, pair_capacity_log2=16,
                                      meta_capacity_log2=12, max_issuers=1024)

    zero = counts()[0]
    if mode == "twice":  # two fresh ctxs, the same call: the results the injected cases are held to agree
        got = []
        for _ in range(2):
            db = fresh()
            got.append((call(db), lc.canonical(db.snapshot(), 1 << 16)))
            db.close()
        return {"torch": "torch" in sys.modules, "outputs": lc.same(got[0][0], got[1][0]),
                "snapshot": lc.same(got[0][1], got[1][1]),
                "differ": [i for i, (x, y) in enumerate(zip(got[0][1], got[1][1])) if not np.array_equal(x, y)]}
    db = fresh()
    before, made0 = counts()
    out1 = call(db)
    live1, made1 = counts()
    snap1 = lc.canonical(db.snapshot(), 1 << 16)
    res = {"torch": "torch" in sys.modules, "live_before": before, "live_after_first": live1,
           "created_by_first": [b - a for a, b in zip(made0, made1)]}
    call(db)
    live2, made2 = counts()
    res["live_after_repeat"] = live2
    res["created_by_repeat"] = [b - a for a, b in zip(made1, made2)]
    db.close()
    res["live_after_destroy"] = counts()[0]
    if mode == "life":
        res["live_before"] = zero
        return res

    problems, runs = [], 0
    for kind, k in enumerate(res["created_by_first"]):
        for nth in range(1, k + 1):
            runs += 1
            tag = f"{lc.KINDS[kind]} #{nth}"
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
            if db.next_index() != 0:
                problems.append(f"{tag}: a failure before any work took indices")
            try:
                out = call(db)
                if counts()[0] != res["live_after_first"]:
                    problems.append(f"{tag}: live {counts()[0]} after the retry, {res['live_after_first']} after a successful call")
                if not lc.same(out, out1):
                    problems.append(f"{tag}: the retry's outputs differ from a fresh ctx's")
                if not lc.same(lc.canonical(db.snapshot(), 1 << 16), snap1):
                    problems.append(f"{tag}: the snapshot after the retry differs from a fresh ctx's")
            except CtmrError as e:
                problems.append(f"{tag}: the retry failed: {e}")
            db.close()
            if counts()[0] != zero:
                problems.append(f"{tag}: live after destroy {counts()[0]}")
    res.update(runs=runs, problems=problems)
    return res


if __name__ == "__main__":
    print(json.dumps(_child(sys.argv[1:]), default=int))
