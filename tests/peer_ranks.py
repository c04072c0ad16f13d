"""Ranks of a multi-process test: one spawned process per rank, each running worker(rank, world, *args) with the
torch.distributed environment set, and nothing left running afterwards.

A rank that fails can leave the others spinning in a peer barrier or a collective until their timeouts run out, so
run_ranks ends every rank that is still alive when it returns or raises, whatever happened."""
import os
import queue
import socket
import sys
import time
import traceback

import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRACE_S = 10   # after a rank's traceback: how long the others have to report theirs before they are ended


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(worker, rank, world, port, args, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    try:
        res = worker(rank, world, *args)
    except BaseException:
        q.put((rank, None, traceback.format_exc()))
        raise
    q.put((rank, res, None))


def run_ranks(worker, world, args=(), timeout=300):
    """{rank: what worker returned} once every rank returned within `timeout` seconds and exited with code 0.  Fails with
    every traceback the ranks sent otherwise.  worker must be a module-level function (it is pickled by name)."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_rank_main, args=(worker, r, world, port, args, q)) for r in range(world)]
    results, errors = {}, {}
    try:
        for p in procs:
            p.start()
        deadline = time.monotonic() + timeout
        while len(results) + len(errors) < world:
            try:
                rank, res, err = q.get(timeout=max(0.0, deadline - time.monotonic()))
            except queue.Empty:
                break
            if err is None:
                results[rank] = res
            else:
                errors[rank] = err
                deadline = min(deadline, time.monotonic() + GRACE_S)
        assert not errors, "\n".join("rank %d failed:\n%s" % (r, errors[r]) for r in sorted(errors))
        missing = [r for r in range(world) if r not in results]
        assert not missing, "no result from rank(s) %s within %d s" % (missing, timeout)
        for r, p in enumerate(procs):  # after the results: a rank exits only once the queue has taken what it put
            p.join(timeout=120)
            assert p.exitcode == 0, "rank %d exited with %s" % (r, p.exitcode)
        return results
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
            if p.is_alive():
                p.kill()
                p.join()
