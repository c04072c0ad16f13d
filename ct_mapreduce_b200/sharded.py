"""Start-up and index arithmetic of the one-process-per-GPU form of the multi-GPU path (include/ctmr.h "ctmr_peer_*").

The map half is embarrassingly parallel over entry index.  The reduce half has ONE real exchange step (SURVEY.md
§8(e), H5): equal keys can land on different GPUs, so every set "serials::<expDate>::<issuer>" has one owner GPU --
owner = hash(exp_hour, issuer) mod world, like a Redis-cluster key -- and the LIBRARY moves the keys there: K_map
appends the 64-byte record of a foreign key to the owner's inbox over NVLink, the owner inserts and resolves
lowest-index-wins locally, the result bits are pulled back, and the histograms are merged by a sum over peer memory
at the end of the chunk.  What is left for the host language is what this module holds: exchanging the peer handles
once (any torch.distributed backend -- NCCL on the GPU box, gloo in the CPU tests) and knowing which sequential order
a collective call is equivalent to.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.distributed as dist

from . import capi

KEY_BYTES = capi.KEY_BYTES


# ---------------------------------------------------------------------------------------------------------------
# One process per GPU, owners' tables attached over CUDA IPC (include/ctmr.h "ctmr_peer_*"): the exact multi-GPU
# path.  torch.distributed only carries the 128-byte handles at start-up (any backend) and the bench's timing
# reductions; there is no collective on the data path -- K_map inserts into the owner's table over NVLink and the
# ranks meet at barriers kept in peer memory.
# ---------------------------------------------------------------------------------------------------------------
def attach_peers(db, group=None):
    """All ranks: exchange peer handles and attach.  Afterwards db.process_device / store_batch / reset_device /
    peer_allreduce_histogram_device are collective calls (same sequence on every rank)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    if world == 1:
        return rank, world
    handles = [None] * world
    dist.all_gather_object(handles, db.peer_export(world), group=group)
    db.peer_attach(rank, world, handles)
    return rank, world


def round_entries(n: int, rounds: int = 0) -> int:
    """E of the collective ctmr_process_device: entries per rank and round (every rank passes the same n).  The last round
    is a quarter of the others (its reduce chain is what a call exposes at its end): E = ceil(4n / (4R - 3)) for R >= 4."""
    if not rounds:
        return int(capi.load().ctmr_peer_round_entries(n))   # the library's own answer (its round count may be overridden)
    return -(-4 * n // (4 * rounds - 3)) if rounds >= 4 else -(-n // rounds)


def call_index_span(n: int, world: int, rounds: int = 0) -> int:
    """How far a collective ctmr_process_device call advances the global index (its next call's first_index)."""
    rounds = rounds or capi.peer_rounds()
    return world * rounds * round_entries(n, rounds)


def sequential_order(n: int, world: int, rounds: int = 0):
    """The order in which the sequential reference (numThreads=1) would have to see the entries of one collective
    call for its result to equal the group's: rounds in order, inside a round the ranks in order, inside a rank's
    slice the entries in order.  Yields (rank, lo, hi) slices of each rank's local batch [0, n)."""
    rounds = rounds or capi.peer_rounds()
    e = round_entries(n, rounds)
    for k in range(rounds):
        lo, hi = min(n, k * e), min(n, (k + 1) * e)
        for r in range(world):
            if hi > lo:
                yield r, lo, hi


def host_batch_order(ns, stage_entries: int):
    """The same for the collective HOST-buffer call (ctmr_process_batch with peers attached): rank r passes ns[r]
    entries, a round takes `stage_entries` per rank, every rank runs max(rounds) rounds.  (Byte-budget shrinking of a
    round is not modelled: callers keep entries below config.max_batch_bytes / stage_entries on average.)"""
    rounds = max(1, max(-(-n // stage_entries) for n in ns))
    for k in range(rounds):
        for r, n in enumerate(ns):
            lo, hi = min(n, k * stage_entries), min(n, (k + 1) * stage_entries)
            if hi > lo:
                yield r, lo, hi


def frontend_chunks(widths, entry_budget: int):
    """The chunk sizes (in entries) one rank's front-end call cuts from its batch by the entry budget: units (entries of
    pages, width 1 each; tiles, their widths) are taken greedily while the chunk stays within `entry_budget` entries.
    (The character / byte budget of the staging buffers may cut earlier; callers keep batches well inside it.)"""
    sizes, cur = [], 0
    for w in widths:
        w = int(w)
        if cur and cur + w > entry_budget:
            sizes.append(cur)
            cur = 0
        cur += w
    if cur:
        sizes.append(cur)
    return sizes


def frontend_indices(chunks, entry_budget: int, next_index: int = 0):
    """The global index of every entry of a collective front-end call (ctmr_process_raw / ctmr_process_tiles and their
    tree forms with peers attached): chunks[r] lists rank r's chunk sizes in entries (frontend_chunks).  Every rank runs
    R = max(chunk counts) rounds, and entry j of rank r's chunk k takes next_index + (k * world + r) * E + j with E =
    entry_budget.  Returns ([one uint64 array of indices per rank, in batch order], the call's span R * world * E)."""
    import numpy as np
    world = len(chunks)
    rounds = max(1, max((len(c) for c in chunks), default=0))
    out = []
    for r, sizes in enumerate(chunks):
        parts = [next_index + (k * world + r) * entry_budget + np.arange(s, dtype=np.uint64) for k, s in enumerate(sizes)]
        out.append(np.concatenate(parts).astype(np.uint64) if parts else np.zeros(0, np.uint64))
    return out, rounds * world * entry_budget
