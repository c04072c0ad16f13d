"""The snapshot and checkpoint formats did not change with table epochs: a snapshot and a checkpoint of one small state,
written by the tree before epochs (tools/gen_snapshot_golden.py), restored into a fresh ctx and into one whose tables
hold slots of earlier epochs, give back the same bytes when the snapshot and a checkpoint are saved again.  Marked gpu."""
import gzip
import os

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden")
KW = dict(table_capacity=1 << 10, log_expired_entries=True, max_issuers=16, pair_capacity_log2=8, meta_capacity_log2=8)
NOW_NS = 1767225600 * 10**9


def _load(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return np.frombuffer(gzip.decompress(f.read()), np.uint8).copy()


def _stale(db):
    """fill db's tables with other keys, then reset three times: every slot they left is of an earlier epoch"""
    from oracle import oracle
    cfg = oracle.synth_cfg(300, n_issuers=8, dup_mode=1, seed=7)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, 300)
    iblob, ioffs = oracle.synth_issuers(cfg)
    db.register_issuers(iblob, ioffs)
    db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS, want_meta=True)
    assert db.table_stats()[0] > 0
    for _ in range(3):
        db.reset_device()


@pytest.mark.parametrize("history", ["fresh", "stale_slots"])
def test_parent_written_snapshot_and_checkpoint_round_trip(history):
    from ct_mapreduce_b200 import engine
    snap, ck = _load("snapshot_small.bin.gz"), _load("checkpoint_small.bin.gz")
    with engine.GpuCertDatabase(device=0, **KW) as db:
        if history == "stale_slots":
            _stale(db)
        db.restore(snap)
        assert db.table_stats()[0] > 0
        assert np.array_equal(db.snapshot(), snap), "snapshot bytes differ from the format's"
        assert np.array_equal(db.checkpoint(), ck), "checkpoint bytes differ from the format's"
