"""Writes tests/golden/snapshot_small.bin.gz and checkpoint_small.bin.gz: a snapshot and a checkpoint of one small state,
which tests/test_gpu_snapshot_golden.py restores and saves again byte for byte.

    python tools/gen_snapshot_golden.py [OUT_DIR]

The fixtures in the repository were written by the tree before table epochs (the commit before "Reset the
known-certificate, pair and string-identity tables by epoch"), so the test pins the snapshot and checkpoint formats to
the bytes that tree wrote.  The state: 48 synthetic entries, a reset, then 72 entries of which 24 repeat the first
batch, with the IssuerMetadata string identities, in tables small enough to keep the files small.
"""
import gzip
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NOW_NS = 1767225600 * 10**9
KW = dict(table_capacity=1 << 10, log_expired_entries=True, max_issuers=16, pair_capacity_log2=8, meta_capacity_log2=8)


def state():
    """(snapshot bytes, checkpoint bytes) of the state, on cuda:0"""
    from ct_mapreduce_b200 import engine
    from oracle import oracle
    cfg = oracle.synth_cfg(96, n_issuers=8, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, 96)
    iblob, ioffs = oracle.synth_issuers(cfg)
    with engine.GpuCertDatabase(device=0, **KW) as db:
        db.register_issuers(iblob, ioffs)
        db.store_batch(blob, offs[:49], iblob, ioffs, idx[:48], NOW_NS, want_meta=True)
        db.reset_device()
        db.store_batch(blob, offs[24:97], iblob, ioffs, idx[24:96], NOW_NS, want_meta=True)
        return db.snapshot().tobytes(), db.checkpoint().tobytes()


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
    snap, ck = state()
    for name, data in (("snapshot_small.bin.gz", snap), ("checkpoint_small.bin.gz", ck)):
        with open(os.path.join(out, name), "wb") as f:
            f.write(gzip.compress(data, compresslevel=9, mtime=0))
        print(name, len(data))


if __name__ == "__main__":
    main()
