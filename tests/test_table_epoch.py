"""The tables' epoch encodings, checked on the host: the slot words, tags and canonical forms of ctmr_common.cuh
(compiled unchanged) must keep a slot live only at its own epoch, keep zeroed memory empty, wrap the epoch to a clear and
give a stamped slot back as the same canonical bytes that snapshots and checkpoints hold."""
import os
import subprocess

from conftest import ROOT


def test_table_epoch_encodings(tmp_path):
    from ct_mapreduce_b200 import build
    out = tmp_path / "table_epoch"
    subprocess.run([build._nvcc(), "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                    "-o", str(out), os.path.join(ROOT, "tests", "cpp", "table_epoch.cu")], check=True)
    r = subprocess.run([str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("ok "), r.stdout
