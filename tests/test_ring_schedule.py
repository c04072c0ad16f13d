"""K_map's per-lane staging ring, checked on the host: the copy schedule the kernel runs (ring_chunk_copy and ring_step
in ctmr_common.cuh, compiled unchanged) must never overwrite a byte the DER walker or the SHA-256 loop still reads,
even when every asynchronous copy lands the moment it is issued.  The case that needs care is a misaligned record:
chunk c+1's last granule shares a ring slot with chunk c's first, so it may only be copied after chunk c is hashed."""
import os
import subprocess

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "ct_mapreduce_b200", "csrc")


@pytest.fixture(scope="module")
def ring_bin(tmp_path_factory):
    from ct_mapreduce_b200 import build
    out = tmp_path_factory.mktemp("ringbin") / "ring_schedule"
    subprocess.run([build._nvcc(), "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                    "-o", str(out), os.path.join(ROOT, "tests", "cpp", "ring_schedule.cu")], check=True)
    return str(out)


def test_schedule_keeps_every_byte_the_walker_and_hash_read(ring_bin):
    # every misalignment x every length from 1 B to 10 chunks: all chunk phases, short and padding-only last chunks
    r = subprocess.run([ring_bin, "1300"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip() == "ok %d" % (16 * 1300)


def test_schedule_fails_when_the_shared_granule_is_copied_before_the_hash(ring_bin, tmp_path):
    # the same simulation with ring_step's second copy moved in front of the hash must report the overwrite
    src = open(os.path.join(CSRC, "ctmr_common.cuh")).read()
    before = "    copy(r.y0, r.ymid);\n    hash();\n    copy(r.ymid, r.y1);\n"
    assert before in src
    early = src.replace(before, "    copy(r.y0, r.ymid);\n    copy(r.ymid, r.y1);\n    hash();\n")
    for rel in ("ct_mapreduce_b200/csrc", "include", "tests/cpp"):  # the headers' relative includes keep working
        os.makedirs(tmp_path / rel)
        for name in os.listdir(os.path.join(ROOT, rel)):
            if name.endswith((".cuh", ".h", "ring_schedule.cu")):
                text = early if name == "ctmr_common.cuh" else open(os.path.join(ROOT, rel, name)).read()
                (tmp_path / rel / name).write_text(text)
    from ct_mapreduce_b200 import build
    subprocess.run([build._nvcc(), "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                    "-o", str(tmp_path / "early"), str(tmp_path / "tests/cpp/ring_schedule.cu")], check=True)
    r = subprocess.run([str(tmp_path / "early"), "300"], capture_output=True, text=True)
    assert r.returncode == 1 and "FAIL m=1 " in r.stdout and "the hash" in r.stdout, r.stdout
