"""The mailbox word of a collective call's agreements, checked on the host: every rank of a front-end, checkpoint, CRL or
batch call posts one word, its payload or its failure with the error code, and every rank decides from the same row of
words.  peer_word and its readers (ctmr_kernels.cuh, compiled unchanged) must give every error code back, leave every
payload below 2^63 untouched, never read a failure as a payload, and name the lowest rank that failed."""
import os
import subprocess

from conftest import ROOT


def test_peer_word_round_trips_codes_and_payloads(tmp_path):
    from ct_mapreduce_b200 import build
    out = tmp_path / "peer_word"
    subprocess.run([build._nvcc(), "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(out),
                    os.path.join(ROOT, "tests", "cpp", "peer_word.cpp")], check=True)
    r = subprocess.run([str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("ok "), r.stdout
