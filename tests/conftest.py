import base64
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")
NOW_SEC = 1767225600  # 2026-01-01T00:00:00Z, the corpus' fixed "now" (SURVEY.md §8(d))
NOW_NS = NOW_SEC * 10**9
README_FILTER = b"Let's Encrypt, ISRG"  # reference README.md:29, split without trimming


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 box)")


def pem_to_der(path):
    body = "".join(l.strip() for l in open(path) if "-----" not in l)
    return base64.b64decode(body)


@pytest.fixture(scope="session")
def golden():
    fx = json.load(open(os.path.join(GOLDEN, "fixtures.json")))
    for name in fx:
        fx[name]["der"] = pem_to_der(os.path.join(GOLDEN, name + ".pem"))
    return fx


@pytest.fixture(scope="session")
def ora():
    from oracle import oracle
    oracle.lib()
    return oracle


def go_pem(der: bytes) -> bytes:
    """encoding/pem.EncodeToMemory(&pem.Block{Type: "CERTIFICATE", Bytes: der}) -- what FilesystemDatabase.Store
    passes to StoreCertificatePEM (storage/filesystemdatabase.go:171-175,197-198): 64-character lines."""
    b = base64.b64encode(der)
    lines = b"".join(b[i:i + 64] + b"\n" for i in range(0, len(b), 64))
    return b"-----BEGIN CERTIFICATE-----\n" + lines + b"-----END CERTIFICATE-----\n"


def pack(ders):
    """list of bytes -> (blob u8, offsets u64)"""
    offsets = np.zeros(len(ders) + 1, np.uint64)
    offsets[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
    blob = np.frombuffer(b"".join(ders), np.uint8).copy() if ders else np.zeros(0, np.uint8)
    return blob, offsets
