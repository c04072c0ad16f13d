"""The reach-doubling split of revokedCertificates (crl_split_model, restating ctmr_crl.cu) equals the serial walk."""
import random

import numpy as np

import crl_build as cb
from crl_split_model import candidates, rounds_for, split, walk


def _content(entries):
    return b"".join(entries)


def test_serials_and_times_full_of_sequence_bytes():
    rng = random.Random(7)
    ents = []
    for i in range(300):
        serial = bytes([0x30, rng.choice([1, 2, 0x21, 0x30]), 0x02]) * rng.randint(1, 4) + bytes([i & 0x7F | 1])
        ents.append(cb.entry(serial[:39], 1767000000 + i, reason=rng.choice([None, 1, 0x30])))
    d = _content(ents)
    assert len(candidates(d)) > len(ents)  # false candidates inside serials
    ok, pos, _ = split(d)
    assert (ok, pos) == walk(d) and ok and len(pos) == len(ents)


def test_false_candidate_that_merges_into_the_chain_is_not_an_entry():
    # a serial holding 30 03 02 01 xx: its next lands on the following entry's start
    e1 = cb.entry(b"\x30\x03\x02\x01\x05", 1767000000)
    e2 = cb.entry(b"\x42", 1767000001)
    d = e1 + e2
    ok, pos, _ = split(d)
    assert ok and pos == [0, len(e1)]


def test_chain_that_overshoots_the_end_is_rejected():
    e = cb.entry(b"\x01", 1767000000)
    d = e + e[:-1]
    assert not split(d)[0] and not walk(d)[0]
    d = e + b"\x30\x05\x02\x01\x01"  # a last TLV whose length runs past the content
    assert not split(d)[0]


def test_adversarial_3_byte_chain():
    d = b"\x30\x01\x02" * 1000
    ok, pos, R = split(d)
    assert not ok  # the chain reaches END only after 1000 steps: more than 3000 // 18 + 1 entries can hold
    assert len(candidates(d)) == 1000 <= len(d) // 2


def test_candidate_density_never_exceeds_half():
    rng = random.Random(3)
    for _ in range(200):
        d = bytes(rng.choice([0x30, 0x02, 0x81, 0x30, 0x01]) for _ in range(rng.randint(1, 64)))
        assert len(candidates(d)) <= len(d) // 2 + 1


def test_round_counts_from_1_to_2_pow_20_entries():
    for k in (1, 2, 3, 17, 1000):
        d = _content([cb.entry(bytes([1 + i % 120]), 1767000000) for i in range(k)])
        ok, pos, R = split(d)
        assert ok and len(pos) == k and (1 << R) >= k and R == rounds_for(len(d))
    # 2^20 entries: the model's round count; the chain itself is checked on the GPU (tests/test_gpu_crl.py)
    n = 1 << 20
    rows = np.zeros((n, 16), np.uint8)
    rows[:, 0] = 1
    d_len = len(cb.bulk_entries(rows[:1], 1767000000)) * n
    assert (1 << rounds_for(d_len)) >= n and rounds_for(d_len) == 21 and d_len // 18 + 1 > n
