"""The classify kernel's bit arithmetic (tests/json_model.py, the words of csrc/ctmr_json.cu) against a byte-at-a-time
reading: every body start mod 64, backslash runs of 0 to 130 ending at and across block edges, quotes as the first or
last byte of a block, abutting bodies."""
import random

import pytest

import json_model as jm


def _check(text, starts):
    e1, s1 = jm.classify(text, starts)
    e2, s2 = jm.byte_scan(text, starts)
    for k in range(len(e2)):
        valid = jm.M64 if 64 * k + 64 <= len(text) else (1 << (len(text) - 64 * k)) - 1
        assert e1[k] & valid == e2[k], (k, text, starts)
        assert s1[k] & valid == s2[k], (k, text, starts)


@pytest.mark.parametrize("start", range(64))
def test_every_body_start_mod_64(start):
    rng = random.Random(start)
    body = bytes(rng.choice(b'ab"\\{}: ') for _ in range(150))
    _check(b"x" * start + body, [0, start] if start else [0])


@pytest.mark.parametrize("run", range(131))
def test_backslash_runs_at_and_across_block_edges(run):
    for end in (63, 64, 65, 127, 128):  # the run's last backslash at these offsets, then a quote
        lead = max(0, end + 1 - run)
        text = b'"' + b"a" * max(0, lead - 1) + b"\\" * run + b'"x"'
        _check(text, [0])
        _check(b'"\\' + text, [0, 2])  # an open string and a dangling backslash before the start: both restart


@pytest.mark.parametrize("pos", [0, 1, 62, 63, 64, 127, 128])
def test_quotes_first_and_last_byte_of_a_block(pos):
    text = bytearray(b"a" * 200)
    text[pos] = 0x22
    text[pos + 70] = 0x22
    _check(bytes(text), [0])
    _check(bytes(text), [0, pos])


def test_abutting_bodies():
    rng = random.Random(7)
    for _ in range(300):
        parts = [bytes(rng.choice(b'"\\a{') for _ in range(rng.randrange(0, 90))) for _ in range(rng.randrange(1, 8))]
        starts, at = [], 0
        for p in parts:
            starts.append(at)
            at += len(p)
        _check(b"".join(parts), starts)


def test_compose_is_associative():
    rng = random.Random(3)
    for _ in range(500):
        a, b, c = (rng.randrange(256) for _ in range(3))
        assert jm.compose(jm.compose(a, b), c) == jm.compose(a, jm.compose(b, c))
        assert jm.compose(jm.IDENTITY, a) == a == jm.compose(a, jm.IDENTITY)
