"""The CRL catalogue (tests/crl_cases.py) without a GPU: crl_oracle gives every hand-written outcome, the split model
equals the serial walk on every revokedCertificates content, the seeded mutants reach every status in a real share,
and the pair hash restated in numpy equals the library's compiled pair_hash."""
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

import crl_cases as cc
import crl_oracle as co
import crl_pair_model as pm
from conftest import ROOT
from crl_split_model import MIN_ENTRY, candidates, split, walk


def test_oracle_gives_every_hand_written_outcome():
    for c in cc.catalogue():
        p = co.parse_crl(c.der)
        assert p["status"] == c.status, c.name
        if c.entries is not None:
            assert [e["status"] for e in p["entries"]] == c.entries, c.name
        f = c.fields
        for k, key in (("this_update", "this_update"), ("next_update", "next_update"), ("flags", "flags")):
            if k in f:
                assert p[key] == f[k], c.name
        for k, key in (("revoked_at", "revoked_at"), ("reason", "reason")):
            if k in f:
                assert [e[key] for e in p["entries"]] == f[k], c.name
        if "serial_len" in f:
            assert [min(len(e["serial"]), 255) for e in p["entries"]] == f["serial_len"], c.name


def test_catalogue_covers_the_families():
    cat = cc.catalogue()
    names = {c.name for c in cat}
    for lv in cc.LEVELS:
        for m in cc.MODS:
            assert f"header_{lv}_{m}" in names
    long = [c for c in cat if "_long_" in c.name and c.status == cc.OK]
    assert {b"\x81\x80", b"\x82\x01\x00", b"\x83\x01\x00\x00"} <= {f for c in long for f in
                                                                     (b"\x81\x80", b"\x82\x01\x00", b"\x83\x01\x00\x00")
                                                                     if f in c.der}
    for nm, _, _, sec in cc.TIMES:
        for where in ("this", "next", "rdate"):
            assert f"time_{where}_{nm}" in names
    assert {co.CRL_OK, co.CRL_BAD, co.CRL_BAD_ENTRIES} == {c.status for c in cat}
    # an entry and a serial of more than 127 octets, and serials of 256 and more octets
    assert any(len(e["serial"]) >= 256 for c in cat for e in co.parse_crl(c.der)["entries"])


def test_split_equals_walk_on_every_content():
    n = 0
    for c in list(cc.catalogue()) + cc.mutants(n_seeds=10):
        p = co.parse_crl(c.der if isinstance(c, cc.Case) else c)
        if p["status"] == co.CRL_BAD or not p.get("content"):
            continue
        d = (c.der if isinstance(c, cc.Case) else c)[p["content"][0]:p["content"][1]]
        ok, pos, _ = split(d)
        wok, wpos = walk(d)
        ends = wpos[1:] + [len(d)]
        if wok and any(e - s < MIN_ENTRY for s, e in zip(wpos, ends)):
            # a chain of TLVs too short to be entries may outrun the rounds; such content is never a list of entries
            assert p["status"] == co.CRL_BAD_ENTRIES and (not ok or pos == wpos), getattr(c, "name", None)
            continue
        assert ok == wok, getattr(c, "name", None)
        if ok:
            assert pos == wpos
        n += 1
    assert n > 1000


def test_split_edges_are_where_the_names_say():
    cat = {c.name: c for c in cc.catalogue()}
    # entries at every phase mod 16 inside one CRL, and CRL lengths of 16k + 1 back to back
    p = co.parse_crl(cat["split_entries_every_phase"].der)
    d = cat["split_entries_every_phase"].der
    starts = walk(d[p["content"][0]:p["content"][1]])[1]
    assert {(p["content"][0] + s) % 16 for s in starts} == set(range(16))
    bnd = [cat[f"split_boundary_{i}"].der for i in range(16)]
    assert all(len(b) % 16 == 1 for b in bnd)
    assert {sum(len(b) for b in bnd[:i]) % 16 for i in range(16)} == set(range(16))
    for k in range(1, 13):
        for n in ((1 << k) - 1, 1 << k, (1 << k) + 1):
            c = cat[f"split_chain_{n}"]
            p = co.parse_crl(c.der)
            assert p["content"][1] - p["content"][0] == 18 * n and len(p["entries"]) == n
    # the false candidates land where their names say, and are candidates of the split
    for c in cat.values():
        if not c.name.startswith("split_false_"):
            continue
        p = co.parse_crl(c.der)
        d = c.der[p["content"][0]:p["content"][1]]
        real = set(walk(d)[1]) if p["status"] == co.CRL_OK else set()
        false = [(q, nx) for q, nx in candidates(d) if q not in real]
        if c.name.endswith("_past"):
            assert not false
        elif c.name.endswith("_end"):
            assert any(nx == len(d) for _, nx in false), c.name
        elif c.name.endswith("_next"):
            assert any(nx in real for _, nx in false), c.name


def test_mutants_reach_every_status():
    ms = cc.mutants()
    assert 15000 <= len(ms) <= 25000
    st = Counter(co.parse_crl(d)["status"] for d in ms)
    for s in (co.CRL_OK, co.CRL_BAD, co.CRL_BAD_ENTRIES):
        assert st[s] >= len(ms) // 10, st
    assert cc.mutants() == ms  # seeded


@pytest.fixture(scope="module")
def pair_hash_bin(tmp_path_factory):
    from ct_mapreduce_b200 import build
    out = tmp_path_factory.mktemp("pairhash") / "pair_hash"
    subprocess.run([build._nvcc(), "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                    "-o", str(out), os.path.join(ROOT, "tests", "cpp", "pair_hash.cu")], check=True)
    return str(out)


def test_pair_hash_equals_the_compiled_function(pair_hash_bin):
    rng = np.random.default_rng(9)
    serials = [b"\x01", b"\x00\x01", b"\x01\x00", b"\xff", b"\x7f" * 39] + \
        [bytes(rng.integers(0, 256, int(n), dtype=np.uint8)) for n in rng.integers(1, 40, 300)]
    issuers = [0, 1, 0xFFFFFFFE, 0xFFFFFFFF] + rng.integers(0, 2**32, len(serials) - 4).tolist()
    w = pm.pair_words(issuers, serials)
    w = np.vstack([w, rng.integers(0, 2**32, (200, 11), dtype=np.uint64).astype(np.uint32)])  # every bit of every word
    r = subprocess.run([pair_hash_bin], input="".join(" ".join(str(int(x)) for x in row) + "\n" for row in w),
                       capture_output=True, text=True, check=True)
    got = np.array([int(x) for x in r.stdout.split()], np.uint64)
    assert got.tolist() == pm.pair_hash(w).astype(np.uint64).tolist()


def test_pair_words_layout():
    w = pm.pair_words([7], [bytes(range(1, 40))])[0]
    assert w[0] == 7 and w[1] == 39 | 1 << 8 | 2 << 16 | 3 << 24 and w[10] == 36 | 37 << 8 | 38 << 16 | 39 << 24
    a, b = pm.pair_words([1, 1], [b"\x01", b"\x01\x00"])
    assert a[1] != b[1] and (a[2:] == b[2:]).all()  # only the length tells them apart


def test_crafted_collisions_collide():
    rng = np.random.default_rng(1)
    tags = pm.tag_collisions(3, rng, 1 << 17)
    assert len(tags) >= 2
    for a, b in tags:
        ha, hb = (int(x) for x in pm.pair_hash(pm.pair_words([3, 3], [a, b])))
        assert ha & ~3 == hb & ~3 and ha != hb and a != b
    full = pm.tag_collisions(3, np.random.default_rng(2), 1 << 18, full=True)
    assert full
    for a, b in full:
        ha, hb = pm.pair_hash(pm.pair_words([3, 3], [a, b]))
        assert ha == hb and a != b
    cl = pm.home_cluster(3, np.random.default_rng(3), 128, 125, 40)
    assert len(set(cl)) == 40 and set((pm.pair_hash(pm.pair_words(3, cl)) & 127).tolist()) == {125}
    assert pm.set_slots(0) == 64 and pm.set_slots(33) == 128 and pm.set_slots(64) == 128 and pm.set_slots(65, 512) == 512
