"""The restated key exchange (tests/xchg_model.py) checked without a GPU: key_owner against the library's compiled
function, the round plan's invariants, the owner-choosing hours, the warp composition claim both map kernels rely on in
tests/test_gpu_exchange.py, and the full regions of that file's T3 corpus."""
import os
import subprocess

import numpy as np
import pytest

import keymodel as K
import xchg_model as X
from conftest import ROOT


@pytest.fixture(scope="module")
def owner_bin(tmp_path_factory):
    from ct_mapreduce_b200 import build
    out = tmp_path_factory.mktemp("ownerbin") / "key_owner"
    subprocess.run([build._nvcc(), "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                    "-o", str(out), os.path.join(ROOT, "tests", "cpp", "key_owner.cu")], check=True)
    return str(out)


def test_key_owner_equals_the_compiled_function(owner_bin):
    rng = np.random.default_rng(5)
    hours = [0, 1, -1, -2, 2**31 - 1, -2**31, X.BASE_HOUR, -X.BASE_HOUR] + rng.integers(-2**31, 2**31, 200).tolist()
    issuers = [0, 1, 2**31, 2**32 - 1, 2**32 - 2, 2**32 - 3] + rng.integers(0, 2**32, 40).tolist()
    triples = [(h, i, w) for w in range(1, 9) for h in hours[:40] for i in issuers[:12]]
    triples += [(int(h), int(i), int(w)) for h, i, w in zip(hours, rng.choice(issuers, len(hours)), rng.integers(1, 9, len(hours)))]
    r = subprocess.run([owner_bin], input="".join("%d %d %d\n" % t for t in triples), capture_output=True, text=True, check=True)
    got = [int(x) for x in r.stdout.split()]
    assert got == [X.key_owner(h, i, w) for h, i, w in triples]
    assert all(g == 0 for g, (_, _, w) in zip(got, triples) if w == 1)


def _offsets(lengths):
    o = np.zeros(len(lengths) + 1, np.uint64)
    o[1:] = np.cumsum(lengths)
    return o


@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
def test_plan_rounds_invariants(W):
    rng = np.random.default_rng(W)
    for n in (0, 1, W - 1, W, W + 1, 255, 256 * W, 256 * W + 1, 3001):
        for E, B in ((256, 2048 * 256), (256, 64 * 1024), (7, 6000), (1, 10**9)):
            lengths = rng.integers(300, 6001, n)
            offs = _offsets(lengths)
            plan = X.plan_rounds(offs, W, E, B)
            seen = np.zeros(n, int)
            pos = 0
            for rnd in plan:
                assert [r for r, _, _ in rnd] == list(range(W))            # every member, ascending
                q = max(hi - lo for _, lo, hi in rnd)
                for r, lo, hi in rnd:
                    assert 0 <= hi - lo <= E and int(offs[hi] - offs[lo]) <= B
                    assert lo == min(n, pos + r * q)                       # contiguous slices of one q, in entry order
                    seen[lo:hi] += 1
                pos = rnd[-1][2]
                assert any(hi > lo for _, lo, hi in rnd)
            assert (seen == 1).all()
            if n < W and n:
                assert len(plan) == 1 and sum(hi > lo for _, lo, hi in plan[0]) == n
            if n == 0:
                assert plan == []
            # the member that maps an entry, and the status counts it keeps
            if n:
                mem = X.member_of(plan, n)
                st = rng.integers(0, 8, n)
                by = X.status_by_member(plan, st, W)
                for r in range(W):
                    assert by[r].tolist() == np.bincount(st[mem == r], minlength=8).tolist()


def test_plan_rounds_shrinks_and_refuses():
    lengths = [300] * 10 + [6000] * 10 + [300] * 10
    plan = X.plan_rounds(_offsets(lengths), 3, 256, 20000)
    assert [max(hi - lo for _, lo, hi in rnd) for rnd in plan][0] < 10    # q = 10 does not fit: halved
    with pytest.raises(ValueError):
        X.plan_rounds(_offsets([300, 7000]), 2, 256, 6000)


def test_stage_budget_and_exchange_entries():
    assert X.stage_budget() == (1 << 18, 2048 << 18) and X.stage_budget(0, 1 << 40) == (1 << 18, 768 << 20)
    assert X.stage_budget(256) == (256, 2048 * 256)
    assert X.stage_budget(1 << 20, 1 << 16) == (1 << 18, 1 << 16)
    assert X.exchange_entries(128, 256) == 256 and X.exchange_entries(256, 0) == 256 and X.exchange_entries(256, 100) == 256
    # the collective device call: n with exactly X per round, and one entry more
    assert X.device_round_entries(1850, 8) == 256 and X.device_round_entries(1857, 8) == 257


@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
def test_hour_for_reaches_every_owner(W):
    for issuer in range(X.N_ISSUERS + 1):
        for owner in range(W):
            h = X.hour_for(issuer, W, owner, X.BASE_HOUR)
            assert h > X.BASE_HOUR and X.key_owner(h, issuer, W) == owner and h - X.BASE_HOUR < 200


def test_warp_composition_claim():
    """Slices of 32-entry groups, each group with its own 128-byte chunk count: the stream kernel's length order makes each
    group exactly one warp, whatever the order inside a bucket; equal chunk counts in two groups break the claim."""
    rng = np.random.default_rng(2)
    for groups in (3, 8):
        lengths = [X.group_length(g) + int(rng.integers(-4, 5)) for g in rng.permutation(groups) for _ in range(32)]
        assert X.warp_sets_are_fixed(lengths)
        want = {frozenset(range(32 * g, 32 * g + 32)) for g in range(groups)}
        assert set(X.stream_warps(lengths)) == want
        # another order inside the buckets: the same warps
        perm = rng.permutation(len(lengths))
        assert {frozenset(int(perm[e]) for e in w) for w in X.stream_warps([lengths[p] for p in perm])} == want
    same = [X.group_length(0)] * 48 + [X.group_length(1)] * 16
    assert not X.warp_sets_are_fixed(same)
    # the builders hit those chunk counts, rejected kinds included
    for g in range(8):
        for pattern in X.WARP_PATTERNS:
            es = X.warp_entries(pattern, 8, g % 8, 1000 * g, g)
            assert {(len(d) + 127) >> 7 for d, _, _ in es} == {3 + g}


def test_len_bucket_longest_first():
    assert X.len_bucket(0) == 255 and X.len_bucket(1) == 254 and X.len_bucket(128) == 254 and X.len_bucket(129) == 253
    assert X.len_bucket(10**6) == 0 and X.len_bucket(255 * 128) == 0 and X.len_bucket(254 * 128) == 1


@pytest.mark.parametrize("W", [3, 8])
def test_warp_targets(W):
    for m in range(W):
        for pattern in X.WARP_PATTERNS:
            t = X.warp_targets(pattern, W, m)
            remote = [x for x in t if not isinstance(x, str) and x != m]
            if pattern == "own":
                assert not remote
            elif pattern == "one_remote":
                assert len(remote) == 1
            elif pattern == "all_remote_but_one":
                assert len(remote) == 31
            elif pattern == "lane_mod_world":
                assert sorted(set(t)) == list(range(W))
            elif pattern == "remote_between_rejected":
                assert set(x for x in t if isinstance(x, str)) == set(X.REJECTED) and len(remote) == 16


def test_t3_inbox_regions():
    es, kinds = X.t3_corpus()
    offs = _offsets([len(d) for d, _, _ in es])
    plan = X.plan_rounds(offs, 3, 256, 2048 * 256)
    assert len(plan) == len(kinds) + 1 and [hi - lo for _, lo, hi in plan[-1]] == [1, 1, 0]
    owners = X.owners_of(es)
    counts, full = X.inbox_counts(plan, owners, owners >= 0, 256)
    assert full == [k for k, kind in enumerate(kinds) if kind == "to2"]
    for k, kind in enumerate(kinds):
        total = sum(v for (kk, _, _, _), v in counts.items() if kk == k)
        if kind == "to2":
            assert counts[(k, k % 3, 0, 2)] == counts[(k, k % 3, 1, 2)] == 256 and total == 512
        elif kind == "own":
            assert total == 0
        else:
            assert 0 < total < 512
    # every parity is reused with another fill: full, empty and partial each meet every parity at least once
    fills = {}
    for k, kind in enumerate(kinds):
        fills.setdefault(k % 3, set()).add(kind)
    assert all(len(v) >= 2 for v in fills.values()) and fills[0] >= {"to2", "own"}
    assert kinds[3] == "own" and kinds[0] == "to2"    # an empty round right after a full round of the same parity
    assert counts[(10, 1, 0, 1)] == 1 and counts[(10, 1, 1, 2)] == 1


def test_shard_expectations_split_the_model():
    km = K.KeyModel()
    for j in range(60):
        h = X.BASE_HOUR + j % 7
        X.preload(km, h, j % 5, [bytes([1 + j, 2])], j)
    for W in (1, 3, 8):
        sh = X.shard_expectations(km, W)
        assert sum(len(s.model.first) for s in sh) == len(km.first)
        assert sum(len(s.model.pair_first) for s in sh) == len(km.pair_first)
        for r, s in enumerate(sh):
            assert all(X.key_owner(k[0], k[1], W) == r for k in s.model.first)
            assert sum(s.hist.values()) == len(s.model.first)
