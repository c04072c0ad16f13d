"""Cluster-local deletion (tests/rollback_model.py, the rule ctmr_rollback.cu runs on the GPU) against a rebuild from
scratch: the same records, every survivor found, none further from home or past its old slot, nothing outside the
rebuilt clusters touched."""
import random

import pytest

from rollback_model import Table, clusters, rollback, rollback_reference


def _check(t: Table, since: int, cyclic: bool = False):
    before = list(t.slots)
    old_pos = {t.slots[i][1]: i for i in range(t.n) if t.live(i)}
    want_records = {k: f for k, f in t.records().items() if f < since}
    touched = set()
    for cl in clusters(t):
        if any(t.live(i) and t.slots[i][2] >= since for i in cl):
            touched.update(cl)
    ref = Table(t.n, t.home, t.epoch)
    ref.slots = list(t.slots)
    rollback_reference(ref, since)
    rollback(t, since)
    assert t.records() == want_records
    for k in want_records:
        pos = t.find(k)
        assert pos is not None, k
        h = t.home(k) % t.n
        assert (pos - h) % t.n <= (old_pos[k] - h) % t.n  # no further from home than before
        assert all(t.live((h + d) % t.n) for d in range((pos - h) % t.n + 1))  # the probe rule: no hole on the way
    for k in set(old_pos) - set(want_records):
        assert t.find(k) is None
    for i in range(t.n):
        if i not in touched:
            assert t.slots[i] == before[i], i
    if not cyclic:
        assert t.slots == ref.slots  # the same placement as clearing each cluster and inserting its survivors in order
    return t


def _fill(n, homes, firsts, epoch=1):
    """keys 0.. with the given homes, inserted in order with the given first-seen indices"""
    t = Table(n, lambda k: homes[k], epoch)
    for k, f in enumerate(firsts):
        t.insert(k, f)
    return t


def test_removed_at_cluster_first_and_last_position():
    # one cluster 2..7, all homed at 2: remove the first and the last record
    t = _fill(16, [2] * 6, [0, 1, 2, 3, 4, 10])
    t.slots[2] = (1, 0, 11)  # the cluster's first slot is removed too
    _check(t, 10)
    assert t.find(1) == 2 and t.find(4) == 5 and t.slots[6] is None and t.slots[7] is None


def test_survivor_whose_home_lies_before_a_removed_slot():
    # keys 0, 1 home 4; key 2 home 4 lands at 6; key 1 removed: key 2 moves to 5
    t = _fill(16, [4, 4, 4, 7], [0, 9, 1, 2])
    _check(t, 9)
    assert t.find(2) == 5 and t.find(3) == 7  # key 3 is at home and stays


def test_cluster_that_wraps_the_table_end():
    n = 16
    homes = [13, 13, 14, 15, 15, 0, 1, 13]
    t = _fill(n, homes, [0, 20, 1, 2, 21, 3, 22, 4])
    assert t.live(15) and t.live(0) and t.live(2)
    _check(t, 20)


def test_removed_slots_on_both_sides_of_the_wrap_elect_one_owner():
    n = 8
    t = _fill(n, [6, 6, 6, 6, 6], [0, 10, 1, 11, 2])  # 6, 7, 0, 1, 2
    from rollback_model import select
    assert select(t, 10) == [(7, 1)]
    _check(t, 10)


def test_slots_of_an_earlier_epoch_inside_a_run():
    t = Table(16, lambda k: k % 16, epoch=2)
    t.slots[5] = (1, 99, 0)  # left by epoch 1: empty now, and claimed by the insert below
    t.slots[6] = (1, 98, 0)  # left by epoch 1 and never claimed: a cluster boundary inside the run 3..9
    for k, f in [(3, 0), (3 + 16, 7), (3 + 32, 1), (7, 8), (7 + 16, 2), (7 + 32, 9), (7 + 48, 3)]:
        t.insert(k, f)
    assert t.slots[5] == (2, 3 + 32, 1)
    assert [t.live(i) for i in range(3, 11)] == [True, True, True, False, True, True, True, True]
    _check(t, 7)
    assert t.slots[6] == (1, 98, 0)  # never touched: the walk of cluster 3..5 ends there, cluster 7..10 starts after it
    assert t.find(3 + 32) == 4 and t.find(7 + 16) == 7 and t.find(7 + 48) == 8


def test_table_with_one_empty_slot():
    n = 16
    rnd = random.Random(5)
    homes = [rnd.randrange(n) for _ in range(n - 1)]
    firsts = list(range(n - 1))
    rnd.shuffle(firsts)
    t = _fill(n, homes, firsts)
    assert sum(not t.live(i) for i in range(n)) == 1
    _check(t, 8)


def test_table_with_no_empty_slot_is_one_cyclic_cluster():
    n = 16
    rnd = random.Random(9)
    homes = [rnd.randrange(n) for _ in range(n)]
    firsts = list(range(n))
    rnd.shuffle(firsts)
    t = _fill(n, homes, firsts)
    assert all(t.live(i) for i in range(n))
    _check(t, 11, cyclic=True)


@pytest.mark.parametrize("seed", range(30))
def test_full_tables(seed):
    rnd = random.Random(1000 + seed)
    n = rnd.choice([4, 8, 16, 32])
    homes = [rnd.randrange(n) if rnd.random() < 0.5 else rnd.choice([0, n - 1]) for _ in range(n)]
    firsts = list(range(n))
    rnd.shuffle(firsts)
    t = _fill(n, homes, firsts)
    assert all(t.live(i) for i in range(n))
    _check(t, rnd.randrange(n + 1), cyclic=True)


def test_nothing_removed_and_everything_removed():
    t = _fill(32, [3] * 10, list(range(10)))
    _check(t, 10)
    assert len(t.records()) == 10
    _check(t, 0)
    assert t.records() == {}
    assert all(s is None for s in t.slots)


def test_clusters_longer_than_the_probe_limit():
    n = 1 << 14
    t = _fill(n, [100] * 5000 + [200] * 50, list(range(5050)))
    _check(t, 4990)
    assert len(t.records()) == 4990


@pytest.mark.parametrize("seed", range(40))
@pytest.mark.parametrize("load", [0.3, 0.7, 0.95])
def test_random_tables(seed, load):
    rnd = random.Random(seed * 7 + int(load * 100))
    n = rnd.choice([8, 16, 64, 256])
    m = max(1, int(n * load))
    homes = [rnd.randrange(n) if rnd.random() < 0.7 else rnd.choice([0, n - 1, n // 2]) for _ in range(m)]
    t = _fill(n, homes, list(range(m)))
    for k in rnd.sample(range(m), m // 4):  # records seen again later keep their lowest index
        t.insert(k, m + k)
    since = rnd.randrange(m + 1)
    _check(t, since)
