"""Cluster-local deletion (ctmr_rollback.cu) restated on a Python linear-probing table.

A slot is None (zeroed) or (epoch, key, first): live only at the current epoch.  home(key) is the probe start.  The
select pass marks the first removed slot of every cluster (a maximal run of live slots, wrapping at the table's end; a
table with no empty slot is one cyclic cluster owned by its lowest removed slot), and each owner walks its cluster from
there: read a slot, clear it, place a survivor again at the first empty slot from its home.  In a table with no empty
slot that walk has no cluster start to begin from: its owner first deletes itself by backward shifting (Knuth's
Algorithm R), which leaves one empty slot, and walks the one cluster that remains from its first removed slot.
"""
from __future__ import annotations


class Table:
    def __init__(self, n: int, home, epoch: int = 1):
        self.n, self.home, self.epoch = n, home, epoch
        self.slots: list = [None] * n

    def live(self, i: int) -> bool:
        s = self.slots[i]
        return s is not None and s[0] == self.epoch

    def insert(self, key, first: int) -> int:
        """Find-or-insert as the batch path does it: the lowest first-seen index wins."""
        pos = self.home(key) % self.n
        for _ in range(self.n):
            if not self.live(pos):
                self.slots[pos] = (self.epoch, key, first)
                return pos
            if self.slots[pos][1] == key:
                e, k, f = self.slots[pos]
                self.slots[pos] = (e, k, min(f, first))
                return pos
            pos = (pos + 1) % self.n
        raise OverflowError("table full")

    def find(self, key):
        pos = self.home(key) % self.n
        for _ in range(self.n):
            if not self.live(pos):
                return None
            if self.slots[pos][1] == key:
                return pos
            pos = (pos + 1) % self.n
        return None

    def records(self) -> dict:
        return {self.slots[i][1]: self.slots[i][2] for i in range(self.n) if self.live(i)}


def removed(t: Table, i: int, since: int) -> bool:
    return t.live(i) and t.slots[i][2] >= since


NOT_OWNER, OWNER, OWNER_NO_EMPTY = 0, 1, 2


def first_removed(t: Table, i: int, since: int) -> int:
    """first_removed of ctmr_rollback.cu: whether removed slot i owns its cluster, and whether the table has no empty slot."""
    wrapped = False
    for k in range(1, t.n):
        q = (i - k) % t.n
        if not t.live(q):
            return NOT_OWNER if wrapped else OWNER
        if removed(t, q, since):
            if q < i:
                return NOT_OWNER
            wrapped = True
    return OWNER_NO_EMPTY


def select(t: Table, since: int) -> list:
    return [(i, o) for i in range(t.n) if removed(t, i, since) for o in [first_removed(t, i, since)] if o != NOT_OWNER]


def shift_delete(t: Table, i: int) -> int:
    """Algorithm R: slot i out, the records behind it shifted back where their probe allows; returns the empty slot left."""
    t.slots[i] = None
    j = i
    while True:
        j = (j + 1) % t.n
        if not t.live(j):
            return i
        k = t.home(t.slots[j][1]) % t.n
        if (k - i - 1) % t.n < (j - i) % t.n:  # home in (i, j]: the record stays
            continue
        t.slots[i], t.slots[j] = t.slots[j], None
        i = j


def rebuild_cluster(t: Table, f: int, since: int, no_empty: bool = False) -> None:
    if no_empty:
        e = shift_delete(t, f)
        f = next((q for q in ((e + d) % t.n for d in range(1, t.n)) if removed(t, q, since)), None)
        if f is None:
            return
    for k in range(t.n):
        r = (f + k) % t.n
        s = t.slots[r]
        if k > 0 and not t.live(r):
            break
        t.slots[r] = None
        if s[2] >= since:
            continue
        pos = t.home(s[1]) % t.n
        while t.live(pos):
            pos = (pos + 1) % t.n
        t.slots[pos] = s


def rollback(t: Table, since: int) -> list:
    """Every record first seen at or above `since` out of t, cluster by cluster; returns the owners."""
    owners = select(t, since)
    for f, o in owners:
        rebuild_cluster(t, f, since, o == OWNER_NO_EMPTY)
    return [f for f, _ in owners]


def clusters(t: Table) -> list:
    """The clusters of t as lists of slot positions in probe order."""
    if all(t.live(i) for i in range(t.n)):
        return [list(range(t.n))]
    start = next(i for i in range(t.n) if not t.live(i))
    out, cur = [], []
    for k in range(1, t.n + 1):
        i = (start + k) % t.n
        if t.live(i):
            cur.append(i)
        elif cur:
            out.append(cur)
            cur = []
    return out


def rollback_reference(t: Table, since: int) -> None:
    """The literal rule, from scratch: every cluster that holds a removed record is cleared whole, and its survivors are
    inserted again in ascending old position (probe order from the cluster's start)."""
    for cl in clusters(t):
        if not any(removed(t, i, since) for i in cl):
            continue
        keep = [t.slots[i] for i in cl if not removed(t, i, since)]
        for i in cl:
            t.slots[i] = None
        for s in keep:
            pos = t.home(s[1]) % t.n
            while t.live(pos):
                pos = (pos + 1) % t.n
            t.slots[pos] = s
