"""The GPU's split of revokedCertificates restated (ctmr_crl.cu): candidates, links and reach doubling, next to the
serial walk it replaces.

A candidate is a position p of the content [0, n) that starts 30 L 02 with a well-formed definite length and a TLV that
stays inside the content; next(p) = p + TLV size.  link(p) is the candidate at next(p), END at n, NONE otherwise.  From
the candidate at 0, round k marks jump_k(c) for every marked c and composes jump_{k+1} = jump_k o jump_k.  The content
splits iff the marked chain ends at END after ceil(log2(n // 18 + 1)) rounds (no chain of well-formed entries is
longer); its entries are the marked candidates.
"""
from __future__ import annotations

from crl_oracle import Bad, read

END, NONE = -1, -2
MIN_ENTRY = 18


def candidates(d: bytes):
    """[(p, next(p))] in position order."""
    out = []
    for p in range(len(d)):
        if d[p] != 0x30:
            continue
        try:
            tag, h, n = read(d, p, len(d))
        except Bad:
            continue
        if n >= 1 and d[p + h] == 0x02:
            out.append((p, p + h + n))
    return out


def rounds_for(n_bytes: int) -> int:
    chain, r = n_bytes // MIN_ENTRY + 1, 0
    while (1 << r) < chain:
        r += 1
    return r


def split(d: bytes, rounds: int | None = None):
    """(complete, entry positions, rounds used) of content d by reach doubling."""
    cand = candidates(d)
    if not d:
        return True, [], 0
    idx = {p: i for i, (p, _) in enumerate(cand)}
    link = [END if nx == len(d) else idx.get(nx, NONE) for _, nx in cand]
    mark = [p == 0 for p, _ in cand]
    jump = list(link)
    R = rounds_for(len(d)) if rounds is None else rounds
    for _ in range(R):  # synchronous rounds: the GPU may mark more, never fewer
        new = list(mark)
        for i, j in enumerate(jump):
            if mark[i] and j >= 0:
                new[j] = True
        jump = [jump[j] if j >= 0 else j for j in jump]
        mark = new
    done = any(m and link[i] == END for i, m in enumerate(mark))
    broken = any(m and link[i] == NONE for i, m in enumerate(mark))
    return done and not broken, [cand[i][0] for i, m in enumerate(mark) if m], R


def walk(d: bytes):
    """The serial walk: (complete, entry positions) following TLV sizes from 0."""
    out, p = [], 0
    while p < len(d):
        try:
            tag, h, n = read(d, p, len(d))
        except Bad:
            return False, out
        if tag != 0x30 or n < 1 or d[p + h] != 0x02:
            return False, out
        out.append(p)
        p += h + n
    return True, out
