"""ctmr_revoked_verify restated (include/ctmr.h states the rules) with cascade_model.query and stash_model.listed:
verify(R, S, filter, stashes, covered_below) -> (counts, list).

R and S are the cascade's sets for a batch and now, as key records (x, exp_hour, first_index) with x = digest(32) ||
serial: a serial under two hours is two records.  A record is answered revoked when the filter's query says so or a stash
lists x; it is counted under 'before' when first_index < covered_below and under 'since' otherwise.  The list holds the
'before' records answered wrongly as (digest, serial, exp_hour, first_index, blocked), ordered by digest, serial (bytes,
a prefix first) and exp_hour.
"""
from __future__ import annotations

import cascade_model as cm
import stash_model as sm

ALL = 2**64 - 1
NAMES = ("revoked", "missed", "valid", "blocked")


def answers(filter, stashes: bytes = b""):
    """x -> answered revoked, for the filter and the stashes (the filter checked as the stash call checks it)"""
    f = sm.check_filter(filter)
    old = sm.listed(stashes)
    return lambda x: x in old or cm.query(f, x)


def verify(R, S, filter, stashes: bytes = b"", covered_below: int = ALL):
    """({'before': {name: n}, 'since': {name: n}}, list) of the key records R (revoked) and S (valid)"""
    ans = answers(filter, stashes)
    counts = {age: dict.fromkeys(NAMES, 0) for age in ("before", "since")}
    out = []
    for recs, in_r in ((R, True), (S, False)):
        for x, hour, first in recs:
            a = ans(x)
            age = "before" if first < covered_below else "since"
            counts[age][("revoked" if a else "missed") if in_r else ("blocked" if a else "valid")] += 1
            if age == "before" and a != in_r:
                out.append((x[:32], x[32:], hour, first, not in_r))
    out.sort(key=lambda e: (e[0], e[1], e[2]))
    return counts, out
