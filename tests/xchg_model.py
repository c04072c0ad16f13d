"""The key exchange of a group, restated in Python: which member owns a key, how a batch is cut into rounds, how many
records each inbox region receives, which shard must hold which key, pair and histogram count, and which member counts
which entry's status.  Plus builders of leaves whose owner, length and warp the tests choose.

Only what the library decides is modelled here; the oracle and tests/keymodel.py stay the truth for per-entry results.

Mirrors, and must change with:
  ctmr_device.cuh   key_owner (mix64((issuer << 32) | (u32)exp_hour) % world)
  ctmr_api.cu       ctmr_create: stage_entries = min(max_batch_entries, 2^18) (2^18 when 0), stage_bytes =
                    min(max_batch_bytes or 2048 * stage_entries, 768 MiB); alloc_exchange: X = max(max_round_entries,
                    stage_entries); device_round_entries; round_resolve's order (K_resolve, inbox resolve, K_pairs,
                    inbox pairs); the owner-side passes count what they resolve (resolve_one at the owner only)
  ctmr_pipeline.cu  plan_rounds (q = min(E, ceil(rest / W)), halved as (q + 1) / 2 until every member's slice fits
                    stage_bytes; member r takes [pos + r q, pos + (r + 1) q)); round k uses exchange parity k % 3;
                    entry i of a call has global index next_index + i; preload takes next_index .. next_index + n
  ctmr_map.cu       route_append (one region per (parity, source, owner), records in lane order of a warp),
                    map_light_kernel (a warp = 32 consecutive entries of the slice), map_stream_kernel with the length
                    order of len_bucket (128-byte chunks, longest first) when a slice has more than 64 entries;
                    K_map counts each entry's status on the member that mapped it
"""
from __future__ import annotations

import numpy as np

import der_build as D
import keymodel as K

M32 = 0xFFFFFFFF
PARITIES = 3
STAGE_ENTRIES_MAX = 1 << 18
STAGE_BYTES_MAX = 768 << 20
LEN_BUCKETS = 256
STATUS_COUNT = 8


def key_owner(hour: int, issuer: int, world: int) -> int:
    """Owner member of the set serials::<expDate>::<issuer> (hour: exp hour, negative allowed; issuer: dense index)."""
    return K.mix64(((issuer & M32) << 32) | (hour & M32)) % world


def stage_budget(max_batch_entries: int = 0, max_batch_bytes: int = 0):
    """(E, B) of a ctx created with these config values: entries and leaf bytes of one member's slice."""
    e = min(max_batch_entries, STAGE_ENTRIES_MAX) if max_batch_entries else STAGE_ENTRIES_MAX
    return e, min(max_batch_bytes or 2048 * e, STAGE_BYTES_MAX)


def exchange_entries(stage_entries: int, max_round_entries: int = 0) -> int:
    """X: records per inbox region."""
    return max(max_round_entries, stage_entries)


def device_round_entries(n: int, rounds: int) -> int:
    if rounds >= 4:
        return (4 * n + 4 * rounds - 4) // (4 * rounds - 3)
    return -(-n // rounds) if rounds else n


def plan_rounds(offsets, W: int, E: int, B: int) -> list:
    """The rounds of one host-buffer call: [[(member, lo, hi)] * W] (empty slices included)."""
    offsets = [int(x) for x in offsets]
    n = len(offsets) - 1
    plan, pos = [], 0
    while pos < n:
        q = min(E, -(-(n - pos) // W))
        while True:
            if all(offsets[min(n, pos + (r + 1) * q)] - offsets[min(n, pos + r * q)] <= B for r in range(W)):
                break
            if q == 1:
                raise ValueError("a single entry exceeds the staging budget")
            q = (q + 1) // 2
        plan.append([(r, min(n, pos + r * q), min(n, pos + (r + 1) * q)) for r in range(W)])
        pos = min(n, pos + W * q)
    return plan


def member_of(plan, n: int) -> np.ndarray:
    """member[i] = the member that mapped entry i."""
    out = np.full(n, -1, np.int64)
    for rnd in plan:
        for r, lo, hi in rnd:
            out[lo:hi] = r
    assert (out >= 0).all()
    return out


def inbox_counts(plan, owners, valid, X: int):
    """Records per (round, parity, source, owner) region, source != owner; asserts none exceeds X.
    Returns (counts dict, sorted rounds in which some region holds exactly X)."""
    owners, valid = np.asarray(owners), np.asarray(valid, bool)
    counts, full = {}, set()
    for k, rnd in enumerate(plan):
        for src, lo, hi in rnd:
            for o in range(len(rnd)):
                if o == src:
                    continue
                c = int((valid[lo:hi] & (owners[lo:hi] == o)).sum())
                assert c <= X, ("region overflow", k, src, o, c)
                counts[(k, k % PARITIES, src, o)] = c
                if c == X:
                    full.add(k)
    return counts, sorted(full)


def owners_of(entries) -> np.ndarray:
    """The owner tags of [(der, idx, tag)] entries as an array, -1 where the entry is rejected or its owner not chosen."""
    return np.array([t if isinstance(t, int) else -1 for _, _, t in entries], np.int64)


def status_by_member(plan, status, W: int) -> np.ndarray:
    """[W, 8] status counts, each entry counted on the member that mapped it."""
    out = np.zeros((W, STATUS_COUNT), np.uint64)
    status = np.asarray(status)
    for rnd in plan:
        for r, lo, hi in rnd:
            out[r] += np.bincount(status[lo:hi], minlength=STATUS_COUNT).astype(np.uint64)
    return out


def hour_for(issuer: int, world: int, owner: int, after: int) -> int:
    """The first exp hour > after whose set (hour, issuer) the given member owns."""
    h = after + 1
    while key_owner(h, issuer, world) != owner:
        h += 1
    return h


def signed_hour(u: int) -> int:
    return u - (1 << 32) if u >= 1 << 31 else u


class Shard:
    """What one member's tables must hold: a KeyModel restricted to the keys and pairs the member owns, and the per-issuer
    histogram of its live keys."""

    def __init__(self):
        self.model = K.KeyModel()
        self.hist: dict = {}


def shard_expectations(km: K.KeyModel, world: int) -> list:
    out = [Shard() for _ in range(world)]
    for k, gi in km.first.items():
        sh = out[key_owner(k[0], k[1], world)]
        sh.model.first[k] = gi
        sh.hist[k[1]] = sh.hist.get(k[1], 0) + 1
    for pk, gi in km.pair_first.items():
        out[key_owner(pk[0], pk[1], world)].model.pair_first[pk] = gi
    return out


def preload(km: K.KeyModel, hour: int, issuer: int, serials, first_index: int):
    """ctmr_group_preload_known as the table sees it: key records with the indices first_index + j, resolved like a batch."""
    for j, s in enumerate(serials):
        k = K.key_body(hour, issuer, s)
        gi = first_index + j
        if k not in km.first:
            pk = (k[0], k[1])
            km.pair_first[pk] = min(km.pair_first.get(pk, gi), gi)
            km.first[k] = gi
    km.next_index = max(km.next_index, first_index + len(serials))


# ------------------------------------------------------------------------------------------------ warp composition

def len_bucket(L: int) -> int:
    """ctmr_map.cu len_bucket: 0 = longest."""
    return (LEN_BUCKETS - 1) - min((L + 127) >> 7, LEN_BUCKETS - 1)


def stream_warps(lengths) -> list:
    """The sets of slice entries that map_stream_kernel's warps take, for a slice of more than 64 entries: a counting sort by
    len_bucket, longest first.  The order inside a bucket is not fixed, so these sets hold only when
    warp_sets_are_fixed(lengths)."""
    order = sorted(range(len(lengths)), key=lambda e: len_bucket(lengths[e]))
    return [frozenset(order[w:w + 32]) for w in range(0, len(order), 32)]


def warp_sets_are_fixed(lengths) -> bool:
    """True when every warp of the stream kernel's order is a whole bucket (or several), so its set of entries does not
    depend on the order inside a bucket."""
    b = [len_bucket(L) for L in lengths]
    order = sorted(range(len(b)), key=lambda e: b[e])
    starts = {0}
    for i in range(1, len(order)):
        if b[order[i]] != b[order[i - 1]]:
            starts.add(i)
    return all(w in starts for w in range(0, len(order), 32))


def group_length(w: int, base_chunks: int = 3) -> int:
    """A leaf length whose chunk count is base_chunks + w, well inside the chunk (so +-4 bytes keep the count)."""
    return 128 * (base_chunks + w) - 60


def sized(L: int, **kw) -> D.Built:
    """D.cert(**kw) padded through the signature length to exactly L bytes (or within 2 bytes of it when a length header
    grows on the way); the chunk count of group_length() lengths is kept either way."""
    b = D.cert(sig_len=17, **kw)
    s = 17
    for _ in range(4):
        d = L - len(b.der)
        if d == 0:
            break
        s = max(1, s + d)
        b = D.cert(sig_len=s, **kw)
    assert abs(len(b.der) - L) <= 2 and (len(b.der) + 127) >> 7 == (L + 127) >> 7, (L, len(b.der))
    return b


# ------------------------------------------------------------------------------------------------ crafted corpora
# Leaves whose key owner the test chooses: issuer k (dense index k: a fresh group registers ISSUERS in order) and an exp
# hour from hour_for.  The last issuer does not parse (CTMR_ISSUER_BAD).

NOW_SEC = 1767225600          # tests/conftest.py NOW_SEC
BASE_HOUR = D.exp_hour(D.NOT_AFTER)
N_ISSUERS = 20
BAD_ISSUER = N_ISSUERS        # issuer_idx of the unparseable issuer certificate
NO_ISSUER = 0xFFFFFFFF
REJECTED = ("ca", "expired", "cn", "no_issuer", "long_serial", "parse", "bad_issuer")
CN_FILTER = b"ca"             # the default issuer CN of der_build leaves; "cn" leaves carry another one


def ca(k: int) -> D.Built:
    key = b"\x00" + D.tlv(0x30, D.tlv(0x02, b"\x00\xc7" + bytes([k + 1]) * 15) + D.tlv(0x02, b"\x01\x00\x01"))
    return D.cert(serial=bytes([0x20 + k]), subject=[[D.cn(b"Exchange CA %d" % k)]], extensions=[D.basic_constraints(True)],
                  spki_bits=key)


def issuers() -> list:
    return [ca(k).der for k in range(N_ISSUERS)] + [b"\x30\x03\x02\x01\x00"]


def leaf(salt: int, hour: int, kind: str = "ok", L: int | None = None):
    """(der, issuer_idx) of one leaf of set (hour, salt % N_ISSUERS); `kind` one of "ok" and REJECTED; L: padded length."""
    issuer = salt % N_ISSUERS
    kw = dict(serial=D.serial_bytes(10, salt=salt), not_after=hour * 3600 + salt % 3600)
    if kind == "ca":
        kw["extensions"] = [D.basic_constraints(True)]
    elif kind == "expired":
        kw["not_after"] = NOW_SEC - 3600 - salt % 1000
    elif kind == "cn":
        kw["issuer"] = [[D.cn(b"zz")]]
    elif kind == "long_serial":
        kw["serial"] = D.serial_bytes(40, salt=salt)
    der = (sized(L, **kw) if L else D.cert(**kw)).der
    if kind == "parse":
        der = b"\x31" + der[1:]
    idx = {"no_issuer": NO_ISSUER, "bad_issuer": BAD_ISSUER}.get(kind, issuer)
    return der, idx


def owned_leaf(salt: int, world: int, owner: int, after: int = BASE_HOUR, L: int | None = None):
    """(der, issuer_idx) of a valid leaf whose key the given member owns."""
    return leaf(salt, hour_for(salt % N_ISSUERS, world, owner, after), "ok", L)


WARP_PATTERNS = ("own", "one_foreign", "lane_mod_world", "one_remote", "all_remote_but_one", "remote_between_rejected")


def warp_targets(pattern: str, world: int, member: int) -> list:
    """Per lane: the owner its key must have, or a REJECTED kind (never routed)."""
    foreign = [o for o in range(world) if o != member]
    out = []
    for i in range(32):
        if pattern == "own":
            t = member
        elif pattern == "one_foreign":
            t = foreign[0]
        elif pattern == "lane_mod_world":
            t = i % world
        elif pattern == "one_remote":
            t = foreign[-1] if i == 17 else member
        elif pattern == "all_remote_but_one":
            t = member if i == 5 else foreign[i % len(foreign)]
        else:  # remote lanes between the rejected entries
            t = foreign[(i // 2) % len(foreign)] if i % 2 == 0 else REJECTED[(i // 2) % len(REJECTED)]
        out.append(t)
    return out


def warp_entries(pattern: str, world: int, member: int, salt: int, group: int):
    """32 entries for one warp: lengths with chunk count 3 + group (so that the stream kernel's length order keeps the group
    one warp when every group of a slice has its own count), keys routed as `pattern` says.  Returns [(der, idx, tag)],
    tag = the key's owner, or the REJECTED kind."""
    out = []
    for i, t in enumerate(warp_targets(pattern, world, member)):
        s = salt + i
        if isinstance(t, str):
            out.append(leaf(s, BASE_HOUR + 3, t, group_length(group)) + (t,))
        else:
            der, idx = owned_leaf(s, world, t, BASE_HOUR + (i % 4) * 9, group_length(group))
            out.append((der, idx, t))
    return out


def t3_corpus(salt: int = 300_000):
    """W = 3, 256 entries per member and round: rounds whose regions are full (members 0 and 1 send all 256 keys to
    member 2), empty (nothing leaves its member) or partly filled, every parity reused with another fill, then a round of
    two entries (member 2 empty).  Returns (entries [(der, idx, tag)] as warp_entries, the kinds of the rounds)."""
    W, E = 3, 256
    kinds = ("to2", "own", "partial", "own", "to2", "own", "partial", "partial", "to2", "to2")
    rng = np.random.default_rng(salt)
    out = []
    for k, kind in enumerate(kinds):
        rnd = []
        for m in range(W):
            for j in range(E):
                s = salt + 1000 * k + 256 * m + j
                if kind == "to2" or kind == "own":
                    t = 2 if kind == "to2" else m
                    rnd.append(owned_leaf(s, W, t, BASE_HOUR + j % 7) + (t,))
                elif j % 9 == 4:
                    kind = REJECTED[j % len(REJECTED)]
                    rnd.append(leaf(s, BASE_HOUR + 1, kind) + (kind,))
                else:
                    t = int(rng.integers(W))
                    rnd.append(owned_leaf(s, W, t, BASE_HOUR + j % 5) + (t,))
        if kind == "to2":  # twins: member 1 repeats some of member 0's keys, member 0 some of member 2's (both routed to 2)
            for j in range(0, E, 16):
                rnd[E + j] = rnd[j]
                rnd[j + 3] = rnd[2 * E + j + 3]
        out += rnd
    out.append(owned_leaf(salt + 99_000, W, 1) + (1,))
    out.append(out[5])
    return out, kinds
