"""Seeded generators of get-entries response bodies for the GPU body scanner (csrc/ctmr_json.cu).  Every family returns a
list of (body, body_max) pairs; what a body should give is always bodies_oracle.parse_body's answer, never the family's
intent.  The families place bytes where the scanner's bit arithmetic can go wrong: carries at every phase of a 64-byte
block (`phased` sets a body's phase with a sacrificial body before it), tokens and quotes at the edges of a warp's
32-block window, nesting past the 63 levels kept in a register, folded and escaped keys, scalars against every
delimiter, `\\u` escapes, a body spanning many scan tiles, and a grammar fuzz with mutations."""
from __future__ import annotations

import contextlib
import functools
import random
import sys

import bodies_oracle as bo

WS = b" \t\n\r"
BLOCK, WINDOW = 64, 64 * 32
# phases of a 64-byte block where carries turn: the last two bytes of one block, the first two of the next
EDGES = (62, 63, 64, 65, 127, 128)


@contextlib.contextmanager
def deep_recursion(limit=100_000):
    """bodies_oracle recurses once per container: let it parse the deep families, then restore the limit"""
    old = sys.getrecursionlimit()
    sys.setrecursionlimit(max(old, limit))
    try:
        yield
    finally:
        sys.setrecursionlimit(old)


@functools.lru_cache(maxsize=None)
def real_strings(n=24, seed=77):
    """n (leaf_input, extra_data) base64 strings of synthetic entries (ctmr_synth_raw_pages_host): real certificates"""
    from bodies_pair import synth_bodies
    from ct_mapreduce_b200 import build
    build.build()  # the synthesizer is in libctmr.so, which a CPU-only run may not have built yet
    _, pages = synth_bodies(n, page=n, seed=seed)
    st, ents = bo.parse_body(pages[0], n)
    assert st == bo.BODY_OK and len(ents) == n
    return tuple((e[0].data, e[1].data) for e in ents)


def escape_b64(s: bytes, rng: random.Random, n: int) -> bytes:
    """n escapes at random positions of a base64 string that leave its decode as it was: '/' as '\\/', a character as
    '\\u00XX' (either hex case), '\\r\\n' or '\\n' inserted"""
    out = [bytes([c]) for c in s]
    for _ in range(n):
        k = rng.randrange(len(out) + 1)
        kind = rng.randrange(4)
        if kind == 0 and k < len(out) and out[k] == b"/":
            out[k] = b"\\/"
        elif kind <= 1 and k < len(out) and len(out[k]) == 1:
            out[k] = (b"\\u%04x" if rng.random() < 0.5 else b"\\u%04X") % out[k][0]
        else:
            out.insert(k, rng.choice([b"\\r\\n", b"\\n", b"\\r", b"\\u000a", b"\\u000D"]))
    return b"".join(out)


def phased(items):
    """(body, body_max, phase) -> (body, body_max) with a sacrificial body before each, so that each body starts at its
    phase of a 64-byte block when the bodies are staged back to back from offset 0 (one chunk, packed, or one copy without
    gaps).  The sacrificial body holds an open quote and ends in a dangling backslash, both of which must not carry."""
    out, at = [], 0
    for body, mx, phase in items:
        n = (phase - at) % BLOCK or BLOCK
        out.append((b"\\" if n == 1 else b'"' + b"a" * (n - 2) + b"\\", 0))
        out.append((body, mx))
        at += n + len(body)
    return out


def ws(rng, n):
    return bytes(rng.choice(WS) for _ in range(n))


# ---- 1. escape and string carries ---------------------------------------------------------------------------------------
def carry_bodies(seed=1):
    """backslash runs of 0..130 in a key and in a value whose last backslash falls on EDGES (from the body's block), then
    a quote: the run's parity makes the body OK or BAD_JSON; body starts at every phase; runs filling whole blocks"""
    rng = random.Random(seed)
    items, k = [], 0
    for run in range(131):
        for end in EDGES:
            for where in ("key", "value"):
                phase = k % BLOCK
                k += 1
                head = b'{"' if where == "key" else b'{"x":"'
                tail = b'":1,"entries":[null]}' if where == "key" else b'","entries":[{}]}'
                # the run's last backslash at phase + offset == end (mod 128), after the head and at least one byte
                fill = (end - phase - len(head) - run + 1) % 128
                items.append((head + b"a" * fill + b"\\" * run + tail, 2, phase))
    for phase in range(BLOCK):  # a whole block of backslashes, entered with and without the first byte escaped
        for run in (63, 64, 65, 127, 128, 129):
            for first in (0, 63):  # the run starts on a block's first byte, or one byte before it
                head = b'{"x":"'
                fill = (first - phase - len(head)) % BLOCK
                items.append((head + b"a" * fill + b"\\" * run + b'"}', 1, phase))
    items += [(b, 1, rng.randrange(BLOCK)) for b in (b'"', b"\\", b'""', b'"\\"', b"{}", b"")]
    return phased(items)


def many_starts(seed=2, blocks=40):
    """blocks holding 10 to 20 body starts each: tiny bodies, valid and not, with junk bodies between them"""
    rng = random.Random(seed)
    small = (b"{}", b"null", b"", b"1", b'"', b'"\\', b"\\", b"[]", b'{"a":"\\"}', b' {"entries":[]} ', b"0", b'"x"', b"{", b"}")
    out = []
    for _ in range(blocks):
        left = BLOCK
        for _ in range(rng.randrange(10, 21)):
            b = rng.choice(small)
            if len(b) > left:
                break
            out.append((b, 1))
            left -= len(b)
        out.append((b'"' * (left % 3) + b"\\" * (left - left % 3), 0))  # the rest of the block: junk that would carry
    return out


# ---- 2. warp window edges -------------------------------------------------------------------------------------------------
def lane_edges():
    """offsets of the first and last byte of lanes 0, 1, 30 and 31 of a window and across window boundaries"""
    out = []
    for lane in (0, 1, 30, 31, 32, 33, 63, 64):
        out += [BLOCK * lane, BLOCK * lane + BLOCK - 1]
    return sorted(set(out))


def window_bodies(seed=3):
    """tokens, opening quotes and closing quotes at lane and window edges (bodies at phase 0, and some at other phases)"""
    rng = random.Random(seed)
    items = []
    for T in lane_edges():
        for phase in (0, 1, 63):
            pad = T - phase if T >= phase else T
            w = ws(rng, max(pad, 0))
            items += [
                (w + b'{"entries":[]}', 1, phase),                                   # '{' at T
                (b'{"entries":' + ws(rng, max(pad - 11, 0)) + b"[]}", 1, phase),       # '[' after a run of whitespace
                (b"{" + ws(rng, max(pad - 1, 0)) + b'"entries":[null]}', 1, phase),   # an opening quote
                (b'{"a":"' + b"y" * max(pad - 6, 0) + b'","entries":[]}', 1, phase),  # a closing quote
                (b'{"' + b"k" * max(pad - 2, 0) + b'":[1,{}]}', 1, phase),             # a key's closing quote
                (b'{"a":1' + b"0" * max(pad - 6, 0) + b"}", 1, phase),                  # a scalar ending at T
                (b'{"a":1' + b"0" * max(pad - 6, 0) + b"x}", 1, phase),                 # ... with a bad last byte
            ]
    for k in (1, 2, 3):  # strings of 2048 k + d characters, a backslash or a bad byte in a far lane
        for d in (-64, -63, -1, 0, 1, 63, 64):
            n = WINDOW * k + d
            far = rng.randrange(n // 2, n - 1)
            s = bytearray(b"z" * n)
            items.append((b'{"a":"' + bytes(s) + b'","entries":[]}', 1, 0))
            t = bytearray(s)
            t[far:far + 2] = b"\\/"
            items.append((b'{"a":"' + bytes(t) + b'","entries":[]}', 1, rng.randrange(BLOCK)))
            t = bytearray(s)
            t[far] = rng.choice([0x01, 0x1F, 0x0A, 0x00])
            items.append((b'{"a":"' + bytes(t) + b'","entries":[]}', 1, rng.randrange(BLOCK)))
            t = bytearray(s)
            t[far:far + 2] = b"\\x"
            items.append((b'{"' + bytes(t) + b'":0}', 1, 0))
            items.append((b'{"entries":[]' + ws(rng, n) + b"}", 1, 0))  # whitespace runs of a window and more
    for (l, x), m in zip(real_strings()[:6], (1, 2, 40, 300, 700, 1100)):  # a leaf whose only escapes are in far lanes
        items.append((b'{"entries":[{"leaf_input":"' + l + b"\\n" * m + b'","extra_data":"' + x + b'"}]}', 1, rng.randrange(BLOCK)))
    return phased(items)


def past_end_bodies():
    """a string whose closing quote would be one byte past the body's end: in the next body (back to back).  Each such
    body is followed by a body starting with a quote; run one copy with b'"' gaps for the junk case."""
    out = []
    for n in (0, 1, 57, 58, 62, 63, 64, 121, 2041, 2042, 2048):
        out += [(b'{"entries":[],"a":"' + b"q" * n, 1), (b'"}', 1), (b'{"' + b"k" * n, 1), (b'":1}', 1),
                (b'{"entries":[{"leaf_input":"QUFB' + b"Q" * n, 1), (b'"}]}', 1)]
    return out


# ---- 3. nesting past the register stack -------------------------------------------------------------------------------------
DEPTHS = (62, 63, 64, 65, 66, 95, 96, 127, 128, 1000, 10000)


def deep_member(D, rng, swap_at=None):
    """`{"deep": <containers at depths 2..D>, "entries": [...]}`: kinds in a seeded pattern; swap_at = d swaps the closer of
    the container at depth d (1: the top object) for the other kind's"""
    kinds = [True] + [rng.random() < 0.5 for _ in range(D - 1)]  # depth 1 is the top object
    opens, closes = [], []
    for d in range(2, D + 1):
        obj = kinds[d - 1]
        opens.append(b'{"k%d":' % d if obj else b"[")
        closes.append(b"}" if obj else b"]")
    inner = rng.choice([b"1", b'"s"', b"null", b"true"])
    closes = closes[::-1]  # closes[i] closes depth D - i
    if swap_at is not None and swap_at >= 2:
        i = D - swap_at
        closes[i] = b"]" if closes[i] == b"}" else b"}"
    top_close = b"]" if swap_at == 1 else b"}"
    return b'{"deep":' + b"".join(opens) + inner + b"".join(closes) + b',"entries":[{"leaf_input":"QUFB"},null]' + top_close


def deep_bodies(seed=4):
    """every depth closed correctly (OK, two entries after the deep member), then with one closer swapped at depth 1, 63,
    64, 65 and D (BAD_JSON)"""
    rng = random.Random(seed)
    out = []
    for D in DEPTHS:
        out.append((deep_member(D, random.Random(rng.random())), 2))
        for d in (1, 63, 64, 65, D):
            if d <= D:
                out.append((deep_member(D, random.Random(rng.random()), swap_at=d), 2))
    return out


def deep_expected(D, swap_at=None):
    """what deep_member's body must give, from its construction alone (checked against the oracle)"""
    return (bo.BODY_OK, 2) if swap_at is None else (bo.BODY_BAD_JSON, 0)


# ---- 4. keys --------------------------------------------------------------------------------------------------------------
def _u(c, upper):
    return (b"\\u%04X" if upper else b"\\u%04x") % c


def key_spellings(name: bytes):
    """every byte upper-cased in turn, then every byte as a \\u escape in lower- and upper-case hex"""
    out = []
    for i, c in enumerate(name):
        if 0x61 <= c <= 0x7A:
            out.append(name[:i] + bytes([c - 32]) + name[i + 1:])
        for up in (False, True):
            out.append(name[:i] + _u(c, up) + name[i + 1:])
    return out


NEAR_ENTRIES = [
    "entrieſ".encode(), b"entrie\\u017f", b"entrie\\u017F", b"entrie\\u0053", b"ENTRIE\\u017f",   # match
    "entrieK".encode(), "entrıes".encode(), b"entrie\\u212a", b"entrie\\u0131", b"entries\\u0000", b"entries\x00",
    b"entriesXXXXXX", b"entries_", b"entrie", b"entrie\\ud800", b"entrie\\ud83d\\ude00", b"entrie\\u00c5\\u00bf",
    b"entrie\xc5", b"entri\\u017fs", b"\\u0065ntries", b"ent\\\\ries", b"entr\\/ies",
]
NEAR_NAMES = [
    b"leaf\\u005finput", b"leaf\\u005Finput", b"leaf\\u002dinput", b"leaf-input", b"leafinput", b"leaf_input\\u0000",
    b"leaf_inpuT", b"LEAF_INPUT", b"leaf_inputX", b"leaf_inpu", b"leaf_\\u0131nput", "leaf_ınput".encode(), b"leaf_input ",
    b"extra\\u005Fdata", b"extra\\u002ddata", b"EXTRA_DATA", b"extra_dat\\u0061", b"extra_data\\ud800", b"extra_dataa",
]


def key_bodies(seed=5):
    """each spelling of "entries", "leaf_input" and "extra_data", and near misses, at phase 0, across a block edge and
    across a window edge; keys at depth 1 of a non-object top level and at depth 3 outside an element"""
    rng = random.Random(seed)
    (l0, x0), (l1, x1) = real_strings()[:2]
    keys = [(k, None) for k in key_spellings(b"entries") + NEAR_ENTRIES]
    keys += [(None, k) for k in key_spellings(b"leaf_input") + key_spellings(b"extra_data") + NEAR_NAMES]
    items = []
    for ek, nk in keys:
        for edge in (None, BLOCK, WINDOW, 2 * WINDOW):
            k = ek if ek is not None else nk
            if ek is not None:
                head = b"{"
                body_after = b'":[{"leaf_input":"' + l0 + b'","extra_data":"' + x0 + b'"}]}'
            else:
                head = b'{"entries":[{"extra_data":"' + x1 + b'",'
                body_after = b'":"' + l1 + b'"}]}'
            pad = b""
            if edge is not None:  # the key's middle byte on the edge: the key straddles it
                pad = ws(rng, max(0, edge - len(head) - 1 - len(k) // 2))
            items.append((head + pad + b'"' + k + body_after, 2, 0))
    items += [(b'[{"entries":[{"leaf_input":"' + l0 + b'"}]}]', 1, 3), (b'[1,{"entries":[]}]', 1, 5),
              (b'{"x":{"y":{"leaf_input":"' + l0 + b'","extra_data":7}},"entries":[{"z":{"leaf_input":1}}]}', 1, 7),
              (b'{"x":[{"leaf_input":"' + l0 + b'"}],"entries":[{"a":[{"extra_data":{}}]}]}', 1, 9)]
    return phased(items)


# ---- 5. scalars -------------------------------------------------------------------------------------------------------------
SCALARS = [b"0", b"-0", b"0e1", b"1E+2", b"-0.5e-3", b"1e400", b"123456789012345678901234567890", b"0.0", b"true", b"false",
           b"null", b"1e-0", b"9E09",
           b"01", b"1.", b"-", b".5", b"tru", b"nulll", b"+1", b"1e", b"1e+", b"--1", b"0x1", b"NaN", b"Infinity", b"1.5.",
           b"falsee", b"nul", b"-01", b"00", b"1E", b".", b"e1", b"TRUE", b"Null", b"1-", b"0.e1", b"-.5", b"1e1.5", b"\x7f"]
DELIMS = b",]} \t\n\r\":{["


def scalar_bodies():
    """each scalar as a member's value, the top level, an element and leaf_input, and directly before each delimiter"""
    out = []
    for s in SCALARS:
        out += [(b'{"a":' + s + b',"entries":[]}', 1), (s, 1), (b'{"entries":[' + s + b"]}", 1),
                (b'{"entries":[{"leaf_input":' + s + b"}]}", 1), (b'{"entries":[{"extra_data":' + s + b"}]}", 1),
                (b"[" + s + b"]", 1), (b"{\"a\":[" + s + b"," + s + b"]}", 1)]
        for c in DELIMS:
            out += [(b'{"a":[' + s + bytes([c]) + b"]}", 1), (b'{"a":' + s + bytes([c]) + b"}", 1),
                    (b"[" + s + bytes([c]) + b"1]", 1)]
    return out


ABUTTING = [(b"1", b"e"), (b"-", b"1"), (b"1.", b"5"), (b"0", b"1"), (b"tru", b"e"), (b"nul", b"l"), (b"1e", b"5"), (b"12", b"x"),
            (b"true", b"1"), (b"null", b"l"), (b'{"a":1', b"2}"), (b'{"a":[0', b".5]}")]


def abutting_scalars():
    """a scalar at the very end of a body with the next body's digits right after it: the scan stops at the body's end"""
    out = []
    for a, b in ABUTTING:
        out += [(a, 1), (b, 1)]
    return out


# ---- 6. \u escapes and unescape ---------------------------------------------------------------------------------------------
def u_escape_bodies(seed=6):
    """'\\u' with 0..4 hex digits (then a quote or a non-hex byte), the backslash at block phases 59..64, and just before
    the body's end"""
    rng = random.Random(seed)
    items = []
    for nd in range(5):
        for at in range(59, 65 + 1):
            for after in (b'"', b"g", b"}", b"0"):
                digits = bytes(rng.choice(b"0123456789abcdefABCDEF") for _ in range(nd))
                head = b'{"a":"'
                items.append((head + b"b" * (at - len(head)) + b"\\u" + digits + after + b'","entries":[]}', 1, 0))
                items.append((b'{"' + b"c" * (at - 2) + b"\\u" + digits + after + b'":[]}', 1, 0))
        items.append((b'{"a":"\\u' + b"1" * nd, 1, rng.randrange(BLOCK)))
        items.append((b'1' * nd + b'"}', 1, rng.randrange(BLOCK)))  # the next body: the digits a scan past the end reads
    return phased(items)


def unescape_bodies(seed=7, n=48):
    """bodies of real entries whose strings went through escape_b64, at random phases"""
    rng = random.Random(seed)
    reals = real_strings()
    items = []
    for _ in range(n):
        ents = []
        for _ in range(rng.randrange(1, 4)):
            l, x = rng.choice(reals)
            l = escape_b64(l, rng, rng.randrange(0, 12))
            x = escape_b64(x, rng, rng.randrange(0, 12))
            ents.append(b'{"leaf_input":"' + l + b'","extra_data":"' + x + b'"}')
        items.append((b'{"entries":[' + b",".join(ents) + b"]}", 4, rng.randrange(BLOCK)))
    return phased(items)


# ---- 7. one body over many scan tiles -----------------------------------------------------------------------------------------
def long_string_body(nbytes, odd, seed=8):
    """a body of about nbytes whose one long string holds a seeded mix of '\\\\' and '\\"' pairs and letters: its validity
    depends on both carries through every block.  odd: the last backslash run made odd, which escapes the closing quote"""
    rng = random.Random(seed)
    (l0, x0), = real_strings()[:1]
    units = (b"\\\\", b'\\"', b"a", b"\\\\\\\\")
    parts, n = [], 0
    while n < nbytes:
        u = rng.choice(units)
        parts.append(u)
        n += len(u)
    s = b"".join(parts) + b"\\\\" + (b"\\" if odd else b"")
    return b'{"pad":"' + s + b'","entries":[{"leaf_input":"' + l0 + b'","extra_data":"' + x0 + b'"}]}'


# ---- 9. grammar fuzz ----------------------------------------------------------------------------------------------------------
class _Ser:
    def __init__(self, rng):
        self.rng = rng

    def ws(self):
        r = self.rng.random()
        if r < 0.7:
            return b""
        if r < 0.995:
            return ws(self.rng, self.rng.randrange(1, 5))
        return ws(self.rng, self.rng.randrange(2049, 4200))  # longer than a window

    def key(self, name: bytes):
        rng, out = self.rng, []
        for c in name:
            r = rng.random()
            if c == 0x73 and name == b"entries" and r < 0.08:
                out.append(rng.choice(["ſ".encode(), b"\\u017f", b"\\u017F"]))
            elif r < 0.12:
                out.append(_u(c, rng.random() < 0.5))
            elif r < 0.3 and 0x61 <= c <= 0x7A:
                out.append(bytes([c - 32]))
            else:
                out.append(bytes([c]))
        return b"".join(out)

    def string(self):
        rng = self.rng
        parts = []
        for _ in range(rng.randrange(0, 12)):
            r = rng.random()
            if r < 0.5:
                parts.append(bytes(rng.choice(b"abcXYZ019 +/=") for _ in range(rng.randrange(1, 8))))
            elif r < 0.8:
                parts.append(rng.choice([b'\\"', b"\\\\", b"\\/", b"\\b", b"\\f", b"\\n", b"\\r", b"\\t"]))
            elif r < 0.9:
                parts.append(_u(rng.randrange(0x10000), rng.random() < 0.5))
            else:
                parts.append(rng.choice(["é".encode(), "ſ".encode(), b"\xff", b"{}[],:"]))
        return b'"' + b"".join(parts) + b'"'

    def value(self, depth=0):
        rng = self.rng
        r = rng.random()
        if depth > 6 or r < 0.35:
            return rng.choice([b"null", b"true", b"false", b"0", b"-1.5e3", b"12", b"0.25", b"-0", b"1E+9"])
        if r < 0.6:
            return self.string()
        if r < 0.8:
            return b"[" + b",".join(self.ws() + self.value(depth + 1) + self.ws() for _ in range(rng.randrange(0, 4))) + b"]"
        return self.obj([(self.key(rng.choice([b"a", b"leaf_input", b"extra_data", b"entries", b"zz"])), self.value(depth + 1))
                         for _ in range(rng.randrange(0, 4))])

    def obj(self, members):
        if not members:
            return b"{" + self.ws() + b"}"
        return b"{" + b",".join(self.ws() + b'"' + k + b'"' + self.ws() + b":" + self.ws() + v + self.ws() for k, v in members) + b"}"


def build_body(rng, reals, max_entries=4):
    """a GetEntriesResponse-shaped document with random spellings, whitespace, unknown members, nulls, repeated and
    missing keys, and now and then a member of the wrong type"""
    s = _Ser(rng)
    elems = []
    for _ in range(rng.randrange(0, max_entries + 1)):
        r = rng.random()
        if r < 0.08:
            elems.append(b"null")
            continue
        if r < 0.1:
            elems.append(rng.choice([b"1", b"[]", b'"x"']))  # the wrong type
            continue
        l, x = rng.choice(reals)
        if rng.random() < 0.3:
            l, x = escape_b64(l, rng, rng.randrange(1, 6)), escape_b64(x, rng, rng.randrange(0, 6))
        members = []
        if rng.random() < 0.95:
            members.append((s.key(b"leaf_input"), b'"' + l + b'"' if rng.random() < 0.95 else b"null"))
        if rng.random() < 0.9:
            members.append((s.key(b"extra_data"), b'"' + x + b'"' if rng.random() < 0.95 else rng.choice([b"null", b"{}"])))
        if rng.random() < 0.1:
            members.append((s.key(rng.choice([b"leaf_input", b"extra_data"])), rng.choice([b'"QUFB"', b"null"])))  # repeated
        for _ in range(rng.randrange(0, 3)):
            members.insert(rng.randrange(len(members) + 1), (s.key(rng.choice([b"y", b"Leaf", b"leaf_inputs"])), s.value()))
        elems.append(s.obj(members))
    arr = b"[" + b",".join(s.ws() + e + s.ws() for e in elems) + b"]" if rng.random() < 0.97 else b"null"
    members = [(s.key(b"entries"), arr)]
    for _ in range(rng.randrange(0, 3)):
        members.insert(rng.randrange(len(members) + 1), (s.key(rng.choice([b"more", b"x", b"Entrie"])), s.value()))
    if rng.random() < 0.06:
        members.append((s.key(b"entries"), rng.choice([b"[]", b"null", b"[{}]"])))  # a second entries member
    body = s.ws() + s.obj(members) + s.ws()
    return body, len(elems)


def mutate(body: bytes, rng: random.Random) -> bytes:
    """one of: delete, insert or replace a byte; swap a closer; truncate; a control byte in a string; one backslash more
    or less in a run; a second entries member"""
    b = bytearray(body)
    kind = rng.randrange(8)
    if not b:
        return b"{"
    i = rng.randrange(len(b))
    if kind == 0:
        del b[i]
    elif kind == 1:
        b.insert(i, rng.choice(b'{}[],:"\\ ax0\x01'))
    elif kind == 2:
        b[i] = rng.randrange(256)
    elif kind == 3:
        cl = [k for k, c in enumerate(b) if c in b"}]"]
        if cl:
            k = rng.choice(cl)
            b[k] = 0x5D if b[k] == 0x7D else 0x7D
    elif kind == 4:
        del b[i:]
    elif kind == 5:
        qs = [k for k, c in enumerate(b) if c == 0x22]
        if qs:
            b.insert(rng.choice(qs) + 1, rng.randrange(0x20))
    elif kind == 6:
        bs = [k for k, c in enumerate(b) if c == 0x5C]
        if bs:
            k = rng.choice(bs)
            if rng.random() < 0.5:
                del b[k]
            else:
                b.insert(k, 0x5C)
    else:
        k = b.rfind(b"}")
        if k >= 0:
            b[k:k] = b',"entries":[]'
    return bytes(b)


def fuzz_bodies(seed=9, n=1000):
    """n bodies, about a third of them mutated once or twice; body_max at, above and below the element count"""
    rng = random.Random(seed)
    reals = real_strings()
    out = []
    while len(out) < n:
        body, cnt = build_body(rng, reals, max_entries=rng.choice([0, 1, 2, 3, 4]))
        if len(body) > 20000:
            continue
        if rng.random() < 0.35:
            for _ in range(rng.randrange(1, 3)):
                body = mutate(body, rng)
        mx = max(0, cnt + rng.choice([0, 0, 0, 1, 3, -1]))
        out.append((body, mx))
    return out
