"""Restatement of how ct-go's jsonclient finds the entries of a get-entries response body: Go 1.13 encoding/json
Unmarshal into GetEntriesResponse{Entries []LeafEntry `json:"entries"`}, LeafEntry{LeafInput, ExtraData []byte}
(reference cmd/ct-fetch/ct-fetch.go:424), which runs checkValid over the whole body first.  Written byte by byte from
those rules, not with Python's json (which accepts NaN, a BOM after decoding, and handles duplicates its own way).

`parse_body(body, body_max)` -> (status, entries): status is one of the BODY_* codes of include/ctmr_frontend.h; entries
(OK bodies only) are (leaf_input, extra_data) pairs of Str, or None for a missing or null string.  Str.data is what the
decode sees: the characters as they are, or for a string with escapes its unescaped text with '\\r' and '\\n' dropped
(base64.StdEncoding skips them) and every non-ASCII byte made '!' (outside the alphabet: BAD_BASE64 either way).
"""
from __future__ import annotations

import re
from typing import NamedTuple

BODY_OK, BODY_BAD_JSON, BODY_BAD_TYPE, BODY_TOO_MANY, BODY_REPEATED_ENTRIES = range(5)

_WS = b" \t\n\r"
_DELIM = set(b" \t\n\r\"{}[]:,")
_NUMBER = re.compile(rb"-?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?\Z")
_HEX = set(b"0123456789abcdefABCDEF")


class Str(NamedTuple):
    off: int        # first character, relative to the body
    len: int        # characters as found, escapes included
    escaped: bool
    data: bytes     # what the base64 decode reads


class _Bad(Exception):
    pass


def _ws(b, i):
    while i < len(b) and b[i] in _WS:
        i += 1
    return i


def _string(b, i):
    """b[i] is the opening quote -> (index after the closing quote, unescaped UTF-8 bytes, had a backslash)"""
    j, out, esc = i + 1, bytearray(), False
    while True:
        if j >= len(b):
            raise _Bad
        c = b[j]
        if c == 0x22:
            return j + 1, bytes(out), esc
        if c < 0x20:
            raise _Bad
        if c != 0x5C:
            out.append(c)
            j += 1
            continue
        esc = True
        if j + 1 >= len(b):
            raise _Bad
        d = b[j + 1]
        if d in b'"\\/':
            out.append(d)
            j += 2
        elif d in b"bfnrt":
            out.append({0x62: 8, 0x66: 12, 0x6E: 10, 0x72: 13, 0x74: 9}[d])
            j += 2
        elif d == 0x75:
            h = b[j + 2:j + 6]
            if len(h) < 4 or any(x not in _HEX for x in h):
                raise _Bad
            v = int(h, 16)
            j += 6
            if 0xD800 <= v < 0xDC00 and b[j:j + 2] == b"\\u" and len(b[j + 2:j + 6]) == 4 and all(x in _HEX for x in b[j + 2:j + 6]) \
                    and 0xDC00 <= int(b[j + 2:j + 6], 16) < 0xE000:
                v = 0x10000 + ((v - 0xD800) << 10) + (int(b[j + 2:j + 6], 16) - 0xDC00)
                j += 6
            elif 0xD800 <= v < 0xE000:
                v = 0xFFFD
            out += chr(v).encode("utf-8")
        else:
            raise _Bad


def is_entries(k: bytes) -> bool:
    """encoding/json's equalFoldRight against "entries": ASCII letters fold, 's' also matches U+017F"""
    j = 0
    for sb in b"entries":
        if j >= len(k):
            return False
        tb = k[j]
        if tb < 0x80:
            if tb & 0xDF != sb & 0xDF:
                return False
            j += 1
        elif sb == 0x73 and k[j:j + 2] == b"\xc5\xbf":
            j += 2
        else:
            return False
    return j == len(k)


def is_name(k: bytes, name: bytes) -> bool:
    """encoding/json's asciiEqualFold: letters case-insensitively, every other byte exactly"""
    if len(k) != len(name):
        return False
    for sb, tb in zip(name, k):
        if sb != tb and not (0x61 <= sb <= 0x7A and sb & 0xDF == tb & 0xDF):
            return False
    return True


def _b64_text(raw: bytes, unescaped: bytes, esc: bool) -> bytes:
    if not esc:
        return raw
    return bytes(0x21 if c >= 0x80 else c for c in unescaped if c not in (10, 13))


class _Walk:
    def __init__(self, b, body_max):
        self.b, self.max = b, body_max
        self.bad_type = False
        self.entries_seen = 0
        self.count = 0
        self.entries = []

    def value(self, i, role, elem=None):
        """role: top, entries, elem, leaf, extra, skip; elem: the element a leaf / extra string belongs to"""
        b = self.b
        i = _ws(b, i)
        if i >= len(b):
            raise _Bad
        c = b[i]
        if c == 0x7B:  # {
            cur = None
            if role == "top":
                pass
            elif role == "elem":
                cur = [None, None]
            elif role != "skip":
                self.bad_type = True
            i = _ws(b, i + 1)
            if i < len(b) and b[i] == 0x7D:
                i += 1
            else:
                while True:
                    i = _ws(b, i)
                    if i >= len(b) or b[i] != 0x22:
                        raise _Bad
                    i, key, _ = _string(b, i)
                    i = _ws(b, i)
                    if i >= len(b) or b[i] != 0x3A:
                        raise _Bad
                    mrole = "skip"
                    if role == "top" and is_entries(key):
                        self.entries_seen += 1
                        mrole = "entries"
                    elif cur is not None and is_name(key, b"leaf_input"):
                        mrole = "leaf"
                    elif cur is not None and is_name(key, b"extra_data"):
                        mrole = "extra"
                    i = self.value(i + 1, mrole, cur)
                    i = _ws(b, i)
                    if i < len(b) and b[i] == 0x2C:
                        i += 1
                        continue
                    if i < len(b) and b[i] == 0x7D:
                        i += 1
                        break
                    raise _Bad
            if cur is not None:
                self.emit(cur)
            return i
        if c == 0x5B:  # [
            if role not in ("entries", "skip"):
                self.bad_type = True
            er = "elem" if role == "entries" else "skip"
            i = _ws(b, i + 1)
            if i < len(b) and b[i] == 0x5D:
                return i + 1
            while True:
                i = self.value(i, er)
                i = _ws(b, i)
                if i < len(b) and b[i] == 0x2C:
                    i += 1
                    continue
                if i < len(b) and b[i] == 0x5D:
                    return i + 1
                raise _Bad
        if c == 0x22:
            end, text, esc = _string(b, i)
            if role in ("leaf", "extra"):
                raw = b[i + 1:end - 1]
                elem[role == "extra"] = Str(i + 1, len(raw), esc, _b64_text(raw, text, esc))
            elif role != "skip":
                self.bad_type = True
            return end
        j = i
        while j < len(b) and b[j] not in _DELIM:
            j += 1
        tok = b[i:j]
        if tok == b"null":
            if role == "elem":
                self.emit([None, None])
            elif role in ("leaf", "extra"):
                elem[role == "extra"] = None
            return j
        if not (tok in (b"true", b"false") or _NUMBER.match(tok)):
            raise _Bad
        if role != "skip":
            self.bad_type = True
        return j

    def emit(self, cur):
        if self.entries_seen != 1:
            return
        if self.count < self.max:
            self.entries.append((cur[0], cur[1]))
        self.count += 1


def parse_body(body: bytes, body_max: int):
    w = _Walk(bytes(body), body_max)
    try:
        i = w.value(0, "top")
        if _ws(w.b, i) != len(w.b):
            raise _Bad
    except _Bad:
        return BODY_BAD_JSON, []
    if w.bad_type:
        return BODY_BAD_TYPE, []
    if w.entries_seen > 1:
        return BODY_REPEATED_ENTRIES, []
    if w.count > body_max:
        return BODY_TOO_MANY, []
    return BODY_OK, w.entries


def go_scanner_spans(body: bytes):
    """`RawPages.AppendLog` (go/ctmr/frontend.go) restated: the exact keys '"leaf_input":"' / '"extra_data":"', the
    closing quote, strings paired by order of occurrence; an error when the counts differ or a string holds a backslash."""
    def spans(key):
        out, at = [], 0
        while True:
            k = body.find(key, at)
            if k < 0:
                return out
            s = k + len(key)
            e = body.index(b'"', s)
            if b"\\" in body[s:e]:
                raise ValueError("escaped base64 string")
            out.append((s, e - s))
            at = e
    li, ex = spans(b'"leaf_input":"'), spans(b'"extra_data":"')
    if len(li) != len(ex):
        raise ValueError("leaf_input and extra_data counts differ")
    return list(zip(li, ex))


def twin_batch(bodies, maxes):
    """What ctmr_process_raw is given for the same bodies: the spans the oracle finds, in (body, position) order, with
    escaped strings replaced by their unescaped text (appended after the bodies).  Returns (text, leaf_off, leaf_len,
    extra_off, extra_len, statuses, counts)."""
    text = bytearray(b"".join(bodies))
    base, lo, ll, xo, xl, sts, cnts = 0, [], [], [], [], [], []
    for body, mx in zip(bodies, maxes):
        st, ents = parse_body(body, mx)
        sts.append(st)
        cnts.append(len(ents))
        for pair in ents:
            for s, (offs, lens) in zip(pair, ((lo, ll), (xo, xl))):
                if s is None:
                    offs.append(0)
                    lens.append(0)
                elif s.escaped:
                    offs.append(len(text))
                    lens.append(len(s.data))
                    text += s.data
                else:
                    offs.append(base + s.off)
                    lens.append(s.len)
        base += len(body)
    return bytes(text), lo, ll, xo, xl, sts, cnts
