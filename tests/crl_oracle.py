"""ctmr_revoked_known's rules restated byte by byte (include/ctmr.h, RFC 5280 §5.1), and the join against the sets a
test created.

`parse_crl(der)` returns the CRL's status, fields and entries as the GPU must report them.  `join(parsed, digest, sets)`
answers each entry from `sets`: {(hour, issuer digest): set of raw serials}, the serials:: sets the test put in the
table (read back from oracle.DB / the preloads).  TLV headers follow Go's encoding/asn1 as the certificate walker does
(single-octet tags, minimal definite lengths of at most 4 octets); Time is UTCTime (pivot 50, seconds optional) or
GeneralizedTime, with Z or a non-zero +-hhmm offset.
"""
from __future__ import annotations

CRL_OK, CRL_BAD, CRL_BAD_ENTRIES, CRL_UNKNOWN_ISSUER = range(4)
RV_OK, RV_INDIRECT, RV_SERIAL_TOO_LONG = range(3)
MAX_SERIAL = 39
INT64_MIN = -(1 << 63)


class Bad(Exception):
    pass


def read(d: bytes, pos: int, end: int):
    """(tag, header length, content length) of the TLV at pos, inside [pos, end)."""
    if pos + 2 > end:
        raise Bad("short")
    tag, l = d[pos], d[pos + 1]
    if tag & 0x1F == 0x1F:
        raise Bad("multi-octet tag")
    if l < 0x80:
        h, n = 2, l
    else:
        nb = l & 0x7F
        if nb == 0 or nb > 4 or pos + 2 + nb > end:
            raise Bad("length")
        v = 0
        for i in range(nb):
            if v >= 1 << 23:
                raise Bad("length")
            v = (v << 8) | d[pos + 2 + i]
            if v == 0:
                raise Bad("non-minimal length")
        if v < 0x80:
            raise Bad("non-minimal length")
        h, n = 2 + nb, v
    if n > end - pos - h:
        raise Bad("overrun")
    return tag, h, n


def _2d(b: bytes) -> int:
    if not (48 <= b[0] <= 57 and 48 <= b[1] <= 57):
        raise Bad("digit")
    return (b[0] - 48) * 10 + b[1] - 48


def parse_time(tag: int, p: bytes) -> int:
    n = len(p)
    if tag == 0x18:
        if n < 15:
            raise Bad("time")
        year, pos = _2d(p[0:2]) * 100 + _2d(p[2:4]), 4
    elif tag == 0x17:
        if n < 11:
            raise Bad("time")
        yy = _2d(p[0:2])
        year, pos = (1900 + yy if yy >= 50 else 2000 + yy), 2
    else:
        raise Bad("time tag")
    mo, dd, hh, mi = (_2d(p[pos + 2 * i:pos + 2 * i + 2]) for i in range(4))
    pos += 8
    ss, has_sec = 0, False
    if pos + 2 <= n and 48 <= p[pos] <= 57:
        ss, has_sec = _2d(p[pos:pos + 2]), True
        pos += 2
    if tag == 0x18 and not has_sec or pos >= n:
        raise Bad("time")
    off = 0
    if p[pos] == ord("Z"):
        if pos + 1 != n:
            raise Bad("time")
    elif p[pos] in b"+-":
        if pos + 5 != n:
            raise Bad("time")
        oh, om = _2d(p[pos + 1:pos + 3]), _2d(p[pos + 3:pos + 5])
        if oh > 23 or om > 59:
            raise Bad("time")
        off = oh * 3600 + om * 60
        if off == 0:
            raise Bad("zero offset")
        if p[pos] == ord("-"):
            off = -off
    else:
        raise Bad("time")
    if not (1 <= mo <= 12 and dd >= 1 and hh <= 23 and mi <= 59 and ss <= 59):
        raise Bad("time")
    maxd = 28 if mo == 2 else (31 if (0xAD5 >> (mo - 1)) & 1 else 30)
    if mo == 2 and year % 4 == 0 and (year % 100 != 0 or year % 400 == 0):
        maxd = 29
    if dd > maxd:
        raise Bad("day")
    days = _days(year, mo, dd)
    return days * 86400 + hh * 3600 + mi * 60 + ss - off


def _days(y: int, m: int, d: int) -> int:
    y -= m <= 2
    era = (y if y >= 0 else y - 399) // 400
    yoe = y - era * 400
    doy = (153 * (m - 3 if m > 2 else m + 9) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def _name(d: bytes, pos: int, end: int):
    while pos < end:
        tag, h, n = read(d, pos, end)
        if tag != 0x31:
            raise Bad("rdn")
        sp, se = pos + h, pos + h + n
        while sp < se:
            t, ah, an = read(d, sp, se)
            if t != 0x30:
                raise Bad("atv")
            ap, ae = sp + ah, sp + ah + an
            t, oh, on = read(d, ap, ae)
            if t != 0x06:
                raise Bad("oid")
            read(d, ap + oh + on, ae)
            sp += ah + an
        pos += h + n


def _extensions(d: bytes, pos: int, end: int):
    """[(oid content, value content)] of an Extensions SEQUENCE filling [pos, end) exactly."""
    tag, h, n = read(d, pos, end)
    if tag != 0x30 or pos + h + n != end:
        raise Bad("extensions")
    out, ep = [], pos + h
    while ep < end:
        tag, h, n = read(d, ep, end)
        if tag != 0x30:
            raise Bad("extension")
        ip, ie = ep + h, ep + h + n
        tag, oh, on = read(d, ip, ie)
        if tag != 0x06:
            raise Bad("oid")
        oid = d[ip + oh:ip + oh + on]
        ip += oh + on
        tag, vh, vn = read(d, ip, ie)
        if tag == 0x01:
            if vn != 1 or d[ip + vh] not in (0, 0xFF):
                raise Bad("critical")
            ip += vh + vn
            tag, vh, vn = read(d, ip, ie)
        if tag != 0x04 or ip + vh + vn != ie:
            raise Bad("extnValue")
        out.append((oid, d[ip + vh:ip + vh + vn]))
        ep = ie
    return out


def parse_entry(d: bytes, p: int, end: int) -> dict:
    tag, h, n = read(d, p, end)
    if tag != 0x30 or p + h + n != end:
        raise Bad("entry")
    q = p + h
    tag, ih, il = read(d, q, end)
    if tag != 0x02 or il == 0:
        raise Bad("serial")
    e = {"serial_pos": q + ih, "serial": d[q + ih:q + ih + il], "reason": 0xFF, "indirect": False}
    q += ih + il
    tag, th, tn = read(d, q, end)
    e["revoked_at"] = parse_time(tag, d[q + th:q + th + tn])
    q += th + tn
    if q != end:
        tag, xh, xn = read(d, q, end)
        if tag != 0x30 or q + xh + xn != end:
            raise Bad("entry extensions")
        for oid, val in _extensions(d, q, end):
            if oid == b"\x55\x1d\x15":
                if len(val) != 3 or val[0] != 0x0A or val[1] != 1:
                    raise Bad("reasonCode")
                e["reason"] = val[2]
            elif oid == b"\x55\x1d\x1d":
                e["indirect"] = True
    e["status"] = RV_INDIRECT if e["indirect"] else RV_SERIAL_TOO_LONG if len(e["serial"]) > MAX_SERIAL else RV_OK
    return e


def parse_crl(d: bytes) -> dict:
    """Status, fields and entries (offsets relative to d) of one DER CRL."""
    r = {"status": CRL_BAD, "flags": 0, "this_update": 0, "next_update": INT64_MIN, "entries": []}
    try:
        L = len(d)
        tag, h, n = read(d, 0, L)
        if tag != 0x30 or h + n != L:
            raise Bad("outer")
        pos = h
        tag, th, tn = read(d, pos, L)
        if tag != 0x30:
            raise Bad("tbs")
        r["tbs"] = (pos, th + tn)
        tp, tend = pos + th, pos + th + tn
        tag, h, n = read(d, tp, tend)
        if tag == 0x02:
            if n != 1 or d[tp + h] != 1:
                raise Bad("version")
            tp += h + n
            tag, h, n = read(d, tp, tend)
        if tag != 0x30:
            raise Bad("sigalg")
        tp += h + n
        tag, h, n = read(d, tp, tend)
        if tag != 0x30:
            raise Bad("issuer")
        r["name"] = (tp, h + n)
        _name(d, tp + h, tp + h + n)
        tp += h + n
        tag, h, n = read(d, tp, tend)
        r["this_update"] = parse_time(tag, d[tp + h:tp + h + n])
        tp += h + n
        content = None
        if tp < tend:
            tag, h, n = read(d, tp, tend)
            if tag in (0x17, 0x18):
                r["next_update"] = parse_time(tag, d[tp + h:tp + h + n])
                tp += h + n
                if tp < tend:
                    tag, h, n = read(d, tp, tend)
        if tp < tend and tag == 0x30:
            content = (tp + h, tp + h + n)
            tp += h + n
            if tp < tend:
                tag, h, n = read(d, tp, tend)
        if tp < tend and tag == 0xA0:
            for oid, _ in _extensions(d, tp + h, tp + h + n):
                if oid == b"\x55\x1d\x1b":
                    r["flags"] |= 1
                if oid == b"\x55\x1d\x1c":
                    r["flags"] |= 2
            tp += h + n
        if tp != tend:
            raise Bad("tbs tail")
        sp = tend
        tag, h, n = read(d, sp, L)
        if tag != 0x30:
            raise Bad("sigalg")
        sp += h + n
        tag, h, n = read(d, sp, L)
        if tag != 0x03 or n == 0 or sp + h + n != L:
            raise Bad("signature")
    except (Bad, IndexError):
        r["flags"] = 0
        return r
    r["status"] = CRL_OK
    r["content"] = content  # the revokedCertificates content span, None when absent
    if content:  # the serial walk the GPU's split must agree with
        p, ce = content
        try:
            while p < ce:
                tag, h, n = read(d, p, ce)
                r["entries"].append(parse_entry(d, p, p + h + n))
                p += h + n
        except (Bad, IndexError):
            r["status"], r["entries"] = CRL_BAD_ENTRIES, []
    return r


def join(parsed: dict, digest: bytes, sets: dict, registered: set) -> dict:
    """The CRL's status once its issuer is looked up, and per entry (known, lowest hour, sets)."""
    st = parsed["status"]
    if st == CRL_OK and digest not in registered:
        st = CRL_UNKNOWN_ISSUER
    ans = []
    for e in parsed["entries"]:
        hours = []
        if st == CRL_OK and e["status"] == RV_OK:
            hours = [h for (h, dg), ss in sets.items() if dg == digest and e["serial"] in ss]
        ans.append((1 if hours else 0, min(hours) if hours else 0, len(hours)))
    return {"status": st, "answers": ans}
