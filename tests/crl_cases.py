"""A catalogue of named CRLs for ctmr_revoked_known, each with the outcome include/ctmr.h's rules give it, written here by
hand (never taken from crl_oracle, so that the oracle is checked too), and seeded mutants whose outcome the oracle gives.

`catalogue()` returns [Case]: the DER, the CRL status, the per-entry CTMR_RV_* of a CRL that lists entries, and the
fields a case is about (times in Unix seconds from calendar.timegm, reasons, flags, serial lengths).  The families:

  header_*   every TLV header level of the CRL (outer, TBS, Name, RDN, ATV, OID, each Time, revokedCertificates, entry,
             INTEGER, entry extensions, one extension, OCTET STRING, [0], signatureAlgorithm, BIT STRING) with a
             multi-octet tag, the indefinite length, non-minimal lengths, five length octets and a length one past its
             parent; and with the minimal long forms 81 80, 82 01 00 and 83 01 00 00
  tbs_*      version, signature, Name, nextUpdate, revokedCertificates, [0] and trailing-byte rules
  time_*     UTCTime / GeneralizedTime rules in thisUpdate, nextUpdate and revocationDate
  entry_*    serial lengths (0 to 300 octets), entry tails, reasonCode, critical flags, certificateIssuer, OIDs
  crlext_*   deltaCRLIndicator / issuingDistributionPoint flags and the Extensions rules inside [0]
  split_*    false `30 L 02` candidates landing on a later entry, on the content end and past it; entries and CRL
             boundaries at every phase mod 16; chains of 2^k - 1, 2^k and 2^k + 1 minimal entries; tails of 30 01 02;
             CRLs of 0 and 1 bytes

Nothing here parses: a header level is named in the tree a CRL is serialised from, and a case changes that one node.
"""
from __future__ import annotations

import calendar
import functools
import random
from dataclasses import dataclass, field

import crl_oracle as co
from crl_build import CERT_ISSUER_OID, CRL_NUMBER_OID, DELTA_OID, IDP_OID, REASON_OID
from der_build import hdr, long_oid

OK, BAD, BADE = co.CRL_OK, co.CRL_BAD, co.CRL_BAD_ENTRIES
RV, IND, LONG = co.RV_OK, co.RV_INDIRECT, co.RV_SERIAL_TOO_LONG
UTC, GEN = 0x17, 0x18
SHA_OID = b"\x2a\x86\x48\x86\xf7\x0d\x01\x01\x0b"
CN_OID = b"\x55\x04\x03"
UNKNOWN_OID = b"\x2b\x06\x01\x04\x01\x82\x37\x15\x01"  # 1.3.6.1.4.1.311.21.1: not one the parser reads


def T(y, mo, d, h=0, mi=0, s=0) -> int:
    return calendar.timegm((y, mo, d, h, mi, s))


@dataclass
class Case:
    name: str
    der: bytes
    status: int
    entries: list | None = None   # CTMR_RV_* per entry of an OK CRL
    fields: dict = field(default_factory=dict)


# ------------------------------------------------------------------------------------------------ the CRL tree

class N:
    """A TLV node: tag, children (N or raw bytes), and an optional name a case may address."""

    def __init__(self, tag: int, *kids, name: str | None = None):
        self.tag, self.kids, self.name = tag, kids, name


def _head(tag: int, n: int, mod: str | None, following: int) -> bytes:
    if mod is None:
        return hdr(tag, n)
    if mod == "tag1f":          # low five bits set: a multi-octet tag
        return bytes([tag | 0x1F]) + hdr(tag, n)[1:]
    if mod == "indef":          # 80: the indefinite length
        return bytes([tag, 0x80])
    if mod == "81":             # 81 05: one length octet below 80
        return bytes([tag, 0x81, n if n < 0x80 else 0x05])
    if mod == "8200":           # 82 00 90: a leading zero octet
        ln = n.to_bytes(max(1, (n.bit_length() + 7) // 8), "big")
        return bytes([tag, 0x81 + len(ln), 0]) + ln
    if mod == "85":             # five length octets
        return bytes([tag, 0x85]) + n.to_bytes(5, "big")
    if mod == "past":           # the length runs one byte past the parent's end
        return hdr(tag, n + following + 1)
    raise ValueError(mod)


def ser(node, ctx: dict, following: int = 0) -> bytes:
    """DER of the tree.  ctx: mods {name: header mod}, repl {name: node}, drop {names}, tag {name: tag},
    after {name: bytes appended after the node}; lens {name: content length} is filled in."""
    if isinstance(node, (bytes, bytearray)):
        return bytes(node)
    nm = node.name
    if nm in ctx.get("drop", ()):
        return b""
    if nm in ctx.get("repl", {}):
        r = ctx["repl"][nm]
        return ser(r, ctx, following) if isinstance(r, N) else bytes(r)
    tail = ctx.get("after", {}).get(nm, b"")
    parts, after = [], following + len(tail)
    sib = 0
    for k in reversed(node.kids):
        b = ser(k, ctx, sib)
        parts.append(b)
        sib += len(b)
    c = b"".join(reversed(parts))
    if nm:
        ctx.setdefault("lens", {})[nm] = len(c)
    tag = ctx.get("tag", {}).get(nm, node.tag)
    return _head(tag, len(c), ctx.get("mods", {}).get(nm), after) + c + tail


def xt(oid: bytes, value: bytes, crit: bytes | None = None, name=None, vname=None) -> N:
    """One Extension; crit = the BOOLEAN's content octets when present."""
    kids = [N(0x06, oid)] + ([N(0x01, crit)] if crit is not None else []) + [N(0x04, value, name=vname)]
    return N(0x30, *kids, name=name)


def ent(serial: bytes = b"\x05", when=(UTC, b"251229000000Z"), exts=None, tail: bytes = b"", name=None, iname=None,
        tname=None) -> N:
    kids = [N(0x02, serial, name=iname), N(when[0], when[1], name=tname)]
    if exts is not None:
        kids.append(exts)
    return N(0x30, *kids, tail, name=name)


RDATE0, RDATE1 = (UTC, b"251229000000Z"), (UTC, b"251230120000Z")
RDATE0_S, RDATE1_S = T(2025, 12, 29), T(2025, 12, 30, 12)
THIS, NEXT = (UTC, b"260101000000Z"), (UTC, b"260108000000Z")
THIS_S, NEXT_S = T(2026, 1, 1), T(2026, 1, 8)


def tree(mini: bool = False, cn: int = 0, oid: int = 0, epad: int = 0, serial: int = 0, xpad: int = 0, spad: int = 0,
         sig: int = 257) -> N:
    """The CertificateList every case starts from.  Full: v2, issuer CN, thisUpdate, nextUpdate, two entries (the first
    with a reasonCode 1 and an unknown extension), [0] with cRLNumber and an unknown extension.  `mini`: v2, issuer,
    thisUpdate only.  The pads grow one leaf each: the issuer CN, the ATV's OID, the first entry's unknown extension
    value, its serial, the unknown crlExtension value, the outer signatureAlgorithm's parameters, the signature."""
    atv = N(0x30, N(0x06, long_oid(oid) if oid else CN_OID, name="oid"), N(0x0C, b"Case CA" + b"c" * cn), name="atv")
    name = N(0x30, N(0x31, atv, name="rdn"), name="name")
    kids = [N(0x02, b"\x01", name="ver"), N(0x30, N(0x06, SHA_OID), N(0x05, b""), name="sig"), name,
            N(THIS[0], THIS[1], name="this")]
    if not mini:
        e0 = ent(b"\x01" + b"\x55" * (serial - 1) if serial else b"\x01\x02", RDATE0,
                 N(0x30, xt(REASON_OID, b"\x0a\x01\x01"), xt(UNKNOWN_OID, b"\x33" * epad, name="ext", vname="ostr"),
                   name="exts"), name="ent", iname="int", tname="rdate")
        x0 = N(0xA0, N(0x30, xt(CRL_NUMBER_OID, b"\x02\x01\x07"), xt(UNKNOWN_OID, b"\x44" * xpad), name="xseq"), name="x0")
        kids += [N(NEXT[0], NEXT[1], name="next"), N(0x30, e0, ent(b"\x05", RDATE1), name="rc"), x0]
    params = N(0x05, b"") if not spad else N(0x04, b"\x00" * spad)
    return N(0x30, N(0x30, *kids, name="tbs"), N(0x30, N(0x06, SHA_OID), params, name="salg"),
             N(0x03, b"\x00" + b"\x5a" * (sig - 1), name="bits"), name="cl")


def build(mini=False, pads=None, **ctx) -> bytes:
    return ser(tree(mini, **(pads or {})), ctx)


def full_ok() -> list:
    """the entry statuses of the full tree: both entries joinable"""
    return [RV, RV]


# ------------------------------------------------------------------------------------------------ header levels

ENTRY_LEVELS = ("ent", "int", "rdate", "exts", "ext", "ostr")
LEVELS = ("cl", "tbs", "ver", "sig", "name", "rdn", "atv", "oid", "this", "next", "rc") + ENTRY_LEVELS + \
         ("x0", "xseq", "salg", "bits")
MODS = ("tag1f", "indef", "81", "8200", "85", "past")
# the leaf a long form grows at each level, and whether the full tree is too large to reach 128
PAD_OF = {"cl": "sig", "tbs": "cn", "name": "cn", "rdn": "cn", "atv": "cn", "oid": "oid", "rc": "epad", "ent": "epad",
          "int": "serial", "exts": "epad", "ext": "epad", "ostr": "epad", "x0": "xpad", "xseq": "xpad", "salg": "spad",
          "bits": "sig"}
TIME_LEVELS = ("this", "next", "rdate")


def _fit(level: str, target: int):
    """(DER, mini) of the CRL whose `level` node has exactly `target` content octets, grown through PAD_OF[level]."""
    pad = PAD_OF[level]
    for mini in (False, True):
        if mini and level not in ("cl", "tbs", "name", "rdn", "atv", "oid", "salg", "bits"):
            break
        k = 6 if pad == "oid" else 1
        for _ in range(16):
            ctx = {}
            der = ser(tree(mini, **{pad: k}), ctx)
            n = ctx["lens"][level]
            if n == target:
                return der, mini
            k += target - n
            if k < 1:
                break
    raise AssertionError((level, target))


def header_cases() -> list:
    out = []
    for lv in LEVELS:
        st = BADE if lv in ENTRY_LEVELS else BAD
        for m in MODS:
            out.append(Case(f"header_{lv}_{m}", build(mods={lv: m}), st))
    for lv in list(PAD_OF) + list(TIME_LEVELS):
        for target, form in ((0x80, b"\x81\x80"), (0x100, b"\x82\x01\x00"), (0x10000, b"\x83\x01\x00\x00")):
            if lv in TIME_LEVELS:  # no Time has that many octets
                der = build(repl={lv: N(UTC, b"0" * target)})
                out.append(Case(f"header_{lv}_long_{target}", der, BADE if lv == "rdate" else BAD))
                continue
            der, mini = _fit(lv, target)
            assert form in der
            ents = [] if mini else [LONG if lv == "int" else RV, RV]
            f = {"serial_len": [min(target, 255), 1]} if lv == "int" else {}
            out.append(Case(f"header_{lv}_long_{target}", der, OK, ents, f))
    return out


# ------------------------------------------------------------------------------------------------ TBSCertList

def tbs_cases() -> list:
    F = full_ok()
    name0 = lambda *k: N(0x30, *k)
    c = [
        Case("tbs_version_absent", build(drop={"ver"}), OK, F),
        Case("tbs_version_1", build(), OK, F, {"this_update": THIS_S, "next_update": NEXT_S, "reason": [1, 0xFF]}),
        Case("tbs_version_0", build(repl={"ver": N(0x02, b"\x00")}), BAD),
        Case("tbs_version_2", build(repl={"ver": N(0x02, b"\x02")}), BAD),
        Case("tbs_version_0001", build(repl={"ver": N(0x02, b"\x00\x01")}), BAD),
        Case("tbs_version_enumerated", build(tag={"ver": 0x0A}), BAD),
        Case("tbs_signature_not_sequence", build(repl={"sig": N(0x05, b"")}), BAD),
        Case("tbs_signature_set", build(tag={"sig": 0x31}), BAD),
        Case("tbs_name_empty", build(repl={"name": name0()}), OK, F),
        Case("tbs_name_not_sequence", build(tag={"name": 0x31}), BAD),
        Case("tbs_name_two_rdns", build(repl={"name": name0(N(0x31, N(0x30, N(0x06, CN_OID), N(0x0C, b"A"))),
                                                             N(0x31, N(0x30, N(0x06, CN_OID), N(0x13, b"B"))))}), OK, F),
        Case("tbs_name_empty_rdn", build(repl={"name": name0(N(0x31))}), OK, F),
        Case("tbs_rdn_sequence", build(tag={"rdn": 0x30}), BAD),
        Case("tbs_atv_set", build(tag={"atv": 0x31}), BAD),
        Case("tbs_atv_no_value", build(repl={"atv": N(0x30, N(0x06, CN_OID))}), BAD),
        Case("tbs_atv_value_past_atv", build(repl={"atv": N(0x30, N(0x06, CN_OID), b"\x0c\x05abc")}), BAD),
        Case("tbs_atv_empty", build(repl={"atv": N(0x30)}), BAD),
        Case("tbs_oid_octet_string", build(tag={"oid": 0x04}), BAD),
        Case("tbs_rdn_byte", build(repl={"name": name0(N(0x31, b"\x00"))}), BAD),
        Case("tbs_next_absent_entries", build(drop={"next"}), OK, F, {"next_update": co.INT64_MIN}),
        Case("tbs_next_absent_extensions", build(drop={"next", "rc"}), OK, [], {"next_update": co.INT64_MIN}),
        Case("tbs_next_absent_nothing_after", build(drop={"next", "rc", "x0"}), OK, []),
        Case("tbs_entries_absent", build(drop={"rc"}), OK, []),
        Case("tbs_entries_empty", build(repl={"rc": N(0x30)}), OK, []),
        Case("tbs_two_revoked_certificates", build(after={"rc": bytes(ser(N(0x30, ent()), {}))}), BAD),
        Case("tbs_entries_set", build(tag={"rc": 0x31}), BAD),
        Case("tbs_crlext_context_1", build(tag={"x0": 0xA1}), BAD),
        Case("tbs_crlext_context_0_primitive", build(tag={"x0": 0x80}), BAD),
        Case("tbs_crlext_empty", build(repl={"x0": N(0xA0)}), BAD),
        Case("tbs_crlext_two_sequences", build(after={"xseq": b"\x30\x00"}), BAD),
        Case("tbs_crlext_byte_after_sequence", build(after={"xseq": b"\x00"}), BAD),
        Case("tbs_crlext_not_sequence", build(tag={"xseq": 0x31}), BAD),
        Case("tbs_crlext_empty_extensions", build(repl={"xseq": N(0x30)}), OK, F, {"flags": 0}),
        Case("tbs_two_crlext", build(after={"x0": bytes(ser(N(0xA0, N(0x30)), {}))}), BAD),
        Case("tbs_bytes_after_extensions", build(after={"x0": b"\x05\x00"}), BAD),
        Case("tbs_byte_after_extensions", build(after={"x0": b"\x00"}), BAD),
        Case("tbs_bytes_after_this_update", build(drop={"next", "rc", "x0"}, after={"this": b"\x05\x00"}), BAD),
        Case("tbs_bytes_after_signature", build(after={"bits": b"\x05\x00"}), BAD),
        Case("tbs_byte_after_signature", build(after={"bits": b"\x00"}), BAD),
        Case("tbs_byte_after_outer", build() + b"\x00", BAD),
        Case("tbs_outer_one_short", build()[:-1], BAD),
        Case("tbs_bit_string_empty", build(repl={"bits": N(0x03, b"")}), BAD),
        Case("tbs_bit_string_one_octet", build(repl={"bits": N(0x03, b"\x00")}), OK, F),
        Case("tbs_signature_octet_string", build(tag={"bits": 0x04}), BAD),
        Case("tbs_salg_not_sequence", build(repl={"salg": N(0x05, b"")}), BAD),
        Case("tbs_no_signature", build(drop={"bits"}), BAD),
        Case("tbs_no_salg", build(drop={"salg"}), BAD),
        Case("tbs_tbs_not_sequence", build(tag={"tbs": 0x31}), BAD),
        Case("tbs_outer_set", build(tag={"cl": 0x31}), BAD),
        Case("tbs_no_this_update", build(drop={"this", "next"}), BAD),
    ]
    return c


# ------------------------------------------------------------------------------------------------ Time

TIMES = [  # (name, tag, content, Unix seconds or None when the rules reject it)
    ("utc10", UTC, b"2601010000", None),
    ("utc11", UTC, b"2601010000Z", T(2026, 1, 1)),
    ("utc12", UTC, b"260101000000", None),
    ("utc13", UTC, b"260101000059Z", T(2026, 1, 1, 0, 0, 59)),
    ("utc15", UTC, b"2601010000+0100", T(2025, 12, 31, 23)),
    ("utc17", UTC, b"260101000000-0130", T(2026, 1, 1, 1, 30)),
    ("utc19_fraction", UTC, b"260101000000.5+0100", None),
    ("utc19", UTC, b"260101000000Z000000", None),
    ("gen10", GEN, b"2026010100", None),
    ("gen11", GEN, b"2026010100Z", None),
    ("gen12", GEN, b"202601010000", None),
    ("gen13_no_seconds", GEN, b"202601010000Z", None),
    ("gen15", GEN, b"20260101000000Z", T(2026, 1, 1)),
    ("gen17_no_seconds", GEN, b"202601010000+0100", None),
    ("gen17_fraction", GEN, b"20260101000000.5Z", None),
    ("gen19", GEN, b"20260101000000+0100", T(2025, 12, 31, 23)),
    ("utc_pivot_49", UTC, b"491231235959Z", T(2049, 12, 31, 23, 59, 59)),
    ("utc_pivot_50", UTC, b"500101000000Z", T(1950, 1, 1)),
    ("utc_00", UTC, b"000101000000Z", T(2000, 1, 1)),
    ("utc_99", UTC, b"991231235959Z", T(1999, 12, 31, 23, 59, 59)),
    ("utc_minus_crosses_year", UTC, b"991231230000-0130", T(2000, 1, 1, 0, 30)),
    ("utc_plus_crosses_year", UTC, b"000101003000+0100", T(1999, 12, 31, 23, 30)),
    ("utc_no_seconds_offset", UTC, b"4912312359-2359", T(2050, 1, 1, 23, 58)),
    ("gen_minus_crosses_day", GEN, b"20240229233000-0045", T(2024, 3, 1, 0, 15)),
    ("gen_plus_2359", GEN, b"20260101000000+2359", T(2025, 12, 31, 0, 1)),
    ("gen_plus_crosses_year", GEN, b"21000101000000+0001", T(2099, 12, 31, 23, 59)),
    ("utc_plus_0000", UTC, b"260101000000+0000", None),
    ("utc_minus_0000", UTC, b"260101000000-0000", None),
    ("gen_plus_0000", GEN, b"20260101000000+0000", None),
    ("offset_hour_24", UTC, b"260101000000+2400", None),
    ("offset_minute_60", UTC, b"260101000000+0060", None),
    ("offset_short", UTC, b"260101000000+010", None),
    ("offset_long", UTC, b"260101000000+01000", None),
    ("offset_nondigit", UTC, b"260101000000+01a0", None),
    ("z_then_byte", UTC, b"260101000000Z0", None),
    ("lowercase_z", UTC, b"260101000000z", None),
    ("no_zone", UTC, b"2601010000000", None),
    ("feb29_2000", UTC, b"000229120000Z", T(2000, 2, 29, 12)),
    ("feb29_2024", GEN, b"20240229000000Z", T(2024, 2, 29)),
    ("feb29_2100", GEN, b"21000229000000Z", None),
    ("feb29_1900", GEN, b"19000229000000Z", None),
    ("feb29_2023", UTC, b"230229000000Z", None),
    ("feb28_2100", GEN, b"21000228235959Z", T(2100, 2, 28, 23, 59, 59)),
    ("feb30_2024", UTC, b"240230000000Z", None),
    ("day0", UTC, b"260100000000Z", None),
    ("apr31", UTC, b"260431000000Z", None),
    ("jun31", UTC, b"260631000000Z", None),
    ("sep31", GEN, b"20260931000000Z", None),
    ("nov31", UTC, b"261131000000Z", None),
    ("jan31", UTC, b"260131000000Z", T(2026, 1, 31)),
    ("dec31", UTC, b"261231235959Z", T(2026, 12, 31, 23, 59, 59)),
    ("month0", UTC, b"260001000000Z", None),
    ("month13", UTC, b"261301000000Z", None),
    ("hour24", UTC, b"260101240000Z", None),
    ("minute60", UTC, b"260101006000Z", None),
    ("second60", UTC, b"260101000060Z", None),
    ("gen_second60", GEN, b"20161231235960Z", None),
    ("nondigit_year", UTC, b"2a0101000000Z", None),
    ("nondigit_century", GEN, b"2x260101000000Z", None),
    ("nondigit_second", UTC, b"2601010000a0Z", None),
    ("nondigit_second_2", UTC, b"26010100000aZ", None),
    ("space", UTC, b"26010100 000Z", None),
    ("gen_0000", GEN, b"00000101000000Z", T(1, 1, 1) - 366 * 86400),  # year 0 is a leap year
    ("gen_9999", GEN, b"99991231235959Z", T(9999, 12, 31, 23, 59, 59)),
    ("wrong_tag", 0x04, b"260101000000Z", None),
    ("empty", UTC, b"", None),
]


def time_cases() -> list:
    out = []
    for nm, tag, content, sec in TIMES:
        tn = N(tag, content)
        out.append(Case(f"time_this_{nm}", build(repl={"this": tn}), OK if sec is not None else BAD,
                        full_ok() if sec is not None else None, {"this_update": sec} if sec is not None else {}))
        out.append(Case(f"time_next_{nm}", build(repl={"next": tn}), OK if sec is not None else BAD,
                        full_ok() if sec is not None else None, {"next_update": sec} if sec is not None else {}))
        out.append(Case(f"time_rdate_{nm}", build(repl={"rdate": tn}), OK if sec is not None else BADE,
                        full_ok() if sec is not None else None, {"revoked_at": [sec, RDATE1_S]} if sec is not None else {}))
    return out


# ------------------------------------------------------------------------------------------------ entries

def _rc(*entries, **ctx) -> bytes:
    return build(repl={"rc": N(0x30, *entries)}, **ctx)


def _reason(v: bytes, crit=None):
    return N(0x30, xt(REASON_OID, v, crit))


def entry_cases() -> list:
    out = []
    for n in list(range(1, 41)) + [127, 128, 255, 256, 300]:
        s = bytes([0x41 + n % 50]) * n
        out.append(Case(f"entry_serial_{n}", _rc(ent(s), ent(b"\x05", RDATE1)), OK, [RV if n <= 39 else LONG, RV],
                        {"serial_len": [min(n, 255), 1], "revoked_at": [RDATE0_S, RDATE1_S]}))
    E = lambda *e: _rc(*e, ent(b"\x05", RDATE1))
    c = [
        Case("entry_serial_0", E(ent(b"")), BADE),
        Case("entry_serial_negative_80", E(ent(b"\x80")), OK, [RV, RV]),
        Case("entry_serial_negative_ff", E(ent(b"\xff")), OK, [RV, RV]),
        Case("entry_serial_negative_ff7f", E(ent(b"\xff\x7f")), OK, [RV, RV]),
        Case("entry_serial_0001", E(ent(b"\x00\x01")), OK, [RV, RV], {"serial_len": [2, 1]}),
        Case("entry_serial_enumerated", E(N(0x30, N(0x0A, b"\x01"), N(UTC, RDATE0[1]))), BADE),
        Case("entry_no_date", E(N(0x30, N(0x02, b"\x01"))), BADE),
        Case("entry_empty", E(N(0x30)), BADE),
        Case("entry_byte_after_date", E(ent(tail=b"\x00")), BADE),
        Case("entry_null_after_date", E(ent(tail=b"\x05\x00")), BADE),
        Case("entry_byte_after_extensions", E(ent(exts=N(0x30), tail=b"\x00")), BADE),
        Case("entry_two_extensions_sequences", E(ent(exts=N(0x30), tail=b"\x30\x00")), BADE),
        Case("entry_extensions_empty", E(ent(exts=N(0x30))), OK, [RV, RV], {"reason": [0xFF, 0xFF]}),
        Case("entry_extensions_set", E(ent(exts=N(0x31, xt(UNKNOWN_OID, b"")))), BADE),
        Case("entry_extensions_context_0", E(ent(exts=N(0xA0, N(0x30, xt(UNKNOWN_OID, b""))))), BADE),
        Case("entry_reason_0", E(ent(exts=_reason(b"\x0a\x01\x00"))), OK, [RV, RV], {"reason": [0, 0xFF]}),
        Case("entry_reason_10", E(ent(exts=_reason(b"\x0a\x01\x0a"))), OK, [RV, RV], {"reason": [10, 0xFF]}),
        Case("entry_reason_trailing_byte", E(ent(exts=_reason(b"\x0a\x01\x01\x00"))), BADE),
        Case("entry_reason_empty_value", E(ent(exts=_reason(b""))), BADE),
        Case("entry_reason_no_octets", E(ent(exts=_reason(b"\x0a\x00"))), BADE),
        Case("entry_reason_integer", E(ent(exts=_reason(b"\x02\x01\x01"))), BADE),
        Case("entry_reason_two_octets", E(ent(exts=_reason(b"\x0a\x02\x00\x01"))), BADE),
        Case("entry_reason_twice", E(ent(exts=N(0x30, xt(REASON_OID, b"\x0a\x01\x01"), xt(REASON_OID, b"\x0a\x01\x05")))),
             OK, [RV, RV], {"reason": [5, 0xFF]}),
        Case("entry_critical_ff", E(ent(exts=_reason(b"\x0a\x01\x03", b"\xff"))), OK, [RV, RV], {"reason": [3, 0xFF]}),
        Case("entry_critical_00", E(ent(exts=_reason(b"\x0a\x01\x03", b"\x00"))), OK, [RV, RV], {"reason": [3, 0xFF]}),
        Case("entry_critical_01", E(ent(exts=_reason(b"\x0a\x01\x03", b"\x01"))), BADE),
        Case("entry_critical_two_octets", E(ent(exts=_reason(b"\x0a\x01\x03", b"\x00\xff"))), BADE),
        Case("entry_critical_empty", E(ent(exts=_reason(b"\x0a\x01\x03", b""))), BADE),
        Case("entry_cert_issuer", E(ent(exts=N(0x30, xt(CERT_ISSUER_OID, b"\x30\x00")))), OK, [IND, RV]),
        Case("entry_cert_issuer_and_reason", E(ent(exts=N(0x30, xt(REASON_OID, b"\x0a\x01\x04"),
                                                          xt(CERT_ISSUER_OID, b"\x30\x00", b"\xff")))),
             OK, [IND, RV], {"reason": [4, 0xFF]}),
        Case("entry_cert_issuer_long_serial", E(ent(b"\x07" * 45, exts=N(0x30, xt(CERT_ISSUER_OID, b"")))), OK, [IND, RV]),
        Case("entry_unknown_extensions", E(ent(exts=N(0x30, xt(UNKNOWN_OID, b"\x01\x02"), xt(b"\x55\x1d\x18", b"", b"\xff")))),
             OK, [RV, RV], {"reason": [0xFF, 0xFF]}),
        Case("entry_extension_no_octet_string", E(ent(exts=N(0x30, N(0x30, N(0x06, UNKNOWN_OID))))), BADE),
        Case("entry_extension_critical_no_octet_string", E(ent(exts=N(0x30, N(0x30, N(0x06, UNKNOWN_OID), N(0x01, b"\xff"))))),
             BADE),
        Case("entry_extension_bit_string_value", E(ent(exts=N(0x30, N(0x30, N(0x06, UNKNOWN_OID), N(0x03, b"\x00"))))), BADE),
        Case("entry_extension_byte_after_value", E(ent(exts=N(0x30, N(0x30, N(0x06, UNKNOWN_OID), N(0x04, b""), b"\x00")))),
             BADE),
        Case("entry_extension_no_oid", E(ent(exts=N(0x30, N(0x30, N(0x04, b""))))), BADE),
        Case("entry_extension_empty", E(ent(exts=N(0x30, N(0x30)))), BADE),
        Case("entry_extension_set", E(ent(exts=N(0x30, N(0x31, N(0x06, UNKNOWN_OID), N(0x04, b""))))), BADE),
        Case("entry_oid_551d1500_not_reason", E(ent(exts=N(0x30, xt(b"\x55\x1d\x15\x00", b"\x05\x00")))), OK, [RV, RV],
             {"reason": [0xFF, 0xFF]}),
        Case("entry_oid_551d1d00_not_issuer", E(ent(exts=N(0x30, xt(b"\x55\x1d\x1d\x00", b"")))), OK, [RV, RV]),
        Case("entry_oid_551d_not_reason", E(ent(exts=N(0x30, xt(b"\x55\x1d", b"\x05\x00")))), OK, [RV, RV]),
        Case("entry_oid_reason_in_four", E(ent(exts=N(0x30, xt(b"\x00\x55\x1d\x15", b"")))), OK, [RV, RV]),
    ]
    return out + c


# ------------------------------------------------------------------------------------------------ crlExtensions

def crlext_cases() -> list:
    F = full_ok()
    X = lambda *x: build(repl={"x0": N(0xA0, N(0x30, *x))})
    delta, idp = xt(DELTA_OID, b"\x02\x01\x01"), xt(IDP_OID, b"\x30\x00")
    return [
        Case("crlext_delta", X(delta), OK, F, {"flags": 1}),
        Case("crlext_idp", X(idp), OK, F, {"flags": 2}),
        Case("crlext_both", X(idp, delta), OK, F, {"flags": 3}),
        Case("crlext_both_critical", X(xt(DELTA_OID, b"\x02\x01\x01", b"\xff"), xt(IDP_OID, b"\x30\x00", b"\xff")), OK, F,
             {"flags": 3}),
        Case("crlext_delta_critical_00", X(xt(DELTA_OID, b"", b"\x00")), OK, F, {"flags": 1}),
        Case("crlext_critical_01", X(xt(DELTA_OID, b"", b"\x01")), BAD),
        Case("crlext_oid_551d1b00", X(xt(b"\x55\x1d\x1b\x00", b"")), OK, F, {"flags": 0}),
        Case("crlext_oid_551d1c01", X(xt(b"\x55\x1d\x1c\x01", b"")), OK, F, {"flags": 0}),
        Case("crlext_oid_551d1b00_and_idp", X(xt(b"\x55\x1d\x1b\x00", b""), idp), OK, F, {"flags": 2}),
        Case("crlext_no_octet_string", X(N(0x30, N(0x06, DELTA_OID))), BAD),
        Case("crlext_value_integer", X(N(0x30, N(0x06, DELTA_OID), N(0x02, b"\x01"))), BAD),
        Case("crlext_reason_code_ignored", X(xt(REASON_OID, b"\xff\xff")), OK, F, {"flags": 0}),
        Case("crlext_delta_without_version", build(drop={"ver"}, repl={"x0": N(0xA0, N(0x30, delta))}), OK, F, {"flags": 1}),
        Case("crlext_bad_after_good", X(delta, N(0x30, N(0x06, IDP_OID))), BAD),
        Case("crlext_on_bad_entries", build(repl={"rc": N(0x30, b"\x30\x01\x02"), "x0": N(0xA0, N(0x30, delta))}), BADE),
    ]


# ------------------------------------------------------------------------------------------------ the split

def _min_crl(content: bytes, sig: int = 1) -> bytes:
    """The smallest CRL around revokedCertificates content: v2, an empty Name, thisUpdate, the entries."""
    return ser(N(0x30, N(0x30, N(0x02, b"\x01"), N(0x30, N(0x06, SHA_OID)), N(0x30), N(UTC, b"260101000000Z"),
                         N(0x30, content)),
                 N(0x30, N(0x06, SHA_OID)), N(0x03, b"\x00" + b"\x5a" * (sig - 1))), {})


def min_entry(i: int) -> bytes:
    """An 18-byte entry: SEQUENCE 2 + INTEGER 3 + UTCTime without seconds 13."""
    e = ser(ent(bytes([1 + i % 0x7F]), (UTC, b"2512290000Z")), {})
    assert len(e) == 18
    return e


PH = b"\xee" * 12  # a placeholder of the false candidate's length


def _false_candidate(entries: list, at: int, target: str) -> bytes:
    """Content of `entries` (built by f(placeholder)) whose entry `at` holds `30 M 02 01 01` in its serial or in an
    extension value, M chosen so that the candidate's next lands on the following entry ('next'), on the content end
    ('end') or one past it ('past')."""
    def make(fill):
        return [ser(e(fill if i == at else PH), {}) for i, e in enumerate(entries)]
    ents = make(PH)
    content = b"".join(ents)
    off = sum(len(e) for e in ents[:at]) + ents[at].index(PH)
    goal = {"next": sum(len(e) for e in ents[:at + 1]), "end": len(content), "past": len(content) + 1}[target]
    m = goal - off - 2
    if m >= 0x80:
        m -= 1
    cand = hdr(0x30, m) + b"\x02\x01\x01"
    assert off + len(hdr(0x30, m)) + m == goal
    out = b"".join(make(cand + b"\xee" * (len(PH) - len(cand))))
    assert len(out) == len(content)
    return out


def split_cases() -> list:
    out = []
    in_serial = lambda s: (lambda ph: ent(b"\x01" + ph, RDATE0))
    in_ext = lambda s: (lambda ph: ent(bytes([s]), RDATE1, N(0x30, xt(UNKNOWN_OID, ph))))
    for kind, mk in (("serial", in_serial), ("ext", in_ext)):
        for at in (0, 2):
            for target in ("next", "end", "past"):
                if at == 2 and target == "next":
                    continue  # the last entry's next entry is the content end
                fs = [mk(i + 1) for i in range(3)]
                content = _false_candidate(fs, at, target)
                out.append(Case(f"split_false_{kind}_entry{at}_{target}", _min_crl(content), OK, [RV] * 3))
    # a false candidate that lands on a later entry while the real chain breaks before it
    fs = [lambda ph: ent(b"\x01" + ph, RDATE0), lambda ph: N(0x30, N(0x02, b"\x01")), lambda ph: ent(b"\x03", RDATE1)]
    c = _false_candidate(fs, 0, "end")
    out.append(Case("split_false_candidate_over_a_broken_entry", _min_crl(c), BADE))
    # entries at every phase mod 16 inside one CRL
    ents = [ser(ent(bytes([0x10 + n]) * n, RDATE0), {}) for n in range(1, 33)]
    out.append(Case("split_entries_every_phase", _min_crl(b"".join(ents)), OK, [RV] * 32))
    # CRL boundaries at every phase mod 16: sixteen CRLs of 16k + 1 bytes back to back
    for i in range(16):
        c = b"".join(ser(ent(bytes([1 + i, j + 1]), RDATE0), {}) for j in range(3))
        s = 1 + 16 * (i % 3)
        while len(_min_crl(c, s)) % 16 != 1:
            s += 1
        out.append(Case(f"split_boundary_{i}", _min_crl(c, s), OK, [RV] * 3))
    # chains of 2^k - 1, 2^k and 2^k + 1 minimal entries
    for n in sorted({(1 << k) + d for k in range(1, 13) for d in (-1, 0, 1)}):
        out.append(Case(f"split_chain_{n}", _min_crl(b"".join(min_entry(i) for i in range(n))), OK, [RV] * n))
    # 2^R good entries, then 30 01 02
    for r in (0, 3, 6, 10):
        out.append(Case(f"split_tail_after_{1 << r}", _min_crl(b"".join(min_entry(i) for i in range(1 << r)) + b"\x30\x01\x02"),
                        BADE))
    out.append(Case("split_30_01_02_only", _min_crl(b"\x30\x01\x02" * 400), BADE))
    out.append(Case("split_last_entry_one_short", _min_crl(min_entry(0) + min_entry(1)[:-1]), BADE))
    out.append(Case("split_crl_of_0_bytes", b"", BAD))
    out.append(Case("split_between_0_and_1", _min_crl(min_entry(5)), OK, [RV]))
    out.append(Case("split_crl_of_1_byte", b"\x30", BAD))
    out.append(Case("split_after_1", _min_crl(min_entry(6) + min_entry(7)), OK, [RV, RV]))
    return out


@functools.lru_cache(maxsize=None)
def catalogue() -> tuple:
    cases = header_cases() + tbs_cases() + time_cases() + entry_cases() + crlext_cases() + split_cases()
    names = [c.name for c in cases]
    assert len(names) == len(set(names)), "case names are unique"
    return tuple(cases)


# ------------------------------------------------------------------------------------------------ seeded mutants

def spans(d: bytes, pos: int = 0, end: int | None = None, out=None) -> list:
    """(start, header length, content length) of every TLV of well-formed DER, descending into constructed ones."""
    out = [] if out is None else out
    end = len(d) if end is None else end
    while pos < end:
        tag, h, n = co.read(d, pos, end)
        out.append((pos, h, n))
        if tag & 0x20:
            spans(d, pos + h, pos + h + n, out)
        pos += h + n
    return out


def _seed(rng: random.Random, i: int):
    """A valid CRL and its entry nodes"""
    ents = []
    for j in range(rng.randint(0, 7)):
        s = bytes([rng.randint(1, 0x7F)]) + bytes(rng.randint(0, 255) for _ in range(rng.randint(0, 20)))
        x = []
        if rng.random() < 0.4:
            x.append(xt(REASON_OID, bytes([0x0A, 1, rng.randint(0, 10)]), b"\xff" if rng.random() < 0.2 else None))
        if rng.random() < 0.2:
            x.append(xt(UNKNOWN_OID, bytes(rng.randint(0, 255) for _ in range(rng.randint(0, 9)))))
        if rng.random() < 0.1:
            x.append(xt(CERT_ISSUER_OID, b"\x30\x00"))
        when = rng.choice([(UTC, b"251229000000Z"), (UTC, b"2512291200Z"), (GEN, b"20251229000000Z"),
                           (UTC, b"251229000000+0130")])
        ents.append(ent(s, when, N(0x30, *x) if x or rng.random() < 0.1 else None))
    ctx = {"repl": {"rc": N(0x30, *ents)}, "drop": set()}
    if not ents and rng.random() < 0.5:
        ctx["drop"].add("rc")
    if rng.random() < 0.3:
        ctx["drop"].add("next")
    if rng.random() < 0.3:
        ctx["repl"]["x0"] = N(0xA0, N(0x30, *([xt(DELTA_OID, b"\x02\x01\x01", b"\xff")] if rng.random() < 0.5 else [])))
    pads = {"sig": rng.randint(1, 40), "cn": rng.randint(0, 10)}
    return ser(tree(False, **pads), ctx), ents, ctx, pads


def mutants(n_seeds: int = 50, seed: int = 1) -> list:
    """About 400 mutants of each of n_seeds valid CRLs: byte flips, inserts and deletes, truncations at every TLV
    boundary, a header's length +-1, and duplicated or swapped entries."""
    rng = random.Random(seed)
    out = []
    for i in range(n_seeds):
        der, ents, ctx, pads = _seed(rng, i)
        assert co.parse_crl(der)["status"] == OK
        L = len(der)
        for _ in range(120):
            p = rng.randrange(L)
            out.append(der[:p] + bytes([der[p] ^ rng.randint(1, 255)]) + der[p + 1:])
        for _ in range(60):
            p = rng.randrange(L + 1)
            out.append(der[:p] + bytes([rng.choice([0x00, 0x02, 0x30, 0x80, 0x81, rng.randint(0, 255)])]) + der[p:])
        for _ in range(60):
            p = rng.randrange(L)
            out.append(der[:p] + der[p + 1:])
        sp = spans(der)
        cuts = sorted({s for s, _, _ in sp} | {s + h + n for s, h, n in sp} | {s + h for s, h, _ in sp})
        out += [der[:c] for c in cuts if c < L]
        for _ in range(80):
            s, h, n = rng.choice(sp)
            b = bytearray(der)
            last = s + h - 1
            b[last] = (b[last] + rng.choice([1, -1])) & 0xFF
            out.append(bytes(b))
        for _ in range(20):
            if len(ents) < 1:
                break
            es = list(ents)
            a, c = rng.randrange(len(es)), rng.randrange(len(es))
            if rng.random() < 0.5:
                es.insert(c, es[a])
            else:
                es[a], es[c] = es[c], es[a]
            ctx2 = dict(ctx, repl=dict(ctx["repl"], rc=N(0x30, *es)))
            out.append(ser(tree(False, **pads), ctx2))
    return out
