"""Property tests of the oracle's leaves against independent Python implementations (hashlib,
base64, datetime, calendar) -- hypothesis-driven.  These pin the arithmetic the reference takes from
Go's standard library: crypto/sha256 (storage/types.go:156), encoding/base64.URLEncoding (:157),
time.Truncate(time.Hour) and the "2006-01-02-15" layout (:339-346, :379-384), encoding/asn1's
UTCTime / GeneralizedTime rules (via ct-go x509, call sites cmd/ct-fetch/ct-fetch.go:202,221)."""
import base64
import calendar
import datetime
import hashlib

import numpy as np
from hypothesis import given, settings, strategies as st

import der_build as D
from conftest import pack


@settings(max_examples=200, deadline=None)
@given(st.binary(min_size=0, max_size=600))
def test_sha256_matches_hashlib(ora, data):
    assert ora.sha256(data) == hashlib.sha256(data).digest()


@settings(max_examples=200, deadline=None)
@given(st.binary(min_size=0, max_size=100))
def test_base64url_matches_python(ora, data):
    assert ora.b64url(data) == base64.urlsafe_b64encode(data).decode()


@settings(max_examples=300, deadline=None)
@given(st.integers(min_value=-62135596800, max_value=253402300799))  # years 0001..9999
def test_exp_hour_and_ids_match_datetime(ora, sec):
    hour = ora.exp_hour(sec)
    assert hour == sec // 3600  # floor, also before 1970
    t = datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc) + datetime.timedelta(seconds=hour * 3600)
    assert ora.expdate_id(hour) == "%04d-%02d-%02d-%02d" % (t.year, t.month, t.day, t.hour)
    d = datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc) + datetime.timedelta(seconds=(sec // 86400) * 86400)
    assert ora.day_id(sec) == "%04d-%02d-%02d" % (d.year, d.month, d.day)


def _cert_with_times(nb: bytes, na: bytes, nb_tag=0x17, na_tag=0x17, serial: bytes = b"\x01") -> bytes:
    """A minimal certificate skeleton (no extensions) with the given validity encodings and serial content octets."""
    return D.cert(serial=serial, subject=[[D.cn(b"ca")]], not_before=D.tlv(nb_tag, nb), not_after=D.tlv(na_tag, na)).der


def _fmt_utc(t: datetime.datetime) -> bytes:
    return t.strftime("%y%m%d%H%M%SZ").encode()


@settings(max_examples=150, deadline=None)
@given(st.datetimes(min_value=datetime.datetime(1950, 1, 1), max_value=datetime.datetime(2049, 12, 31, 23, 59, 59)))
def test_utctime_pivot_and_value(ora, t):
    t = t.replace(microsecond=0)
    der = _cert_with_times(_fmt_utc(datetime.datetime(1990, 1, 1)), _fmt_utc(t))
    rc, c = ora.parse_cert(der)
    assert rc == 0
    assert c.not_after == calendar.timegm(t.timetuple())  # yy >= 50 -> 19yy, else 20yy


@settings(max_examples=150, deadline=None)
@given(st.datetimes(min_value=datetime.datetime(1, 1, 1), max_value=datetime.datetime(9999, 12, 31, 23, 59, 59)))
def test_generalizedtime_value(ora, t):
    t = t.replace(microsecond=0)
    s = ("%04d%02d%02d%02d%02d%02dZ" % (t.year, t.month, t.day, t.hour, t.minute, t.second)).encode()
    der = _cert_with_times(_fmt_utc(datetime.datetime(1990, 1, 1)), s, na_tag=0x18)
    rc, c = ora.parse_cert(der)
    assert rc == 0
    assert c.not_after == calendar.timegm(t.timetuple())


def test_time_forms_go_accepts_and_rejects(ora):
    ok = lambda na, tag=0x17: ora.parse_cert(_cert_with_times(b"900101000000Z", na, na_tag=tag))
    base = calendar.timegm((2030, 6, 15, 12, 30, 45))
    assert ok(b"300615123045Z")[1].not_after == base
    assert ok(b"3006151230Z")[1].not_after == base - 45                  # UTCTime without seconds ("0601021504Z0700")
    assert ok(b"300615123045+0130")[1].not_after == base - 5400          # numeric offset
    assert ok(b"300615123045-0800")[1].not_after == base + 8 * 3600
    assert ok(b"20300615123045Z", 0x18)[1].not_after == base
    for bad in (b"300615123045+0000",   # zero offset re-serialises as Z -> rejected
                b"301315123045Z", b"300632123045Z", b"300615243045Z", b"300615126045Z", b"300615123060Z",
                b"300229123045Z",       # 2030 is not a leap year
                b"30061512304Z", b"300615123045", b"3006151230456Z", b"30061512304xZ"):
        assert ok(bad)[0] != 0, bad
    assert ok(b"280229123045Z")[0] == 0                                   # 2028 is a leap year
    assert ok(b"203006151230Z", 0x18)[0] != 0                             # GeneralizedTime needs seconds
    assert ok(b"300615123045Z", 0x18)[0] != 0                             # wrong tag for the form


def test_der_length_rules(ora, golden):
    """encoding/asn1 parseTagAndLength: non-minimal and indefinite lengths are structural errors."""
    der = golden["kLeadingZeroes"]["der"]
    assert ora.parse_cert(der)[0] == 0
    assert der[:4] == bytes.fromhex("308202a3")
    assert ora.parse_cert(bytes.fromhex("30830002a3") + der[4:])[0] != 0   # superfluous leading zero in the length
    assert ora.parse_cert(bytes.fromhex("3080") + der[4:])[0] != 0         # indefinite
    assert ora.parse_cert(der + b"\x00")[0] != 0                           # trailing data
    assert ora.parse_cert(der[:-1])[0] != 0
    short = bytes.fromhex("308103") + b"\x02\x01\x00"                       # 0x81 used for a length < 128
    assert ora.parse_cert(short)[0] != 0


@settings(max_examples=60, deadline=None)
@given(st.lists(st.binary(min_size=1, max_size=20), min_size=1, max_size=40), st.integers(0, 2**31))
def test_set_semantics_match_python_sets(ora, members, hour):
    """MockRemoteCache.SetInsert (mockcache.go:38-61): true exactly on first sight; sorted unique listing."""
    cache = ora.Cache()
    seen = set()
    for m in members:
        assert cache.was_unknown(hour, "issuer", m) == (m not in seen)
        seen.add(m)
    key = ora.serials_key(hour, "issuer")
    assert cache.set_cardinality(key) == len(seen)
    assert cache.set_list(key) == sorted(seen)


@settings(max_examples=200, deadline=None)
@given(st.binary(min_size=0, max_size=400))
def test_pem_expectation_matches_an_independent_encoder(data):
    """conftest.go_pem is what the GPU's PEM output is compared with (encoding/pem.EncodeToMemory, 64-character lines,
    storage/filesystemdatabase.go:171-175,197-198); pin it against Python's ssl module for every length residue."""
    import ssl
    from conftest import go_pem
    if data:
        assert go_pem(data).decode() == ssl.DER_cert_to_PEM_cert(data)
    else:  # Go writes no body line for an empty block; ssl emits an empty one
        assert go_pem(data) == b"-----BEGIN CERTIFICATE-----\n-----END CERTIFICATE-----\n"


def test_oracle_has_no_serial_length_limit(ora):
    """NewSerial keeps the raw INTEGER content whatever its length (storage/types.go:171-178): the oracle states the
    reference, so serials of 40 and 200 octets are stored and de-duplicated like any other (VERDICT r1, weak #2)."""
    from conftest import NOW_NS
    ders = []
    for n in (20, 39, 40, 200):
        ser = bytes([0x01]) + bytes([n & 0xFF]) * (n - 1)
        ders += [_cert_with_times(b"900101000000Z", b"300615123045Z", serial=ser)] * 2
    blob, offs = pack(ders)
    iblob, ioffs = pack([ders[0]])
    r = ora.DB(b"", True).process(blob, offs, iblob, ioffs, np.zeros(len(ders), np.uint32), NOW_NS)
    assert (r.status == 0).all()
    assert r.serial_len.tolist() == [20, 20, 39, 39, 40, 40, 200, 200]
    assert r.was_unknown.tolist() == [1, 0, 1, 0, 1, 0, 1, 0]
