"""crl_oracle (the rules of ctmr_revoked_known restated) against `cryptography` on CRLs it builds and signs, and the
ctypes mirrors of the two CRL structs against include/ctmr.h."""
import ctypes as C
import datetime
import subprocess

import pytest

import crl_build as cb
import crl_oracle as co
from conftest import ROOT

x509 = pytest.importorskip("cryptography.x509")
from cryptography.hazmat.primitives import hashes  # noqa: E402
from cryptography.hazmat.primitives.asymmetric import ec  # noqa: E402
from cryptography.x509.oid import NameOID  # noqa: E402

KEY = ec.generate_private_key(ec.SECP256R1())
T0 = datetime.datetime(2026, 1, 1, tzinfo=datetime.timezone.utc)


def _signed(serials, next_update=True, reasons=None, delta=False):
    b = (x509.CertificateRevocationListBuilder()
         .issuer_name(x509.Name([x509.NameAttribute(NameOID.COMMON_NAME, "Oracle CA")]))
         .last_update(T0))
    if next_update:
        b = b.next_update(T0 + datetime.timedelta(days=7))
    if delta:
        b = b.add_extension(x509.DeltaCRLIndicator(1), critical=True)
    for i, s in enumerate(serials):
        rb = x509.RevokedCertificateBuilder().serial_number(s).revocation_date(T0 - datetime.timedelta(hours=i))
        if reasons and reasons[i] is not None:
            rb = rb.add_extension(x509.CRLReason(reasons[i]), critical=False)
        b = b.add_revoked_certificate(rb.build())
    return b.sign(KEY, hashes.SHA256())


@pytest.mark.parametrize("case", ["v2", "no_next_update", "empty", "reasons", "large_serials", "leading_zero", "delta"])
def test_oracle_agrees_with_cryptography(case):
    serials = [1, 2, 0x7F, 0x80, 0xFFFF, 12345678901234567890]
    kw = {}
    if case == "empty":
        serials = []
    if case == "large_serials":
        serials = [(1 << 159) - 1, 1 << 158, 0x00AA]
    if case == "leading_zero":
        serials = [0x80, 0xAA, 0xFF00]  # encoded 00 80, 00 aa, 00 ff 00
    if case == "reasons":
        kw["reasons"] = [x509.ReasonFlags.key_compromise, None, x509.ReasonFlags.superseded, None, x509.ReasonFlags.cessation_of_operation, None]
    if case == "no_next_update":
        kw["next_update"] = False
    if case == "delta":
        kw["delta"] = True
    if kw.pop("next_update", True):
        crl = _signed(serials, **kw)
        der = crl.public_bytes(__import__("cryptography.hazmat.primitives.serialization", fromlist=["Encoding"]).Encoding.DER)
    else:  # cryptography's builder always writes nextUpdate: build it here and let cryptography parse it
        der = cb.crl(next_update=None, entries=[cb.entry(cb.serial_der(s), 1767000000 - i) for i, s in enumerate(serials)])
        crl = x509.load_der_x509_crl(der)
    r = co.parse_crl(der)
    assert r["status"] == co.CRL_OK
    assert r["this_update"] == int(crl.last_update_utc.timestamp())
    if crl.next_update_utc is None:
        assert r["next_update"] == co.INT64_MIN
    else:
        assert r["next_update"] == int(crl.next_update_utc.timestamp())
    off, ln = r["tbs"]
    assert der[off:off + ln] == crl.tbs_certlist_bytes
    assert r["flags"] == (1 if case == "delta" else 0)
    got = {int.from_bytes(e["serial"], "big", signed=True): e for e in r["entries"]}
    want = {rc.serial_number: rc for rc in crl}
    assert set(got) == set(want)
    for s, rc in want.items():
        e = got[s]
        assert e["serial"] == cb.serial_der(s)
        assert e["revoked_at"] == int(rc.revocation_date_utc.timestamp())
        try:
            reason = rc.extensions.get_extension_for_class(x509.CRLReason).value.reason
            codes = {x509.ReasonFlags.key_compromise: 1, x509.ReasonFlags.superseded: 4, x509.ReasonFlags.cessation_of_operation: 5}
            assert e["reason"] == codes[reason]
        except x509.ExtensionNotFound:
            assert e["reason"] == 0xFF


def test_oracle_rules_on_crafted_crls():
    good = cb.crl(entries=[cb.entry(b"\x01", 1767000000), cb.entry(b"\x02", 1767000000, seconds=False)])
    assert co.parse_crl(good)["status"] == co.CRL_OK and len(co.parse_crl(good)["entries"]) == 2
    assert len(cb.entry(b"\x01", 1767000000, seconds=False)) == 18  # the smallest entry
    assert co.parse_crl(cb.crl(entries=None, version=None))["status"] == co.CRL_OK  # v1, no revokedCertificates
    assert co.parse_crl(good + b"\x00")["status"] == co.CRL_BAD
    assert co.parse_crl(cb.crl(entries=[], version=2))["status"] == co.CRL_BAD  # version 2 is v3: not a CRL version
    bad = cb.crl(entries_raw=cb.entry(b"\x01", 1767000000) + b"\x30\x01\x02")
    assert co.parse_crl(bad)["status"] == co.CRL_BAD_ENTRIES
    ind = co.parse_crl(cb.crl(entries=[cb.entry(b"\x05", 1767000000, cert_issuer=True)]))
    assert ind["entries"][0]["status"] == co.RV_INDIRECT
    long = co.parse_crl(cb.crl(entries=[cb.entry(b"\x01" * 40, 1767000000)]))
    assert long["entries"][0]["status"] == co.RV_SERIAL_TOO_LONG
    flags = co.parse_crl(cb.crl(entries=[], delta=True, idp=True))
    assert flags["flags"] == 3


def test_crl_struct_layouts_match_header(tmp_path):
    from ct_mapreduce_b200 import capi
    src = tmp_path / "probe.c"
    src.write_text('#include "include/ctmr.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(ctmr_crl_batch), sizeof(ctmr_crl_out),'
                   'offsetof(ctmr_crl_out, known_sets), offsetof(ctmr_crl_out, entry_cap), offsetof(ctmr_crl_out, n_entries));return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", ROOT, str(src), "-o", str(exe)], check=True, cwd=ROOT)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(capi.CrlBatch), C.sizeof(capi.CrlOut), capi.CrlOut.known_sets.offset, capi.CrlOut.entry_cap.offset,
                   capi.CrlOut.n_entries.offset]
