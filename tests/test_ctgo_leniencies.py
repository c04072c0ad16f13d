"""What the path does NOT model of ct-go's x509 fork -- as tests, not prose (VERDICT r1, next-round item 7).

The reference parses with github.com/google/certificate-transparency-go v1.1.0 (go.mod:10), a fork of Go's crypto/x509
+ encoding/asn1 whose source is NOT in the reference repository, so none of this can be pinned against the reference here
("parity unpinned", SURVEY.md §8(c)).  What CAN be stated is (i) what the oracle and the CUDA walker do today -- asserted
below, so a change is noticed -- and (ii) what Go's own encoding/asn1 / crypto/x509 (1.13, the base of the fork) is
documented to do with the same bytes -- recorded as a strict xfail: the test "fails as expected" for as long as the
divergence exists, and turns into an error the day someone models the behaviour without removing the marker.

Why each divergence is tolerated: the worker only reaches Store for certificates ct-go parsed; an input that Go would
REJECT and this path ACCEPTS ends up as one extra serial in a set (status OK instead of PARSE_ERR) -- never a crash,
never a mis-attributed key.  CT logs only accept certificates that chain to a trusted root, so such inputs are rare in
the wild; the synthetic corpus and the reference's three fixtures contain none.
"""
import numpy as np
import pytest

import der_build as D
from conftest import NOW_NS, pack
from der_build import tlv

ST_OK, ST_PARSE_ERR, ST_FILTER_CA, ST_FILTER_EXPIRED, ST_FILTER_CN = 0, 1, 2, 3, 4


ALG = D.SHA256_RSA
RSA_ALG = D.RSA_ENC
GOOD_KEY = D.RSA_KEY_BITS[1:]


def name(cn_tag=0x0C, cn=b"ca"):
    return [[D.cn(cn, cn_tag)]]


def cert(issuer=None, serial=b"\x01", key=GOOD_KEY, extensions=None):
    return D.cert(issuer=issuer, serial=serial, subject=name(), spki_bits=b"\x00" + key, extensions=extensions).der


def extension(oid_hex, value, critical=False):
    return tlv(0x30, bytes.fromhex(oid_hex) + (b"\x01\x01\xff" if critical else b"") + tlv(0x04, value))


def status_of(ora, der, flt=b""):
    blob, offs = pack([der])
    iblob, ioffs = pack([cert()])
    r = ora.DB(flt, True).process(blob, offs, iblob, ioffs, np.zeros(1, np.uint32), NOW_NS)
    return int(r.status[0])


# (name, DER, what this path does, what Go 1.13 encoding/asn1 + crypto/x509 does, why)
CASES = [
    ("printablestring_with_invalid_character",
     cert(issuer=name(0x13, b"bad@char_")), ST_OK, ST_PARSE_ERR,
     "encoding/asn1 parsePrintableString: '@' and '_' are outside the PrintableString alphabet -> 'asn1: syntax error: "
     "PrintableString contains invalid character'; the walker does not validate string alphabets inside Names"),
    ("ia5string_with_high_bit",
     cert(issuer=name(0x16, b"caf\xe9")), ST_OK, ST_PARSE_ERR,
     "encoding/asn1 parseIA5String rejects bytes >= 0x80; not validated here"),
    ("utf8string_that_is_not_utf8",
     cert(issuer=name(0x0C, b"\xff\xfe")), ST_OK, ST_PARSE_ERR,
     "encoding/asn1 parseUTF8String: 'asn1: invalid UTF-8 string'; not validated here"),
    ("rsa_key_with_zero_exponent",
     cert(key=tlv(0x30, tlv(0x02, b"\x00\xc1" + b"\x11" * 15) + tlv(0x02, b"\x00"))), ST_OK, ST_PARSE_ERR,
     "crypto/x509 parsePublicKey: 'x509: RSA public exponent is not a positive number'; the path never decodes the "
     "subject's key (only the ISSUER's SubjectPublicKeyInfo bytes are hashed)"),
    ("rsa_key_that_is_not_a_sequence",
     cert(key=tlv(0x04, b"\x01\x02\x03")), ST_OK, ST_PARSE_ERR,
     "crypto/x509 parsePublicKey: asn1.Unmarshal into pkcs1PublicKey fails; key bytes are skipped here"),
    ("malformed_subject_alt_name",
     cert(extensions=[extension("0603551d11", b"\x01\x02\x03")]), ST_OK, ST_PARSE_ERR,
     "crypto/x509 parseSANExtension fails on a value that is not a SEQUENCE of GeneralName (ct-go keeps a usable certificate "
     "and reports a NonFatalError, which the worker still treats as a skip for precerts and issuers, ct-fetch.go:206-209,221-225); "
     "of the known extensions only basicConstraints and cRLDistributionPoints are decoded here"),
    ("malformed_key_usage",
     cert(extensions=[extension("0603551d0f", b"\x04\x00", critical=True)]), ST_OK, ST_PARSE_ERR,
     "crypto/x509: keyUsage must be a BIT STRING; not decoded here"),
    ("negative_serial_number",
     cert(serial=b"\x80\x01"), ST_OK, ST_PARSE_ERR,
     "crypto/x509: 'x509: negative serial number' (ct-go downgrades it to a NonFatalError: accepted for X.509 log entries, "
     "a skip for precertificates); raw serial octets are taken as they are here, like NewSerial does (storage/types.go:171-178)"),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_what_this_path_does_with_it_is_pinned(ora, case):
    _, der, ours, _, _ = case
    assert status_of(ora, der) == ours


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
@pytest.mark.xfail(strict=True, reason="ct-go / Go x509 behaviour not modelled (DESIGN.md §4); see the case's text")
def test_what_go_x509_does_with_it_is_not_modelled(ora, case):
    _, der, _, go, why = case
    assert status_of(ora, der) == go, why


def test_bmpstring_common_name_is_not_read_as_a_cn(ora):
    """BMPString (tag 0x1E) CommonNames: Go >= 1.14 decodes them, 1.13's encoding/asn1 does not know the tag; whether
    ct-go v1.1.0's asn1 fork does is unverifiable here.  This path treats the attribute as not-a-CN: the certificate parses,
    Issuer.CommonName is "" and an issuerCNFilter with non-empty prefixes filters it out.  Pinned so that a change is seen."""
    der = cert(issuer=name(0x1E, "Let's Encrypt".encode("utf-16-be")))
    assert status_of(ora, der) == ST_OK
    assert status_of(ora, der, flt=b"Let's Encrypt") == ST_FILTER_CN
