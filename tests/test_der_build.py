"""tests/der_build.py against two references: the oracle (every field of the builder's truth) and the `cryptography`
package (wherever it loads the certificate).  The GPU tests take the builder's truth as the expected value, so the
builder itself has to be right first."""
import datetime
import warnings

import pytest
from cryptography import x509
from cryptography.x509.oid import ExtensionOID, NameOID

import der_build as D

warnings.filterwarnings("ignore")


def _catalogue():
    """(id, Built) over the builder's knobs."""
    out = []
    add = lambda name, **kw: out.append((name, D.cert(**kw)))
    add("default")
    add("v1_no_extensions", version=1)
    add("unique_ids", issuer_uid=b"\x11\x22", subject_uid=b"\x33", extensions=[D.basic_constraints(False)])
    add("issuer_uid_only", issuer_uid=b"\x44" * 9, extensions=[D.crl_distribution_points(b"http://c.example/1.crl")])
    add("subject_uid_only_v1", version=1, subject_uid=b"\x55")
    add("multi_valued_rdn_last_cn_wins", issuer=[[D.cn(b"first"), D.attr(D.O_OID, 0x13, b"Org")], [D.cn(b"second", 0x13)]])
    add("cn_then_bmp_cn", issuer=[[D.cn(b"visible")], [D.cn("hidden".encode("utf-16-be"), D.BMP_STRING)]])
    add("only_bmp_cn", issuer=[[D.cn("bmp".encode("utf-16-be"), D.BMP_STRING)]])
    add("no_cn", issuer=[[D.attr(D.O_OID, 0x0C, b"No CN Org")]])
    for tag in D.CN_STRING_TAGS:
        add("cn_tag_%02x" % tag, issuer=[[D.cn(b"12345" if tag == 0x12 else b"Tag CA", tag)]])
    for n in (1, 40, 127, 128, 200, 255, 256, 300):
        add("cn_%d_bytes" % n, issuer=[[D.cn(bytes(0x41 + i % 26 for i in range(n)))]])
    add("long_oid_in_issuer", issuer=[[D.attr(D.long_oid(45), 0x0C, b"v")], [D.cn(b"after long oid")]])
    add("long_oid_in_subject", subject=[[D.attr(D.long_oid(60), 0x13, b"w")]])
    add("long_oid_extension", extensions=[D.Ext(D.long_oid(30), b"\x05\x00"), D.basic_constraints(True)])
    add("long_oid_extension_critical", extensions=[D.Ext(D.long_oid(25), b"\x04\x00", critical=True)])
    add("rsa_pss_everywhere", tbs_sig_alg=D.RSA_PSS, spki_alg=D.RSA_PSS, sig_alg=D.RSA_PSS, sig_len=300)
    add("ecdsa", tbs_sig_alg=D.ECDSA_SHA256, spki_alg=D.EC_P256, spki_bits=b"\x00\x04" + b"\x11" * 64, sig_alg=D.ECDSA_SHA256)
    add("dsa_spki", spki_alg=D.dsa_alg())
    add("ec_explicit_spki", spki_alg=D.ec_explicit_alg(), spki_bits=b"\x00\x04" + b"\x22" * 64)
    add("critical_crldp", extensions=[D.Ext(D.CRLDP_OID, D.crl_distribution_points(b"http://x/y").value, critical=True)])
    add("bc_ca_true", extensions=[D.basic_constraints(True, pathlen=0)])
    add("bc_ca_false_noncritical", extensions=[D.basic_constraints(False, critical=False)])
    add("bc_repeated_later_wins_ca", extensions=[D.basic_constraints(False), D.key_usage(), D.basic_constraints(True)])
    add("bc_repeated_later_wins_not_ca", extensions=[D.basic_constraints(True), D.basic_constraints(False)])
    for n in (1, 2, 20, 38, 39, 40, 41):
        add("serial_%d" % n, serial=D.serial_bytes(n, salt=n))
        if n >= 2:
            add("serial_%d_lead00" % n, serial=D.serial_bytes(n, lead00=True, salt=n))
    for k in (0, 1, 63, 127):
        add("filler_%d" % k, filler=k, extensions=[D.crl_distribution_points(b"http://f/%d" % k)])
    for na in (D.unix(1960, 3, 1, 5, 59, 59), D.unix(1969, 12, 31, 23, 0, 0), D.unix(2049, 12, 31, 23, 59, 59),
               D.unix(2050, 1, 1), D.unix(9999, 12, 31, 23, 59, 59)):
        add("not_after_%d" % na, not_after=na)
    add("signature_600", sig_len=600)
    return out


CATALOGUE = _catalogue()


def _cn_of(cert):
    """Last CommonName whose value is a string type the path reads (not BMPString), per `cryptography`."""
    vals = [a for a in cert.issuer.get_attributes_for_oid(NameOID.COMMON_NAME)
            if a._type != x509.name._ASN1Type.BMPString]
    return vals[-1].value.encode() if vals else None


@pytest.mark.parametrize("name,b", CATALOGUE, ids=[c[0] for c in CATALOGUE])
def test_builder_truth_matches_the_oracle(ora, name, b):
    rc, c = ora.parse_cert(b.der)
    assert rc == 0
    d = b.der
    assert d[c.serial_off:c.serial_off + c.serial_len] == b.serial
    assert c.serial_off == b.mark("serial")[0]
    assert c.not_after == b.not_after
    assert (c.issuer_off, c.issuer_len) == b.issuer
    assert (c.crldp_off, c.crldp_len) == b.crldp
    assert bool(c.has_cn) == (b.cn is not None)
    if b.cn is not None:
        assert d[c.cn_off:c.cn_off + c.cn_len] == b.cn and c.cn_off == b.mark("issuer_cn")[-1]
    assert (c.bc_valid, c.is_ca) == {D.BC_ABSENT: (0, 0), D.BC_NOT_CA: (1, 0), D.BC_CA: (1, 1)}[b.bc]
    assert c.spki_off == b.mark("spki")[0]


@pytest.mark.parametrize("name,b", CATALOGUE, ids=[c[0] for c in CATALOGUE])
def test_builder_truth_matches_cryptography(name, b):
    try:
        cert = x509.load_der_x509_certificate(b.der)
        serial = cert.serial_number
    except ValueError:
        pytest.skip("cryptography does not load this shape")
    assert serial == int.from_bytes(b.serial, "big")
    assert int(cert.not_valid_after_utc.timestamp()) == b.not_after
    a, l = b.issuer
    assert b.der[a:a + l] == cert.issuer.public_bytes()
    try:
        cn = _cn_of(cert)
    except ValueError:
        cn = b.cn  # a value cryptography refuses to decode (e.g. a CN of the wrong string type): nothing to compare
    assert cn == b.cn
    try:
        exts = cert.extensions
    except (ValueError, x509.DuplicateExtension):  # duplicates: RFC 5280 forbids them, Go's x509 takes the last
        return
    try:
        bc = exts.get_extension_for_oid(ExtensionOID.BASIC_CONSTRAINTS).value
        assert b.bc == (D.BC_CA if bc.ca else D.BC_NOT_CA)
    except x509.ExtensionNotFound:
        assert b.bc == D.BC_ABSENT
    try:
        dp = exts.get_extension_for_oid(ExtensionOID.CRL_DISTRIBUTION_POINTS).value
        a, l = b.crldp
        assert l and dp[0].full_name[0].value.encode() in b.der[a:a + l]
    except x509.ExtensionNotFound:
        assert b.crldp == (0, 0)


def test_cryptography_loads_most_of_the_catalogue():
    """The second reference is not vacuous: it loads the bulk of the shapes."""
    loaded = 0
    for _, b in CATALOGUE:
        try:
            x509.load_der_x509_certificate(b.der).serial_number
            loaded += 1
        except ValueError:
            pass
    assert loaded >= len(CATALOGUE) * 3 // 4


def test_filler_shifts_every_later_element_by_k():
    """A filler of 256 + k bytes keeps every enclosing length in its two-octet form, so the later elements move by
    exactly k, and over k = 0..127 each of them meets every phase of a 128-byte chunk."""
    base = D.cert(filler=256)
    phases = {"spki": set(), "sig": set(), "issuer_cn": set()}
    for k in range(128):
        b = D.cert(filler=256 + k)
        assert b.issuer[0] == base.issuer[0]
        for m in phases:
            assert b.mark(m)[-1] - base.mark(m)[-1] == k, (m, k)
            phases[m].add(b.mark(m)[-1] % 128)
    assert all(len(v) == 128 for v in phases.values())


def test_not_after_before_1970_is_floored_to_the_hour(ora):
    na = D.unix(1969, 12, 31, 22, 30, 0)
    b = D.cert(not_after=na)
    rc, c = ora.parse_cert(b.der)
    assert rc == 0 and c.not_after == na < 0
    assert D.exp_hour(na) == -2 == ora.exp_hour(na)
    assert datetime.datetime(1970, 1, 1) + datetime.timedelta(hours=D.exp_hour(na)) == datetime.datetime(1969, 12, 31, 22)
