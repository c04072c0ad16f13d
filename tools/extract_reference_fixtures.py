#!/usr/bin/env python3
"""Extract the reference's own test fixtures into tests/golden/ (run in the build container only).

The reference's Go tests embed three PEM certificates -- the only real-world DER in its tree:
    storage/types_test.go:21-39               kLeadingZeroes (serial 0x00AA, GeneralizedTime)
    storage/filesystemdatabase_test.go:17-33  kEmptySPKI     (CA:TRUE, UTF8 CN "ca")
    storage/filesystemdatabase_test.go:35-64  kRealSPKI      (UTCTime, 5-RDN PrintableString issuer, CRL-DP)
The reference is not part of this repository, so the PEMs (public certificates, test data) are copied
to tests/golden/*.pem and the values an independent implementation derives from them -- Python
hashlib + `cryptography`, NOT this repository's oracle -- are written to tests/golden/fixtures.json.
The Go tests' literal expectations (types_test.go:50,93,98 ...) are cited in tests/test_oracle_kat.py.
"""
import base64, hashlib, json, os, re, sys, warnings

from cryptography import x509
from cryptography.hazmat.primitives import serialization
from cryptography.x509.oid import ExtensionOID, NameOID

warnings.filterwarnings("ignore")
REF = sys.argv[1] if len(sys.argv) > 1 else sys.exit("usage: extract_reference_fixtures.py <reference checkout>")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
SRC = {
    "kLeadingZeroes": "storage/types_test.go",
    "kEmptySPKI": "storage/filesystemdatabase_test.go",
    "kRealSPKI": "storage/filesystemdatabase_test.go",
}


def main():
    os.makedirs(OUT, exist_ok=True)
    fx = {}
    for name, rel in SRC.items():
        text = open(os.path.join(REF, rel)).read()
        m = re.search(name + r"\s*=\s*`(-----BEGIN CERTIFICATE-----.*?-----END CERTIFICATE-----)`", text, re.S)
        assert m, name
        pem = m.group(1) + "\n"
        open(os.path.join(OUT, name + ".pem"), "w").write(pem)
        cert = x509.load_pem_x509_certificate(pem.encode())
        der = cert.public_bytes(serialization.Encoding.DER)
        spki = cert.public_key().public_bytes(serialization.Encoding.DER, serialization.PublicFormat.SubjectPublicKeyInfo)
        cns = cert.issuer.get_attributes_for_oid(NameOID.COMMON_NAME)
        try:
            bc = cert.extensions.get_extension_for_oid(ExtensionOID.BASIC_CONSTRAINTS).value
            bc_valid, is_ca = True, bool(bc.ca)
        except x509.ExtensionNotFound:
            bc_valid, is_ca = False, False
        crls = []
        try:
            for dp in cert.extensions.get_extension_for_oid(ExtensionOID.CRL_DISTRIBUTION_POINTS).value:
                for gn in dp.full_name or []:
                    crls.append(gn.value)
        except x509.ExtensionNotFound:
            pass
        # raw serial octets: locate the INTEGER inside the TBS by hand (cryptography only gives the int)
        tbs = cert.tbs_certificate_bytes
        off = 2 if tbs[1] < 0x80 else 2 + (tbs[1] & 0x7F)
        if tbs[off] == 0xA0:
            off += 2 + tbs[off + 1]
        assert tbs[off] == 0x02
        raw_serial = tbs[off + 2: off + 2 + tbs[off + 1]]
        fx[name] = {
            "source": rel,
            "der_len": len(der),
            "sha256_der": hashlib.sha256(der).hexdigest(),
            "spki_len": len(spki),
            "issuer_id_of_own_spki": base64.urlsafe_b64encode(hashlib.sha256(spki).digest()).decode(),
            "raw_serial_hex": raw_serial.hex(),
            "not_after_unix": int(cert.not_valid_after_utc.timestamp()),
            "not_before_unix": int(cert.not_valid_before_utc.timestamp()),
            "issuer_cn": cns[-1].value if cns else "",
            "bc_valid": bc_valid,
            "is_ca": is_ca,
            "crl_dps": crls,
        }
    json.dump(fx, open(os.path.join(OUT, "fixtures.json"), "w"), indent=1, sort_keys=True)
    print(json.dumps(fx, indent=1))


if __name__ == "__main__":
    sys.exit(main())
