"""The Chain[0] hash model and the collision / SPKI builders of fe_model.py, on the CPU: the inverse of the mixer, the
crafted collisions, and SPKIs at every length across two SHA-256 block boundaries against the oracle and hashlib."""
import hashlib
import random

import pytest

import der_build as D
import fe_model as F


def test_inv_mix_inverts_fe_mix64():
    rng = random.Random(1)
    edges = [0, 1, 2, F.M64, F.M64 - 1, F.TOP, F.TOP - 1, 1 << 31, 1 << 32, (1 << 32) - 1, F.WORD_C, F.MIX_C1, F.MIX_C2]
    for x in edges + [rng.getrandbits(64) for _ in range(5000)]:
        assert F.inv_mix(F.fe_mix64(x)) == x
        assert F.fe_mix64(F.inv_mix(x)) == x


def test_hash_model_known_values():
    """Fixed values of the restated hash (pinned so that the model cannot drift with the code that uses it): the empty
    string, one byte, one word and a word and a byte -- the tail mask at 0, 1, 8 and 9 bytes."""
    assert F.chain0_hash(b"") == F.fe_mix64(0) | F.TOP
    assert F.chain0_hash(b"\x01") == F.fe_mix64(F.issuer_cert_word(1, 0) ^ (1 << 32)) | F.TOP
    w = int.from_bytes(b"ABCDEFGH", "little")
    assert F.chain0_hash(b"ABCDEFGH") == F.fe_mix64(F.issuer_cert_word(w, 0) ^ (8 << 32)) | F.TOP
    acc = (F.issuer_cert_word(w, 0) + F.issuer_cert_word(0x49, 1)) & F.M64
    assert F.chain0_hash(b"ABCDEFGHI") == F.fe_mix64(acc ^ (9 << 32)) | F.TOP
    # the zero padding of the last word is what the length term separates
    assert F.chain0_hash(b"AB") != F.chain0_hash(b"AB\x00")


@pytest.mark.parametrize("kind", F.PAIR_KINDS)
def test_crafted_pairs_collide(ora, kind):
    for salt in range(6):
        for length in (400, 601, 1203):
            a, b = F.colliding_pair(kind, salt, length)
            assert a != b and len(a) == len(b) == length
            assert F.chain0_hash(a) == F.chain0_hash(b)
            ra, ca = ora.parse_cert(a)
            rb, cb = ora.parse_cert(b)
            assert ra == 0
            spki_a = a[ca.spki_off:ca.spki_off + ca.spki_len]
            if kind == F.ONE_UNPARSEABLE:
                assert rb != 0
                continue
            assert rb == 0
            spki_b = b[cb.spki_off:cb.spki_off + cb.spki_len]
            assert (spki_a == spki_b) == (kind == F.SAME_SPKI)
            assert (ora.issuer_id(spki_a) == ora.issuer_id(spki_b)) == (kind == F.SAME_SPKI)


def test_crafted_targets_hit_their_bits():
    rng = random.Random(5)
    for k in range(20):
        t = F.TOP | rng.getrandbits(63)
        a, b = F.colliding_pair(F.PAIR_KINDS[k % 3], 10 + k, 500 + k, target=t)
        assert F.chain0_hash(a) == F.chain0_hash(b) == t
    for low16 in (0xFFFF, 0xFFFE, 0x0000, 0x003F):
        ders = F.clustered(12, low16, 520, salt=low16 & 7)
        assert len(set(ders)) == 12
        hs = [F.chain0_hash(d) for d in ders]
        assert len(set(hs)) == 12 and all(h & 0xFFFF == low16 and h >> 63 for h in hs)
        assert all(h % F.mirror_slots(16) == low16 % 64 for h in hs)


def test_cert_of_length_is_exact():
    for length in list(range(300, 420)) + [1000, 4095, 4096, 70000]:
        b = F.cert_of_length(length, **F._ca_kw(3, 0))
        assert len(b.der) == length


def test_spki_builder_covers_two_block_boundaries(ora):
    """Every SPKI length 50..140 (the SHA-256 padding splits at 55/56 and 119/120, block edges 64 and 128): the certificate
    parses, the span der_build marks is the SPKI, and the oracle's Issuer.ID digest is hashlib's.  130 is the one length
    no DER TLV has (a 128-byte body takes a 3-byte header, a 127-byte body a 2-byte one)."""
    with pytest.raises(ValueError):
        F.rsa_spki(130)
    for n in F.SPKI_LENGTHS:
        spki = F.rsa_spki(n)
        assert len(spki) == n
        b = F.ca(n, spki)
        assert F.spki_span(b) == spki
        rc, c = ora.parse_cert(b.der)
        assert rc == 0, n
        assert b.der[c.spki_off:c.spki_off + c.spki_len] == spki
        assert ora.issuer_id(spki)[0] == hashlib.sha256(spki).digest()
