"""Walker geometry: the streaming map kernel's DER walker (ctmr_stream.cuh) steps through a certificate in 128-byte
chunks with a 48-byte overlap, and four of its states exist only to resume an element that does not fit one step.
These tests build certificates that reach each of those states -- accepted and rejected -- and move every element
through all 128 phases of a chunk (a filler attribute of 256 + k bytes early in the issuer Name, k = 0..127) and all
16 record misalignments (pad records in front).  Both map kernels and the oracle see every input; the outputs must
agree bit for bit, the fingerprints must equal hashlib's, and status, serial span, expiry hour, filter outcomes and
metadata spans must equal what the builder wrote.

Whether an input really reaches a rare state is not left to chance: `rare_states()` restates the thresholds of
walk_advance, and a CPU test requires every state to be reached at every chunk phase by accepted and by rejected inputs.
"""
import hashlib

import numpy as np
import pytest

import der_build as D
from conftest import NOW_NS, pack

CHUNK = 128  # StreamCfg::kChunk (ctmr_common.cuh)
NEED = 48    # kWalkNeed (ctmr_stream.cuh)
ST_OK, ST_PARSE_ERR, ST_FILTER_CA, ST_FILTER_CN = 0, 1, 2, 4

CA = D.cert(serial=b"\x7f", subject=[[D.cn(b"Geometry CA")]], extensions=[D.basic_constraints(True)])
LONG_CN = bytes(0x41 + (i * 7) % 26 for i in range(300))


# ------------------------------------------------------------------------------------------------ the predicate

def runs_before_last_chunk(pos: int, L: int) -> bool:
    """W_NEED: a step at `pos` runs once pos + kWalkNeed bytes are staged, i.e. in the chunk that ends at
    roundup(pos + 48, 128); `final` (avail >= L) is false there exactly when that chunk ends before the record does."""
    return -(-(pos + NEED) // CHUNK) * CHUNK < L


def rare_states(b: D.Built) -> set:
    """{(state, pos % 128)} of the rare walker states this certificate enters, by the thresholds of walk_advance."""
    L, out = len(b.der), set()
    for who in ("issuer", "subject"):  # W_NAMEWALK: `if (!final && vp + 6u > w.pos + kWalkNeed)` -> W_ATV_VAL_FAR
        for pos, vp in zip(b.mark(who + "_atv"), b.mark(who + "_vp")):
            if vp + 6 > pos + NEED and runs_before_last_chunk(pos, L):
                out.add(("W_ATV_VAL_FAR", pos % CHUNK))
    pos, bp = b.mark("spki")[0], b.mark("spki_bits")[0]  # W_SPKI: `if (!final && bp + 6u > w.pos + kWalkNeed)`
    if bp + 6 > pos + NEED and runs_before_last_chunk(pos, L):
        out.add(("W_SPKI_BITS", pos % CHUNK))
    for pos, rest in zip(b.mark("ext"), b.mark("ext_rest")):  # W_EXTWALK: `if (!final && rest + 24u > w.pos + kWalkNeed)`
        if rest + 24 > pos + NEED and runs_before_last_chunk(pos, L):
            out.add(("W_EXT_REST", pos % CHUNK))
    pos, sp = b.mark("sigalg")[0], b.mark("sig")[0]  # W_TAIL: `if (!final && sp + 6u > w.pos + kWalkNeed)` -> W_SIG
    if sp + 6 > pos + NEED and runs_before_last_chunk(pos, L):
        out.add(("W_SIG", pos % CHUNK))
    return out


RARE = ("W_ATV_VAL_FAR", "W_SPKI_BITS", "W_EXT_REST", "W_SIG")

# ------------------------------------------------------------------------------------------------ the shapes
# (name, rejected?, knobs); each is built for k = 0..127 with `filler=256 + k` and a 300-byte signature, so that every
# element of interest lies before the record's last chunk.

LONG_EXT = D.Ext(D.long_oid(30), b"\x05\x00")
PSS_BITS = D.tlv(0x03, D.RSA_KEY_BITS)

SHAPES = [
    ("atv_far_issuer", False, dict(issuer=[[D.attr(D.long_oid(44), 0x0C, b"far value")], [D.cn(b"Geo CA")]])),
    ("atv_far_subject", False, dict(subject=[[D.attr(D.long_oid(60), 0x13, b"s")], [D.cn(b"leaf")]])),
    ("atv_far_multivalued", False, dict(issuer=[[D.cn(b"Geo"), D.attr(D.long_oid(50), 0x16, b"x"), D.cn(b"Last", 0x13)]])),
    ("spki_rsa_pss", False, dict(spki_alg=D.RSA_PSS)),
    ("spki_dsa", False, dict(spki_alg=D.dsa_alg(64, 20))),
    ("spki_ec_explicit", False, dict(spki_alg=D.ec_explicit_alg(), spki_bits=b"\x00\x04" + b"\x22" * 64)),
    ("ext_rest", False, dict(extensions=[LONG_EXT, D.crl_distribution_points(b"http://geo.example/crl"), D.basic_constraints(False)])),
    ("ext_rest_critical_then_ca", False, dict(extensions=[D.Ext(D.long_oid(22), b"\x30\x00", critical=True), D.basic_constraints(True)])),
    ("ext_rest_between_repeated_bc", False, dict(extensions=[D.basic_constraints(True), LONG_EXT, D.basic_constraints(False)])),
    ("sig_rsa_pss", False, dict(sig_alg=D.RSA_PSS, tbs_sig_alg=D.RSA_PSS)),
    ("all_rare_with_unique_ids", False, dict(issuer=[[D.attr(D.long_oid(44), 0x0C, b"v")], [D.cn(b"All")]], spki_alg=D.RSA_PSS,
                                             issuer_uid=b"\x01\x02", subject_uid=b"\x03", sig_alg=D.RSA_PSS,
                                             extensions=[D.Ext(D.long_oid(40), b"\x04\x01\x00", critical=False),
                                                         D.crl_distribution_points(b"ldap://geo.example/cn=crl")])),
    ("v1_ecdsa", False, dict(version=1, tbs_sig_alg=D.ECDSA_SHA256, sig_alg=D.ECDSA_SHA256, spki_alg=D.EC_P256,
                             spki_bits=b"\x00\x04" + b"\x11" * 64)),
    # rejected: the element the rare state reads is malformed
    ("atv_far_value_overruns", True, dict(issuer=[[D.attr(D.long_oid(44), 0x0C, b"value", value_hdr=b"\x0c\x06")], [D.cn(b"Geo CA")]])),
    ("atv_far_value_multibyte_tag", True, dict(subject=[[D.attr(D.long_oid(60), 0x13, b"s", value_hdr=b"\x1f\x01")]])),
    ("spki_bits_wrong_tag", True, dict(spki_alg=D.RSA_PSS, spki_bits_raw=D.tlv(0x04, D.RSA_KEY_BITS))),
    ("spki_bits_empty", True, dict(spki_alg=D.dsa_alg(64, 20), spki_bits_raw=b"\x03\x00")),
    ("spki_bits_overrun", True, dict(spki_alg=D.RSA_PSS, spki_bits_raw=PSS_BITS[:1] + bytes([PSS_BITS[1] + 1]) + PSS_BITS[2:])),
    ("ext_rest_bad_boolean", True, dict(extensions=[D.Ext(D.long_oid(30), b"\x05\x00", critical=b"\x01\x01\x01")])),
    ("ext_rest_long_boolean", True, dict(extensions=[D.Ext(D.long_oid(30), b"\x05\x00", critical=b"\x01\x02\xff\xff")])),
    ("ext_rest_value_not_octets", True, dict(extensions=[D.Ext(D.long_oid(30), b"\x05\x00", value_tag=0x05)])),
    ("sig_wrong_tag", True, dict(sig_alg=D.RSA_PSS, sig_raw=D.tlv(0x04, b"\x00" + b"\x5a" * 299))),
    ("sig_multibyte_tag", True, dict(sig_alg=D.RSA_PSS, sig_raw=D.tlv(0x1F, b"\x00" + b"\x5a" * 299))),
    ("sig_overrun", True, dict(sig_alg=D.RSA_PSS, sig_raw=D.hdr(0x03, 301) + b"\x00" + b"\x5a" * 299)),
]


def build_shape(i: int, k: int, knobs: dict) -> D.Built:
    kw = dict(serial=D.serial_bytes(8, salt=i * 131 + k), filler=256 + k, sig_len=300, extensions=None)
    kw.update(knobs)
    return D.cert(**kw)


def corpus():
    """[(shape name, rejected, k, Built)] over all shapes and k = 0..127."""
    return [(name, bad, k, build_shape(i, k, knobs)) for i, (name, bad, knobs) in enumerate(SHAPES) for k in range(128)]


def expected_status(b: D.Built, bad: bool, prefixes) -> int:
    if bad:
        return ST_PARSE_ERR
    if b.bc == D.BC_CA:
        return ST_FILTER_CA
    if prefixes and not any((b.cn or b"").startswith(p) for p in prefixes):
        return ST_FILTER_CN
    return ST_OK


def with_misalignments(ders, ms):
    """Entry list with a pad record (junk, rejected) in front of every certificate so that it starts at offset = m (mod 16).
    The host pipeline uploads a stage's records back to back from a 16-byte aligned buffer, so this is the record's
    misalignment on the device.  Returns (entries, positions of the certificates)."""
    out, where, off = [], [], 0
    for d, m in zip(ders, ms):
        p = (m - off) % 16
        out.append(b"\xff" * p)
        out.append(d)
        where.append(len(out) - 1)
        off += p + len(d)
    return out, np.array(where)


# ------------------------------------------------------------------------------------------------ coverage (CPU)

def test_corpus_reaches_every_rare_state_at_every_phase():
    pos_cov, neg_cov = {s: set() for s in RARE}, {s: set() for s in RARE}
    for name, bad, k, b in corpus():
        for st, ph in rare_states(b):
            (neg_cov if bad else pos_cov)[st].add(ph)
    for st in RARE:
        assert len(pos_cov[st]) == CHUNK, (st, "accepted", sorted(set(range(CHUNK)) - pos_cov[st])[:10])
        assert len(neg_cov[st]) == CHUNK, (st, "rejected", sorted(set(range(CHUNK)) - neg_cov[st])[:10])


def test_rejected_shapes_fail_only_at_their_rare_element(ora):
    """Each rejected shape is the accepted one with one element broken: the oracle rejects it, and the element the walker
    must reject it at is a rare state on every k."""
    for name, bad, k, b in corpus():
        if bad:
            assert ora.parse_cert(b.der)[0] != 0, (name, k)
            assert rare_states(b), (name, k)
        elif k % 37 == 0:
            assert ora.parse_cert(b.der)[0] == 0, (name, k)


def test_basic_constraints_never_reaches_w_ext_rest():
    """W_EXT_REST is entered only for an OID longer than 20 octets, and basicConstraints / cRLDistributionPoints are
    recognised only by a 3-octet OID: the rare path never decodes them.  Pinned so that a change of either threshold is
    seen here."""
    for pos_hdr in (2, 3, 4):  # Extension SEQUENCE header of 2, 3 or 4 octets
        rest = pos_hdr + 2 + 3  # + OID header + 2.5.29.x
        assert rest + 24 <= NEED


def long_cn_corpus():
    return [D.cert(serial=D.serial_bytes(8, salt=k), filler=256 + k, sig_len=300, issuer=[[D.cn(LONG_CN, 0x13)]])
            for k in range(128)]


def test_long_cn_prefixes_are_compared_past_the_staged_window():
    """The differing byte of a filter prefix lies beyond the bytes staged when the CN's attribute is walked (the global
    memory path of w_note_cn) for every prefix length used below, and before it for some."""
    far = {d: 0 for d in (40, 127, 200)}
    near = {d: 0 for d in (40, 127, 200)}
    for b in long_cn_corpus():
        pos, c0 = b.mark("issuer_atv")[-1], b.mark("issuer_cn")[-1]
        avail = min(-(-(pos + NEED) // CHUNK) * CHUNK, len(b.der))
        for d in far:
            if c0 + d >= avail:
                far[d] += 1
            else:
                near[d] += 1
    assert all(far.values()) and near[40] and near[127], (far, near)


# ------------------------------------------------------------------------------------------------ the GPU runs

@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def _run_both_kernels(eng, ora, entries, flt):
    from test_gpu_parity import assert_same
    blob, offs = pack(entries)
    iblob, ioffs = pack([CA.der])
    idx = np.zeros(len(entries), np.uint32)
    want = ora.DB(flt, True).process(blob, offs, iblob, ioffs, idx, NOW_NS)
    got = {}
    for want_sha in (True, False):  # map_stream_kernel, then map_light_kernel
        with eng.GpuCertDatabase(issuer_cn_filter=flt, log_expired_entries=True, table_capacity=1 << 16) as db:
            r = db.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS, want_sha=want_sha, want_meta=True)
        assert_same(r, want, sha=want_sha)
        parsed = want.status != ST_PARSE_ERR
        for f in ("issuer_name_off", "issuer_name_len", "crldp_off", "crldp_len"):
            assert np.array_equal(getattr(r, f)[parsed], getattr(want, f)[parsed]), (want_sha, f)
        for f in ("first_issuer_dn", "first_crldp"):
            assert np.array_equal(getattr(r, f), getattr(want, f)), (want_sha, f)
        got[want_sha] = r
    for i, d in enumerate(entries):
        assert got[True].sha256[i].tobytes() == hashlib.sha256(d).digest(), i
    return got


def _check_truth(r, where, items, prefixes, tag):
    for j, (name, bad, k, b) in enumerate(items):
        i = int(where[j])
        st = expected_status(b, bad, prefixes)
        assert int(r.status[i]) == st, (tag, name, k, int(r.status[i]), st)
        if bad:
            continue
        assert int(r.serial_off[i]) == b.mark("serial")[0] and int(r.serial_len[i]) == len(b.serial), (tag, name, k)
        assert int(r.exp_hour[i]) == D.exp_hour(b.not_after), (tag, name, k)
        assert (int(r.issuer_name_off[i]), int(r.issuer_name_len[i])) == b.issuer, (tag, name, k)
        assert (int(r.crldp_off[i]), int(r.crldp_len[i])) == b.crldp, (tag, name, k)


@pytest.mark.gpu
def test_rare_states_at_every_phase_and_misalignment(eng, ora):
    items = corpus()
    # accepted shapes at all 16 misalignments, rejected ones at one each
    rows = [(it, m) for it in items for m in (range(16) if not it[1] else (it[2] % 16,))]
    entries, where = with_misalignments([it[3].der for it, _ in rows], [m for _, m in rows])
    got = _run_both_kernels(eng, ora, entries, b"")
    for want_sha, r in got.items():
        _check_truth(r, where, [it for it, _ in rows], (), "stream" if want_sha else "light")


@pytest.mark.gpu
@pytest.mark.parametrize("d", (40, 127, 200))
def test_long_cn_filter_prefixes(eng, ora, d):
    """An issuer CN of 300 bytes against prefixes that agree with it up to byte d and then agree (kept) or differ
    (filtered); the differing byte lies beyond the staged window for most phases."""
    certs = long_cn_corpus()
    items = [("long_cn", False, k, b) for k, b in enumerate(certs)]
    entries, where = with_misalignments([b.der for b in certs], [k % 16 for k in range(len(certs))])
    match, miss = LONG_CN[:d + 1], LONG_CN[:d] + bytes([LONG_CN[d] ^ 0x20])
    for prefixes in ((match,), (miss,), (miss, match)):
        got = _run_both_kernels(eng, ora, entries, b",".join(prefixes))
        for want_sha, r in got.items():
            _check_truth(r, where, items, prefixes, ("stream" if want_sha else "light", d, len(prefixes)))
