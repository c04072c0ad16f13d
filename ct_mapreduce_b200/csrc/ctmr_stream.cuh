// ctmr_stream.cuh -- resumable DER walker for the streaming map kernel.
//
// The v1 kernel walked the TLV tree with byte loads from global memory; with ~210 KB of shared
// memory carved out per SM the remaining L1 (~45 KB) thrashes under 384 lanes each touching its
// own lines, and the walk stalls on global loads.  This walker
// instead consumes the certificate from the SAME shared-memory chunks the SHA-256 loop streams
// through, so every certificate byte crosses L2->SM exactly once, by an asynchronous copy.
//
// It is a flat state machine (one switch in a loop) rather than recursive descent: a lane can
// suspend between any two TLV headers when it runs out of staged bytes and resume when the next
// chunk has landed.  Every state reads at most kNeed bytes from `pos`, and a step only runs when
// those bytes are staged (or the record is complete), so reads never leave the window.
//
// Fields extracted = what the reference worker reads from ct-go's x509.Certificate (SURVEY.md
// §8(a) a3); acceptance rules = Go encoding/asn1 as restated in oracle/ctmr_oracle.c -- the two
// implementations are deliberately structured differently (nested loops there, states here).
#pragma once
#include "ctmr_device.cuh"
#include "ctmr_kernels.cuh"

namespace ctmr {

enum WalkState : uint32_t {
    W_HEAD = 0,     // Certificate + TBSCertificate headers, optional [0] version
    W_SERIAL,       // serialNumber (captured)
    W_SIGALG,       // signature AlgorithmIdentifier (skipped)
    W_NAME,         // issuer / subject Name header
    W_NAMEWALK,     // SET OF { SEQ { OID, value } } ... loops inside the state
    W_ATV_VAL_FAR,  // value header of an attribute whose OID was too long for one window (rare)
    W_VALIDITY,     // both times in one step
    W_SPKI,         // SubjectPublicKeyInfo: SEQ { AlgorithmIdentifier, BIT STRING }
    W_SPKI_BITS,    // ... the BIT STRING header when the AlgorithmIdentifier was long (rare)
    W_OPT,          // [1] issuerUniqueID, [2] subjectUniqueID, [3] extensions + their SEQUENCE header
    W_EXTWALK,      // Extension ... loops inside the state, basicConstraints decoded inline
    W_EXT_REST,     // critical / extnValue of an extension whose OID was too long for one window (rare)
    W_TAIL,         // signatureAlgorithm + signatureValue headers
    W_SIG,          // ... signatureValue header alone when the AlgorithmIdentifier was long (rare)
    W_DONE, W_ERR
};

enum : uint32_t {
    WF_HAS_CN = 1u, WF_BC_VALID = 2u, WF_IS_CA = 4u, WF_IN_SUBJECT = 8u, WF_IS_CN_OID = 16u, WF_CN_MATCH = 32u,
    WF_BC_CA_TMP = 64u
};

struct Walker {
    uint32_t pos, st, flags;
    uint32_t end_tbs, end_b, end_c, end_d;  // tbs | name or extensions | set, validity, spki or extension | atv or bc value
    uint32_t which;                          // last arc of a 2.5.29.x extension OID, 0 otherwise
    uint32_t serial_off, serial_len;
    uint32_t name_off, name_len;    // issuer Name, full TLV
    uint32_t crldp_off, crldp_len;  // cRLDistributionPoints extnValue content
    int64_t not_after;

    __device__ __forceinline__ void init() {
        pos = 0; st = W_HEAD; flags = 0; end_tbs = end_b = end_c = end_d = 0; which = 0;
        serial_off = serial_len = 0; not_after = 0;
        name_off = name_len = crldp_off = crldp_len = 0;
    }
};

constexpr uint32_t kWalkNeed = 48;  // most bytes any single state reads from `pos` (W_SERIAL: 6 + 39)

// Byte x of the record, read from the lane's shared-memory ring: record offset x sits at ring offset (x + m) mod
// kRingBytes, where `ring` is the ring's 32-bit shared-space address and m the record's misalignment.  A read never
// leaves the ring; only staged offsets are ever used.
constexpr uint32_t kRingBytes = 256;  // StreamCfg::kRing

struct SmemWindow {
    uint32_t ring, m;
    __device__ __forceinline__ uint32_t at(uint32_t x) const { return ring + ((x + m) & (kRingBytes - 1u)); }
    __device__ __forceinline__ uint32_t operator()(uint32_t x) const {
        uint32_t v;
        asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(at(x)));
        return v;
    }
};

// TLV header at `pos` inside [pos, lim): Go parseTagAndLength rules (single-octet tag, definite
// minimal length, value inside the container).  Deliberately NOT inlined: the walker has ~30 call
// sites and the map kernel's instruction footprint is what the SHA loop competes with for I-cache.
static __device__ __noinline__ uint64_t w_hdr_packed(SmemWindow rd, uint32_t pos, uint32_t lim) {
    constexpr uint64_t kFail = ~0ull;
    if (pos + 2u > lim) return kFail;
    // the four bytes at `pos` in one go: two aligned 32-bit shared loads + a funnel shift
    // (tag | len0 << 8 | len1 << 16 | len2 << 24); each word's ring offset is masked on its own, so the
    // second one wraps to the ring's start where the first one ends at the ring's end
    const uint32_t a = pos + rd.m;
    uint32_t lo, hi;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(lo) : "r"(rd.ring + (a & (kRingBytes - 4u))));
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(hi) : "r"(rd.ring + ((a + 4u) & (kRingBytes - 4u))));
    const uint32_t v = __funnelshift_r(lo, hi, (a & 3u) * 8u);
    const uint32_t tag = v & 0xffu, l = (v >> 8) & 0xffu;
    if ((tag & 0x1fu) == 0x1fu) return kFail;
    uint32_t hdr, len;
    if (l < 0x80u) {
        hdr = 2;
        len = l;
    } else {
        const uint32_t nb = l & 0x7fu;
        if (nb == 0u || nb > 4u || pos + 2u + nb > lim) return kFail;
        if (nb == 1u) {
            len = (v >> 16) & 0xffu;
            if (len < 0x80u) return kFail;  // non-minimal (covers the leading-zero rule too)
        } else if (nb == 2u) {
            len = ((v >> 8) & 0xff00u) | (v >> 24);
            if (len < 0x100u) return kFail;  // superfluous leading zero
        } else {  // 3 or 4 length octets: certificates of 64 KiB and more, byte by byte
            len = 0;
            for (uint32_t i = 0; i < nb; ++i) {
                if (len >= (1u << 23)) return kFail;
                len = (len << 8) | rd(pos + 2u + i);
                if (len == 0u) return kFail;
            }
            if (len < 0x80u) return kFail;
        }
        hdr = 2u + nb;
    }
    if (len > lim - pos - hdr) return kFail;
    return ((uint64_t)len << 32) | (hdr << 8) | tag;  // registers only: no out-parameter, no stack
}

__device__ __forceinline__ bool w_hdr(SmemWindow rd, uint32_t pos, uint32_t lim, Tlv& t) {
    const uint64_t r = w_hdr_packed(rd, pos, lim);
    t.tag = (uint32_t)r & 0xffu;
    t.hdr = ((uint32_t)r >> 8) & 0xffu;
    t.len = (uint32_t)(r >> 32);
    return r != ~0ull;
}

template <class R>
__device__ __forceinline__ bool w_2d(const R& rd, uint32_t p, uint32_t& v) {
    const uint32_t a = rd(p) - (uint32_t)'0', b = rd(p + 1) - (uint32_t)'0';
    v = a * 10u + b;
    return a <= 9u && b <= 9u;
}

// UTCTime / GeneralizedTime content at cert offset p (same acceptance rules as der_time)
constexpr int64_t kBadTime = INT64_MIN;

template <class R>
__device__ __noinline__ int64_t w_time_raw(const R rd, uint32_t tag, uint32_t p, uint32_t len) {
    uint32_t yy, cc, mo, dd, hh, mi, ss = 0, pos;
    int64_t year;
    if (tag == 0x18u) {
        if (len < 15u || !w_2d(rd, p, cc) || !w_2d(rd, p + 2, yy)) return kBadTime;
        year = (int64_t)cc * 100 + yy;
        pos = 4;
    } else if (tag == 0x17u) {
        if (len < 11u || !w_2d(rd, p, yy)) return kBadTime;
        year = yy >= 50u ? 1900 + (int64_t)yy : 2000 + (int64_t)yy;
        pos = 2;
    } else {
        return kBadTime;
    }
    if (len > 19u) return kBadTime;  // longest legal form is YYYYMMDDhhmmss+hhmm
    if (!w_2d(rd, p + pos, mo) || !w_2d(rd, p + pos + 2, dd) || !w_2d(rd, p + pos + 4, hh) || !w_2d(rd, p + pos + 6, mi))
        return kBadTime;
    pos += 8;
    bool has_sec = false;
    if (pos + 2u <= len) {
        const uint32_t c0 = rd(p + pos);
        if (c0 >= '0' && c0 <= '9') {
            if (!w_2d(rd, p + pos, ss)) return kBadTime;
            pos += 2;
            has_sec = true;
        }
    }
    if (tag == 0x18u && !has_sec) return kBadTime;
    if (pos >= len) return kBadTime;
    int64_t off = 0;
    const uint32_t z = rd(p + pos);
    if (z == 'Z') {
        if (pos + 1u != len) return kBadTime;
    } else if (z == '+' || z == '-') {
        uint32_t oh, om;
        if (pos + 5u != len || !w_2d(rd, p + pos + 1, oh) || !w_2d(rd, p + pos + 3, om)) return kBadTime;
        if (oh > 23u || om > 59u) return kBadTime;
        off = (int64_t)oh * 3600 + (int64_t)om * 60;
        if (off == 0) return kBadTime;
        if (z == '-') off = -off;
    } else {
        return kBadTime;
    }
    if (mo < 1u || mo > 12u || dd < 1u || hh > 23u || mi > 59u || ss > 59u) return kBadTime;
    uint32_t maxd = (mo == 2u) ? 28u : ((0xAD5u >> (mo - 1u)) & 1u ? 31u : 30u);
    if (mo == 2u && (year % 4 == 0) && (year % 100 != 0 || year % 400 == 0)) maxd = 29u;
    if (dd > maxd) return kBadTime;
    return days_from_civil(year, mo, dd) * 86400 + (int64_t)hh * 3600 + (int64_t)mi * 60 + (int64_t)ss - off;
}

template <class R>
__device__ __forceinline__ bool w_time(const R rd, uint32_t tag, uint32_t p, uint32_t len, int64_t& out) {
    const int64_t v = w_time_raw(rd, tag, p, len);
    if (v == kBadTime) return false;
    out = v;
    return true;
}

// basicConstraints ::= SEQUENCE { cA BOOLEAN DEFAULT FALSE, pathLenConstraint INTEGER OPTIONAL } filling
// exactly the extnValue [vp, ve); "trailing data" and malformed members are errors (Go x509).
template <class R>
__device__ __forceinline__ bool w_basic_constraints(Walker& w, const R& rd, uint32_t vp, uint32_t ve) {
    Tlv bc, f;
    if (!w_hdr(rd, vp, ve, bc) || bc.tag != 0x30u || vp + bc.hdr + bc.len != ve) return false;
    uint32_t bp = vp + bc.hdr;
    bool ca = false;
    if (bp < ve) {
        if (!w_hdr(rd, bp, ve, f)) return false;
        if (f.tag == 0x01u) {
            if (f.len != 1u) return false;
            const uint32_t bv = rd(bp + f.hdr);
            if (bv != 0x00u && bv != 0xffu) return false;
            ca = bv != 0u;
            bp += f.hdr + f.len;
            if (bp < ve && !w_hdr(rd, bp, ve, f)) return false;
        }
        if (bp < ve && (f.tag != 0x02u || f.len == 0u)) return false;
    }
    w.flags |= WF_BC_VALID;  // a later basicConstraints overrides an earlier one
    w.flags = ca ? (w.flags | WF_IS_CA) : (w.flags & ~WF_IS_CA);
    return true;
}

// critical BOOLEAN DEFAULT FALSE + extnValue OCTET STRING of the extension ending at `ee`, starting at `ip`
template <class R>
__device__ __forceinline__ bool w_ext_rest(Walker& w, const R& rd, uint32_t ip, uint32_t ee) {
    Tlv v;
    if (!w_hdr(rd, ip, ee, v)) return false;
    if (v.tag == 0x01u) {
        if (v.len != 1u) return false;
        const uint32_t bv = rd(ip + v.hdr);
        if (bv != 0x00u && bv != 0xffu) return false;
        ip += v.hdr + v.len;
        if (!w_hdr(rd, ip, ee, v)) return false;
    }
    if (v.tag != 0x04u) return false;
    const uint32_t vp = ip + v.hdr;
    if (w.which == 0x13u) return w_basic_constraints(w, rd, vp, vp + v.len);
    if (w.which == 0x1fu) { w.crldp_off = vp; w.crldp_len = v.len; }  // cRLDistributionPoints
    return true;
}

// Issuer.CommonName = the last 2.5.4.3 value of a string type; the issuerCNFilter prefixes are
// evaluated right here, while the bytes are in shared memory (ct-fetch.go:57-63).
template <class R, class F>
__device__ __forceinline__ void w_note_cn(Walker& w, const R& rd, const F& far, uint32_t avail, uint32_t c0, uint32_t cnl,
                                          const FilterCfg& flt) {
    bool match = false;
    for (uint32_t q = 0; q < flt.n_prefix && !match; ++q) {
        const uint32_t po = flt.off[q], pl = flt.off[q + 1] - po;
        if (pl > cnl) continue;
        bool eq = true;
        for (uint32_t i = 0; i < pl; ++i) {
            const uint32_t x = c0 + i;
            const uint32_t b = x < avail ? rd(x) : far(x);
            if (b != flt.bytes[po + i]) { eq = false; break; }
        }
        match = eq;
    }
    w.flags |= WF_HAS_CN;
    w.flags = match ? (w.flags | WF_CN_MATCH) : (w.flags & ~WF_CN_MATCH);
}

// Runs the walker as far as the staged bytes allow.
//   rd(x)      byte x of the record from the shared-memory window (valid for x < avail)
//   far(x)     byte x from global memory (only for a CommonName running past the window)
//   avail      record bytes staged so far; avail >= L means the whole record has been seen
//   key_words  where the raw serial goes when it is met (10 words: len | serial[39], zero padded)
// A state may loop over several TLVs; before every header it reads it makes sure kWalkNeed bytes from
// `pos` are staged (or the record is complete) and otherwise returns with (st, pos, end_*) describing
// exactly where to resume.  No single TLV step reads further than kWalkNeed bytes from its `pos`.
template <class R, class F>
__device__ inline void walk_advance(Walker& w, const R& rd, const F& far, uint32_t avail, uint32_t L,
                                    const FilterCfg& flt, uint32_t* __restrict__ key_words) {
    const bool final = avail >= L;
#define W_NEED()                                              \
    if (!final && w.pos + kWalkNeed > avail) return /* suspend until the next chunk lands */
#define W_FAIL()         \
    {                    \
        w.st = W_ERR;    \
        return;          \
    }
    Tlv t;
    for (;;) {
        switch (w.st) {
        case W_HEAD: {
            W_NEED();
            Tlv tbs;
            if (!w_hdr(rd, 0, L, t) || t.tag != 0x30u || t.hdr + t.len != L) W_FAIL();
            uint32_t p = t.hdr;
            if (!w_hdr(rd, p, L, tbs) || tbs.tag != 0x30u) W_FAIL();
            p += tbs.hdr;
            w.end_tbs = p + tbs.len;
            if (!w_hdr(rd, p, w.end_tbs, t)) W_FAIL();
            if (t.tag == 0xa0u) p += t.hdr + t.len;  // [0] EXPLICIT version
            w.pos = p;
            w.st = W_SERIAL;
            break;
        }
        case W_SERIAL: {  // raw content octets, leading zeros kept (storage/types.go:171-178)
            W_NEED();
            if (!w_hdr(rd, w.pos, w.end_tbs, t) || t.tag != 0x02u || t.len == 0u) W_FAIL();
            const uint32_t c0 = w.pos + t.hdr;
            if (t.len > 1u) {
                const uint32_t b0 = rd(c0), b1 = rd(c0 + 1);
                if ((b0 == 0x00u && (b1 & 0x80u) == 0u) || (b0 == 0xffu && (b1 & 0x80u) != 0u)) W_FAIL();
            }
            w.serial_off = c0;
            w.serial_len = t.len;
            if (key_words != nullptr) {  // {len, serial[39]} zero padded = words 4..13 of the key record
                const uint32_t n = t.len < CTMR_MAX_SERIAL ? t.len : CTMR_MAX_SERIAL;
#pragma unroll 1
                for (uint32_t wi = 0; wi < 10u; ++wi) {
                    uint32_t v = 0;
#pragma unroll
                    for (uint32_t k = 0; k < 4u; ++k) {
                        const uint32_t i = 4u * wi + k;  // byte i of {len, serial...}
                        const uint32_t b = i == 0u ? n : (i - 1u < n ? rd(c0 + i - 1u) : 0u);
                        v |= b << (8u * k);
                    }
                    key_words[wi] = v;
                }
            }
            w.pos = c0 + t.len;
            w.st = W_SIGALG;
            break;
        }
        case W_SIGALG:
            W_NEED();
            if (!w_hdr(rd, w.pos, w.end_tbs, t) || t.tag != 0x30u) W_FAIL();
            w.pos += t.hdr + t.len;
            w.st = W_NAME;
            break;
        case W_NAME:  // issuer, then (WF_IN_SUBJECT) subject
            W_NEED();
            if (!w_hdr(rd, w.pos, w.end_tbs, t) || t.tag != 0x30u) W_FAIL();
            if (!(w.flags & WF_IN_SUBJECT)) { w.name_off = w.pos; w.name_len = t.hdr + t.len; }
            w.pos += t.hdr;
            w.end_b = w.pos + t.len;
            w.end_c = 0;  // no SET open
            w.st = W_NAMEWALK;
            break;
        case W_NAMEWALK:
            for (;;) {
                if (w.pos >= w.end_b) {
                    w.st = (w.flags & WF_IN_SUBJECT) ? W_SPKI : W_VALIDITY;
                    break;
                }
                W_NEED();
                if (w.pos >= w.end_c) {  // next RelativeDistinguishedName
                    if (!w_hdr(rd, w.pos, w.end_b, t) || t.tag != 0x31u) W_FAIL();
                    w.pos += t.hdr;
                    w.end_c = w.pos + t.len;
                    continue;
                }
                Tlv oid;
                if (!w_hdr(rd, w.pos, w.end_c, t) || t.tag != 0x30u) W_FAIL();  // AttributeTypeAndValue
                const uint32_t ap = w.pos + t.hdr, ae = ap + t.len;
                if (!w_hdr(rd, ap, ae, oid) || oid.tag != 0x06u) W_FAIL();
                const uint32_t o = ap + oid.hdr, vp = o + oid.len;
                w.flags &= ~WF_IS_CN_OID;
                if (!(w.flags & WF_IN_SUBJECT) && oid.len == 3u && rd(o) == 0x55u && rd(o + 1) == 0x04u && rd(o + 2) == 0x03u)
                    w.flags |= WF_IS_CN_OID;
                if (!final && vp + 6u > w.pos + kWalkNeed) {  // unusually long OID: value header in its own step
                    w.end_d = ae;
                    w.pos = vp;
                    w.st = W_ATV_VAL_FAR;
                    break;
                }
                Tlv val;
                if (!w_hdr(rd, vp, ae, val)) W_FAIL();
                if ((w.flags & WF_IS_CN_OID) &&
                    (val.tag == 0x0cu || val.tag == 0x13u || val.tag == 0x16u || val.tag == 0x14u || val.tag == 0x12u))
                    w_note_cn(w, rd, far, avail, vp + val.hdr, val.len, flt);
                w.pos = ae;
            }
            break;
        case W_ATV_VAL_FAR:
            W_NEED();
            if (!w_hdr(rd, w.pos, w.end_d, t)) W_FAIL();
            w.pos = w.end_d;
            w.st = W_NAMEWALK;
            break;
        case W_VALIDITY: {
            W_NEED();
            Tlv a, b;
            int64_t nb;
            if (!w_hdr(rd, w.pos, w.end_tbs, t) || t.tag != 0x30u) W_FAIL();
            uint32_t vp = w.pos + t.hdr;
            const uint32_t ve = vp + t.len;
            if (!w_hdr(rd, vp, ve, a) || !w_time(rd, a.tag, vp + a.hdr, a.len, nb)) W_FAIL();
            vp += a.hdr + a.len;
            if (!w_hdr(rd, vp, ve, b) || !w_time(rd, b.tag, vp + b.hdr, b.len, w.not_after)) W_FAIL();
            w.pos = ve;
            w.flags |= WF_IN_SUBJECT;
            w.st = W_NAME;
            break;
        }
        case W_SPKI: {
            W_NEED();
            Tlv a;
            if (!w_hdr(rd, w.pos, w.end_tbs, t) || t.tag != 0x30u) W_FAIL();
            const uint32_t kp = w.pos + t.hdr, ke = kp + t.len;
            if (!w_hdr(rd, kp, ke, a) || a.tag != 0x30u) W_FAIL();
            const uint32_t bp = kp + a.hdr + a.len;
            w.end_c = ke;
            w.which = 0;
            if (!final && bp + 6u > w.pos + kWalkNeed) {  // long AlgorithmIdentifier (DSA / PSS parameters)
                w.pos = bp;
                w.st = W_SPKI_BITS;
                break;
            }
            if (!w_hdr(rd, bp, ke, t) || t.tag != 0x03u || t.len == 0u) W_FAIL();
            w.pos = ke;
            w.st = W_OPT;
            break;
        }
        case W_SPKI_BITS:
            W_NEED();
            if (!w_hdr(rd, w.pos, w.end_c, t) || t.tag != 0x03u || t.len == 0u) W_FAIL();
            w.pos = w.end_c;
            w.which = 0;
            w.st = W_OPT;
            break;
        case W_OPT:  // which: 0 expecting [1] issuerUniqueID, 1 expecting [2] subjectUniqueID, 2 expecting [3] extensions
            for (;;) {
                if (w.pos >= w.end_tbs) {
                    w.pos = w.end_tbs;
                    w.st = W_TAIL;
                    break;
                }
                W_NEED();
                if (!w_hdr(rd, w.pos, w.end_tbs, t)) W_FAIL();
                if (w.which == 0u) {
                    w.which = 1;
                    if (t.tag == 0x81u || t.tag == 0xa1u) { w.pos += t.hdr + t.len; continue; }
                }
                if (w.which == 1u) {
                    w.which = 2;
                    if (t.tag == 0x82u || t.tag == 0xa2u) { w.pos += t.hdr + t.len; continue; }
                }
                if (t.tag == 0xa3u) {  // [3] EXPLICIT Extensions ::= SEQUENCE OF Extension
                    Tlv seq;
                    const uint32_t xp = w.pos + t.hdr, xe = xp + t.len;
                    if (!w_hdr(rd, xp, xe, seq) || seq.tag != 0x30u) W_FAIL();
                    w.pos = xp + seq.hdr;
                    w.end_b = w.pos + seq.len;
                    w.st = W_EXTWALK;
                } else {  // anything else is tolerated trailing data (encoding/asn1 struct parsing)
                    w.pos = w.end_tbs;
                    w.st = W_TAIL;
                }
                break;
            }
            break;
        case W_EXTWALK:
            for (;;) {
                if (w.pos >= w.end_b) {
                    w.pos = w.end_tbs;
                    w.st = W_TAIL;
                    break;
                }
                W_NEED();
                Tlv oid;
                if (!w_hdr(rd, w.pos, w.end_b, t) || t.tag != 0x30u) W_FAIL();
                const uint32_t ip = w.pos + t.hdr, ee = ip + t.len;
                if (!w_hdr(rd, ip, ee, oid) || oid.tag != 0x06u) W_FAIL();
                const uint32_t o = ip + oid.hdr, rest = o + oid.len;
                w.which = (oid.len == 3u && rd(o) == 0x55u && rd(o + 1) == 0x1du) ? rd(o + 2) : 0u;
                if (!final && rest + 24u > w.pos + kWalkNeed) {  // long OID: the remainder in its own step
                    w.end_c = ee;
                    w.pos = rest;
                    w.st = W_EXT_REST;
                    break;
                }
                if (!w_ext_rest(w, rd, rest, ee)) W_FAIL();
                w.pos = ee;
            }
            break;
        case W_EXT_REST:
            W_NEED();
            if (!w_ext_rest(w, rd, w.pos, w.end_c)) W_FAIL();
            w.pos = w.end_c;
            w.st = W_EXTWALK;
            break;
        case W_TAIL: {
            W_NEED();
            if (!w_hdr(rd, w.pos, L, t) || t.tag != 0x30u) W_FAIL();  // signatureAlgorithm
            const uint32_t sp = w.pos + t.hdr + t.len;
            if (!final && sp + 6u > w.pos + kWalkNeed) {
                w.pos = sp;
                w.st = W_SIG;
                break;
            }
            if (!w_hdr(rd, sp, L, t) || t.tag != 0x03u || t.len == 0u) W_FAIL();  // signatureValue
            w.st = W_DONE;
            return;
        }
        case W_SIG:
            W_NEED();
            if (!w_hdr(rd, w.pos, L, t) || t.tag != 0x03u || t.len == 0u) W_FAIL();
            w.st = W_DONE;
            return;
        default:
            return;  // W_DONE / W_ERR
        }
    }
#undef W_NEED
#undef W_FAIL
}

}  // namespace ctmr
