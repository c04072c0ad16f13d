// ctmr_device.cuh -- device-side building blocks of the CT map path (sm_90a).
//
//   * SHA-256 compression held entirely in registers (8 state + 16 rolling schedule words);
//     rotations are funnel shifts (SHF.R.W), Ch/Maj/xor3 fold into LOP3, round constants are
//     immediates after full unrolling.  One lane hashes one certificate: the 64-round chain of a
//     single message is serial, so lane-level parallelism over 32 certificates per warp is the
//     only mapping that keeps the INT pipe full (DESIGN.md "Why lane-per-certificate").
//   * a bounds-checked DER TLV walker that extracts what the reference's worker reads from
//     ct-go's x509.Certificate (SURVEY.md §8(a) a3): raw serial, issuer CommonName (last 2.5.4.3),
//     notAfter, basicConstraints cA, SPKI span, cRLDistributionPoints span.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ctmr {

// ------------------------------------------------------------------------------------------------
// SHA-256
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t rotr32(uint32_t x, int n) { return __funnelshift_r(x, x, n); }
__device__ __forceinline__ uint32_t bsig0(uint32_t x) { return rotr32(x, 2) ^ rotr32(x, 13) ^ rotr32(x, 22); }
__device__ __forceinline__ uint32_t bsig1(uint32_t x) { return rotr32(x, 6) ^ rotr32(x, 11) ^ rotr32(x, 25); }
__device__ __forceinline__ uint32_t ssig0(uint32_t x) { return rotr32(x, 7) ^ rotr32(x, 18) ^ (x >> 3); }
__device__ __forceinline__ uint32_t ssig1(uint32_t x) { return rotr32(x, 17) ^ rotr32(x, 19) ^ (x >> 10); }
__device__ __forceinline__ uint32_t ch(uint32_t e, uint32_t f, uint32_t g) { return (e & f) ^ (~e & g); }
__device__ __forceinline__ uint32_t maj(uint32_t a, uint32_t b, uint32_t c) { return (a & b) ^ (a & c) ^ (b & c); }

struct Sha256State {
    uint32_t h[8];
    __device__ __forceinline__ void init() {
        h[0] = 0x6a09e667u; h[1] = 0xbb67ae85u; h[2] = 0x3c6ef372u; h[3] = 0xa54ff53au;
        h[4] = 0x510e527fu; h[5] = 0x9b05688cu; h[6] = 0x1f83d9abu; h[7] = 0x5be0cd19u;
    }
};

// Additions are steered onto the FMA pipe.  Rotations (SHF) and the boolean functions (LOP3) can
// only issue on the ALU datapath, and that datapath is the binding unit while the FMA datapath
// idles, because ptxas turns every add into IADD3 -- including `mad.lo x, 1, y`, which it folds
// back.  Multiplying by a run-time 1 (a kernel parameter it cannot fold) keeps a genuine IMAD,
// which issues on the otherwise idle FMA datapath and takes the adds off the ALU pipe
// (DESIGN.md §3, K_map).
__device__ __forceinline__ uint32_t fadd(uint32_t a, uint32_t b, uint32_t one) {
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(one), "r"(b));
    return d;
}

#ifndef CTMR_SHA_KADD_FMA
#define CTMR_SHA_KADD_FMA 1
#endif
#if CTMR_SHA_KADD_FMA
#define CTMR_SHA_HWK(h, w, k) fadd(fadd((h), (w), one), (k), one) /* K + (h + w) as two IMADs: no ALU slot at all */
#else
#define CTMR_SHA_HWK(h, w, k) ((h) + (w) + (k)) /* one IADD3 with the constant */
#endif

#define CTMR_SHA_ROUND(a, b, c, d, e, f, g, h, k, w)                     \
    do {                                                                 \
        uint32_t t1_ = CTMR_SHA_HWK(h, w, k);                            \
        t1_ = fadd(fadd(bsig1(e), t1_, one), ch((e), (f), (g)), one);    \
        uint32_t t2_ = fadd(bsig0(a), maj((a), (b), (c)), one);          \
        (d) = fadd((d), t1_, one);                                       \
        (h) = fadd(t1_, t2_, one);                                       \
    } while (0)

#define CTMR_SHA_SCHED(w, i)                                                                                    \
    ((w)[(i) & 15] = fadd(fadd(fadd(ssig1((w)[((i) - 2) & 15]), (w)[(i) & 15], one), (w)[((i) - 7) & 15], one), \
                          ssig0((w)[((i) - 15) & 15]), one))

// One 64-byte block; w[16] holds the big-endian message words and is clobbered.
__device__ __forceinline__ void sha256_compress(Sha256State& s, uint32_t (&w)[16], const uint32_t one) {
    constexpr uint32_t K[64] = {
        0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
        0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
        0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
        0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
        0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
        0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
        0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
        0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};
    uint32_t a = s.h[0], b = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4], f = s.h[5], g = s.h[6], h = s.h[7];
#pragma unroll
    for (int i = 0; i < 64; i += 8) {
        if (i >= 16) {
#pragma unroll
            for (int j = 0; j < 8; ++j) CTMR_SHA_SCHED(w, i + j);
        }
        CTMR_SHA_ROUND(a, b, c, d, e, f, g, h, K[i + 0], w[(i + 0) & 15]);
        CTMR_SHA_ROUND(h, a, b, c, d, e, f, g, K[i + 1], w[(i + 1) & 15]);
        CTMR_SHA_ROUND(g, h, a, b, c, d, e, f, K[i + 2], w[(i + 2) & 15]);
        CTMR_SHA_ROUND(f, g, h, a, b, c, d, e, K[i + 3], w[(i + 3) & 15]);
        CTMR_SHA_ROUND(e, f, g, h, a, b, c, d, K[i + 4], w[(i + 4) & 15]);
        CTMR_SHA_ROUND(d, e, f, g, h, a, b, c, K[i + 5], w[(i + 5) & 15]);
        CTMR_SHA_ROUND(c, d, e, f, g, h, a, b, K[i + 6], w[(i + 6) & 15]);
        CTMR_SHA_ROUND(b, c, d, e, f, g, h, a, K[i + 7], w[(i + 7) & 15]);
    }
    s.h[0] += a; s.h[1] += b; s.h[2] += c; s.h[3] += d; s.h[4] += e; s.h[5] += f; s.h[6] += g; s.h[7] += h;
}

// Same compression with the 64 rounds rolled into 4 passes of 16 (round constants from the constant
// bank instead of immediates).  ~7 KB of code instead of ~26 KB: the fully unrolled body misses in
// the instruction cache once 8-16 desynchronised warps per SM walk it at different offsets.
static __constant__ uint32_t kSha256K[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
    0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
    0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
    0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
    0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};

__device__ __forceinline__ void sha256_compress_rolled(Sha256State& s, uint32_t (&w)[16], const uint32_t one) {
    uint32_t a = s.h[0], b = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4], f = s.h[5], g = s.h[6], h = s.h[7];
#pragma unroll 1
    for (int it = 0; it < 4; ++it) {
        if (it != 0) {
#pragma unroll
            for (int j = 0; j < 16; ++j) CTMR_SHA_SCHED(w, j);
        }
        const uint32_t* kp = kSha256K + 16 * it;
#pragma unroll
        for (int j = 0; j < 16; j += 8) {
            CTMR_SHA_ROUND(a, b, c, d, e, f, g, h, kp[j + 0], w[j + 0]);
            CTMR_SHA_ROUND(h, a, b, c, d, e, f, g, kp[j + 1], w[j + 1]);
            CTMR_SHA_ROUND(g, h, a, b, c, d, e, f, kp[j + 2], w[j + 2]);
            CTMR_SHA_ROUND(f, g, h, a, b, c, d, e, kp[j + 3], w[j + 3]);
            CTMR_SHA_ROUND(e, f, g, h, a, b, c, d, kp[j + 4], w[j + 4]);
            CTMR_SHA_ROUND(d, e, f, g, h, a, b, c, kp[j + 5], w[j + 5]);
            CTMR_SHA_ROUND(c, d, e, f, g, h, a, b, kp[j + 6], w[j + 6]);
            CTMR_SHA_ROUND(b, c, d, e, f, g, h, a, kp[j + 7], w[j + 7]);
        }
    }
    s.h[0] += a; s.h[1] += b; s.h[2] += c; s.h[3] += d; s.h[4] += e; s.h[5] += f; s.h[6] += g; s.h[7] += h;
}

// Padding for the trailing blocks of a message of `len` bytes.  `q` is the byte position of word
// w inside the message; data bytes at positions >= len are garbage and get masked here.
__device__ __forceinline__ uint32_t sha256_pad_word(uint32_t w, uint32_t q, uint32_t len) {
    int k = (int)len - (int)q;  // valid data bytes in this word
    if (k >= 4) return w;
    if (k <= 0) return k == 0 ? 0x80000000u : 0u;
    uint32_t keep = 0xFFFFFFFFu << (32 - 8 * k);
    return (w & keep) | (0x80u << (24 - 8 * k));
}

// Straightforward SHA-256 of a short message in global memory (issuer SPKI: <= ~600 bytes,
// a few hundred distinct issuers per run) -- not the hot loop.
__device__ inline void sha256_global(const uint8_t* __restrict__ p, uint32_t len, uint32_t (&out)[8]) {
    Sha256State s;
    s.init();
    uint32_t nb = (len + 9 + 63) / 64;
    for (uint32_t b = 0; b < nb; ++b) {
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            uint32_t q = b * 64 + i * 4, v = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) v = (v << 8) | (q + j < len ? (uint32_t)p[q + j] : 0u);
            w[i] = sha256_pad_word(v, q, len);
        }
        if (b == nb - 1) { w[14] = 0; w[15] = len * 8u; }
        sha256_compress_rolled(s, w, 1u);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) out[i] = s.h[i];
}

// ------------------------------------------------------------------------------------------------
// DER walking
// ------------------------------------------------------------------------------------------------
struct ParsedCert {
    uint32_t serial_off, serial_len;
    uint32_t cn_off, cn_len;       // issuer CommonName value octets (cn_len = 0 and !has_cn -> "")
    uint32_t spki_off, spki_len;   // RawSubjectPublicKeyInfo, full TLV
    uint32_t crldp_off, crldp_len; // cRLDistributionPoints extnValue content, 0 = absent
    uint32_t issuer_off, issuer_len; // issuer Name, full TLV
    int64_t not_after;             // unix seconds
    uint32_t flags;                // PC_*
};
enum : uint32_t { PC_HAS_CN = 1u, PC_BC_VALID = 2u, PC_IS_CA = 4u };

struct Tlv {
    uint32_t tag, hdr, len;
};

// Go encoding/asn1 parseTagAndLength rules: single-octet tags, definite minimal lengths, value
// must fit inside [pos, end).  Returns false on violation.
__device__ __forceinline__ bool der_read(const uint8_t* __restrict__ d, uint32_t pos, uint32_t end, Tlv& t) {
    if (pos + 2u > end) return false;
    uint32_t tag = __ldg(d + pos), l = __ldg(d + pos + 1);
    if ((tag & 0x1fu) == 0x1fu) return false;
    t.tag = tag;
    if (l < 0x80u) {
        t.hdr = 2;
        t.len = l;
    } else {
        uint32_t nb = l & 0x7fu;
        if (nb == 0u || nb > 4u || pos + 2u + nb > end) return false;
        uint32_t v = 0;
        for (uint32_t i = 0; i < nb; ++i) {
            if (v >= (1u << 23)) return false;
            v = (v << 8) | __ldg(d + pos + 2u + i);
            if (v == 0u) return false;
        }
        if (v < 0x80u) return false;
        t.hdr = 2u + nb;
        t.len = v;
    }
    return t.len <= end - pos - t.hdr;
}

__device__ __forceinline__ bool der_2d(const uint8_t* __restrict__ p, uint32_t& v) {
    uint32_t a = __ldg(p) - (uint32_t)'0', b = __ldg(p + 1) - (uint32_t)'0';
    v = a * 10u + b;
    return a <= 9u && b <= 9u;
}

__device__ __forceinline__ int64_t days_from_civil(int64_t y, uint32_t m, uint32_t d) {
    y -= m <= 2;
    int64_t era = (y >= 0 ? y : y - 399) / 400;
    uint32_t yoe = (uint32_t)(y - era * 400);
    uint32_t doy = (153u * (m > 2 ? m - 3 : m + 9) + 2u) / 5u + d - 1u;
    uint32_t doe = yoe * 365u + yoe / 4u - yoe / 100u + doy;
    return era * 146097 + (int64_t)doe - 719468;
}

// UTCTime YYMMDDhhmm[ss](Z|+-hhmm) with the 1950 pivot, GeneralizedTime YYYYMMDDhhmmss(Z|+-hhmm);
// a numeric zero offset is rejected (Go re-serialises and compares).
__device__ inline bool der_time(uint32_t tag, const uint8_t* __restrict__ p, uint32_t len, int64_t& out) {
    uint32_t yy, cc, mo, dd, hh, mi, ss = 0, pos;
    int64_t year;
    if (tag == 0x18u) {
        if (len < 15u || !der_2d(p, cc) || !der_2d(p + 2, yy)) return false;
        year = (int64_t)cc * 100 + yy;
        pos = 4;
    } else if (tag == 0x17u) {
        if (len < 11u || !der_2d(p, yy)) return false;
        year = yy >= 50u ? 1900 + (int64_t)yy : 2000 + (int64_t)yy;
        pos = 2;
    } else {
        return false;
    }
    if (!der_2d(p + pos, mo) || !der_2d(p + pos + 2, dd) || !der_2d(p + pos + 4, hh) || !der_2d(p + pos + 6, mi))
        return false;
    pos += 8;
    bool has_sec = false;
    if (pos + 2u <= len) {
        uint32_t c0 = __ldg(p + pos);
        if (c0 >= '0' && c0 <= '9') {
            if (!der_2d(p + pos, ss)) return false;
            pos += 2;
            has_sec = true;
        }
    }
    if (tag == 0x18u && !has_sec) return false;
    if (pos >= len) return false;
    int64_t off = 0;
    uint32_t z = __ldg(p + pos);
    if (z == 'Z') {
        if (pos + 1u != len) return false;
    } else if (z == '+' || z == '-') {
        uint32_t oh, om;
        if (pos + 5u != len || !der_2d(p + pos + 1, oh) || !der_2d(p + pos + 3, om)) return false;
        if (oh > 23u || om > 59u) return false;
        off = (int64_t)oh * 3600 + (int64_t)om * 60;
        if (off == 0) return false;
        if (z == '-') off = -off;
    } else {
        return false;
    }
    if (mo < 1u || mo > 12u || dd < 1u || hh > 23u || mi > 59u || ss > 59u) return false;
    uint32_t maxd = (mo == 2u) ? 28u : ((0xAD5u >> (mo - 1u)) & 1u ? 31u : 30u);  // bitmask of 31-day months
    if (mo == 2u && (year % 4 == 0) && (year % 100 != 0 || year % 400 == 0)) maxd = 29u;
    if (dd > maxd) return false;
    out = days_from_civil(year, mo, dd) * 86400 + (int64_t)hh * 3600 + (int64_t)mi * 60 + (int64_t)ss - off;
    return true;
}

// RDNSequence: SET OF SEQUENCE { OID, value }.  Records the LAST 2.5.4.3 whose value is a string
// type (UTF8 0x0c, Printable 0x13, IA5 0x16, T61 0x14, Numeric 0x12): pkix.Name.FillFromRDNSequence.
__device__ inline bool der_name(const uint8_t* __restrict__ d, uint32_t pos, uint32_t end, ParsedCert* pc) {
    while (pos < end) {
        Tlv set;
        if (!der_read(d, pos, end, set) || set.tag != 0x31u) return false;
        uint32_t sp = pos + set.hdr, se = sp + set.len;
        while (sp < se) {
            Tlv atv, oid, val;
            if (!der_read(d, sp, se, atv) || atv.tag != 0x30u) return false;
            uint32_t ap = sp + atv.hdr, ae = ap + atv.len;
            if (!der_read(d, ap, ae, oid) || oid.tag != 0x06u) return false;
            uint32_t vp = ap + oid.hdr + oid.len;
            if (!der_read(d, vp, ae, val)) return false;
            if (pc != nullptr && oid.len == 3u) {
                uint32_t o = ap + oid.hdr;
                if (__ldg(d + o) == 0x55u && __ldg(d + o + 1) == 0x04u && __ldg(d + o + 2) == 0x03u) {
                    uint32_t t = val.tag;
                    if (t == 0x0cu || t == 0x13u || t == 0x16u || t == 0x14u || t == 0x12u) {
                        pc->cn_off = vp + val.hdr;
                        pc->cn_len = val.len;
                        pc->flags |= PC_HAS_CN;
                    }
                }
            }
            sp += atv.hdr + atv.len;
        }
        pos += set.hdr + set.len;
    }
    return true;
}

// Certificate ::= SEQ { TBS, sigAlg, BIT STRING }.  Returns false on anything a strict reading of
// RFC 5280 rejects in the fields the path uses; never reads outside [d, d+len).
// TBSCertificate at d[pos..len): everything the path reads from it.  tbs_end = offset just past it.
__device__ inline bool parse_tbs(const uint8_t* __restrict__ d, uint32_t pos, uint32_t len, ParsedCert& pc, uint32_t& tbs_end) {
    pc.serial_off = pc.serial_len = pc.cn_off = pc.cn_len = 0;
    pc.spki_off = pc.spki_len = pc.crldp_off = pc.crldp_len = 0;
    pc.issuer_off = pc.issuer_len = 0;
    pc.not_after = 0;
    pc.flags = 0;
    Tlv tbs, t;
    if (!der_read(d, pos, len, tbs) || tbs.tag != 0x30u) return false;
    uint32_t tp = pos + tbs.hdr, tend = tp + tbs.len;
    if (!der_read(d, tp, tend, t)) return false;
    if (t.tag == 0xa0u) {  // [0] EXPLICIT version
        tp += t.hdr + t.len;
        if (!der_read(d, tp, tend, t)) return false;
    }
    if (t.tag != 0x02u || t.len == 0u) return false;  // serialNumber
    if (t.len > 1u) {
        uint32_t b0 = __ldg(d + tp + t.hdr), b1 = __ldg(d + tp + t.hdr + 1);
        if ((b0 == 0x00u && (b1 & 0x80u) == 0u) || (b0 == 0xffu && (b1 & 0x80u) != 0u)) return false;
    }
    pc.serial_off = tp + t.hdr;
    pc.serial_len = t.len;
    tp += t.hdr + t.len;
    if (!der_read(d, tp, tend, t) || t.tag != 0x30u) return false;  // signature AlgorithmIdentifier
    tp += t.hdr + t.len;
    if (!der_read(d, tp, tend, t) || t.tag != 0x30u) return false;  // issuer
    pc.issuer_off = tp;
    pc.issuer_len = t.hdr + t.len;
    if (!der_name(d, tp + t.hdr, tp + t.hdr + t.len, &pc)) return false;
    tp += t.hdr + t.len;
    if (!der_read(d, tp, tend, t) || t.tag != 0x30u) return false;  // validity
    {
        uint32_t vp = tp + t.hdr, ve = vp + t.len;
        Tlv a, b;
        int64_t nb;
        if (!der_read(d, vp, ve, a) || !der_time(a.tag, d + vp + a.hdr, a.len, nb)) return false;
        vp += a.hdr + a.len;
        if (!der_read(d, vp, ve, b) || !der_time(b.tag, d + vp + b.hdr, b.len, pc.not_after)) return false;
    }
    tp += t.hdr + t.len;
    if (!der_read(d, tp, tend, t) || t.tag != 0x30u) return false;  // subject
    if (!der_name(d, tp + t.hdr, tp + t.hdr + t.len, nullptr)) return false;
    tp += t.hdr + t.len;
    if (!der_read(d, tp, tend, t) || t.tag != 0x30u) return false;  // subjectPublicKeyInfo
    pc.spki_off = tp;
    pc.spki_len = t.hdr + t.len;
    {
        uint32_t kp = tp + t.hdr, ke = kp + t.len;
        Tlv a, b;
        if (!der_read(d, kp, ke, a) || a.tag != 0x30u) return false;
        kp += a.hdr + a.len;
        if (!der_read(d, kp, ke, b) || b.tag != 0x03u || b.len == 0u) return false;
    }
    tp += t.hdr + t.len;
    if (tp < tend) {
        if (!der_read(d, tp, tend, t)) return false;
        if (t.tag == 0x81u || t.tag == 0xa1u) {  // issuerUniqueID
            tp += t.hdr + t.len;
            if (tp < tend && !der_read(d, tp, tend, t)) return false;
        }
    }
    if (tp < tend && (t.tag == 0x82u || t.tag == 0xa2u)) {  // subjectUniqueID
        tp += t.hdr + t.len;
        if (tp < tend && !der_read(d, tp, tend, t)) return false;
    }
    if (tp < tend && t.tag == 0xa3u) {  // [3] EXPLICIT extensions
        uint32_t xp = tp + t.hdr, xe = xp + t.len;
        Tlv seq;
        if (!der_read(d, xp, xe, seq) || seq.tag != 0x30u) return false;
        uint32_t ep = xp + seq.hdr, ee = ep + seq.len;
        while (ep < ee) {
            Tlv ext, oid, v;
            if (!der_read(d, ep, ee, ext) || ext.tag != 0x30u) return false;
            uint32_t ip = ep + ext.hdr, ie = ip + ext.len;
            if (!der_read(d, ip, ie, oid) || oid.tag != 0x06u) return false;
            uint32_t oidp = ip + oid.hdr;
            ip += oid.hdr + oid.len;
            if (!der_read(d, ip, ie, v)) return false;
            if (v.tag == 0x01u) {  // critical
                if (v.len != 1u) return false;
                uint32_t bv = __ldg(d + ip + v.hdr);
                if (bv != 0x00u && bv != 0xffu) return false;
                ip += v.hdr + v.len;
                if (!der_read(d, ip, ie, v)) return false;
            }
            if (v.tag != 0x04u) return false;
            uint32_t vp = ip + v.hdr, ve = vp + v.len;
            if (oid.len == 3u && __ldg(d + oidp) == 0x55u && __ldg(d + oidp + 1) == 0x1du) {
                uint32_t which = __ldg(d + oidp + 2);
                if (which == 0x13u) {  // basicConstraints
                    Tlv bc, f;
                    if (!der_read(d, vp, ve, bc) || bc.tag != 0x30u || vp + bc.hdr + bc.len != ve) return false;
                    uint32_t bp = vp + bc.hdr, be = bp + bc.len;
                    bool ca = false;
                    if (bp < be) {
                        if (!der_read(d, bp, be, f)) return false;
                        if (f.tag == 0x01u) {
                            if (f.len != 1u) return false;
                            uint32_t bv = __ldg(d + bp + f.hdr);
                            if (bv != 0x00u && bv != 0xffu) return false;
                            ca = bv != 0u;
                            bp += f.hdr + f.len;
                            if (bp < be && !der_read(d, bp, be, f)) return false;
                        }
                        if (bp < be && (f.tag != 0x02u || f.len == 0u)) return false;
                    }
                    pc.flags |= PC_BC_VALID;
                    pc.flags = ca ? (pc.flags | PC_IS_CA) : (pc.flags & ~PC_IS_CA);
                } else if (which == 0x1fu) {  // cRLDistributionPoints
                    pc.crldp_off = vp;
                    pc.crldp_len = v.len;
                }
            }
            ep += ext.hdr + ext.len;
        }
    }
    tbs_end = pos + tbs.hdr + tbs.len;
    return true;
}

__device__ inline bool parse_cert(const uint8_t* __restrict__ d, uint32_t len, ParsedCert& pc) {
    Tlv cert, t;
    if (!der_read(d, 0, len, cert) || cert.tag != 0x30u || cert.hdr + cert.len != len) return false;
    uint32_t pos = cert.hdr;
    if (!parse_tbs(d, pos, len, pc, pos)) return false;
    if (!der_read(d, pos, len, t) || t.tag != 0x30u) return false;  // signatureAlgorithm
    pos += t.hdr + t.len;
    if (!der_read(d, pos, len, t) || t.tag != 0x03u || t.len == 0u) return false;  // signatureValue
    return true;
}

// ------------------------------------------------------------------------------------------------
// hashing for the dedup tables
// ------------------------------------------------------------------------------------------------
__device__ __host__ __forceinline__ uint64_t mix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}

// owner of a Redis set "serials::<expDate>::<issuer>" in a multi-GPU run
__device__ __host__ __forceinline__ uint32_t key_owner(int32_t exp_hour, uint32_t issuer, uint32_t world) {
    return (uint32_t)(mix64(((uint64_t)issuer << 32) | (uint32_t)exp_hour) % world);
}

}  // namespace ctmr
