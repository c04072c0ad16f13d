// ctmr_crl.cu -- ctmr_revoked_known / ctmr_group_revoked_known: parse CRLs on the GPU and join their entries with the
// known-certificate table (include/ctmr.h states the contract, DESIGN.md "Revoked known certificates" the design).
//
// A chunk of whole CRLs goes through:
//   crl_frame        thread per CRL: CertificateList / TBSCertList fields, spans, the revokedCertificates content span
//   crl_candidates   thread per 16 staged bytes, twice around a scan: positions p inside a content span that start
//                    `30 L 02` with a well-formed definite length that stays inside the content; next(p) = p + TLV size
//   crl_link         thread per candidate: next(p) -> candidate index (binary search), END or NONE; marks the chain starts
//   crl_reach        thread per candidate, one launch per round: reach doubling along the jumps from each chain start
//   crl_check        thread per reached candidate: entry syntax; crl_settle (thread per CRL) decides the CRL's status
//   scan + crl_compact: the reached candidates of good CRLs become the chunk's entries, in (CRL, position) order
//   crl_entry        thread per entry: serial span, revocationDate, reasonCode, certificateIssuer, status
//   crl_set_insert   thread per entry: the chunk's (issuer, serial) pairs into an open-addressing set
//   crl_known_scan   grid-stride over the table: every ready key probes the set; a hit takes the lowest hour and counts
//   crl_finish       thread per entry: the pair's answer
#include <cub/device/device_scan.cuh>

#include "ctmr_common.cuh"
#include "ctmr_ctx.cuh"

namespace ctmr {
namespace {

constexpr uint32_t kEnd = 0xFFFFFFFFu;   // the chain's last entry ends exactly at the content's end
constexpr uint32_t kNone = 0xFFFFFFFEu;  // next(p) is no candidate: the chain breaks there
constexpr uint32_t kMinEntry = 18u;      // SEQUENCE 2 + INTEGER 3 + UTCTime YYMMDDhhmmZ 13

__device__ __forceinline__ bool oid_is_ce(const uint8_t* d, uint32_t p, const Tlv& oid, uint32_t last) {
    return oid.len == 3u && __ldg(d + p) == 0x55u && __ldg(d + p + 1) == 0x1du && __ldg(d + p + 2) == last;
}

// Extensions ::= SEQUENCE OF SEQUENCE { OID, BOOLEAN DEFAULT FALSE, OCTET STRING } filling [pos, end) exactly.  For
// each extension, f(oid_pos, oid, value_pos, value_len) returns false to reject it.
template <class F>
__device__ __forceinline__ bool walk_extensions(const uint8_t* d, uint32_t pos, uint32_t end, F&& f) {
    Tlv seq;
    if (!der_read(d, pos, end, seq) || seq.tag != 0x30u || pos + seq.hdr + seq.len != end) return false;
    uint32_t ep = pos + seq.hdr;
    const uint32_t ee = end;
    while (ep < ee) {
        Tlv ext, oid, v;
        if (!der_read(d, ep, ee, ext) || ext.tag != 0x30u) return false;
        uint32_t ip = ep + ext.hdr;
        const uint32_t ie = ip + ext.len;
        if (!der_read(d, ip, ie, oid) || oid.tag != 0x06u) return false;
        const uint32_t oidp = ip + oid.hdr;
        ip += oid.hdr + oid.len;
        if (!der_read(d, ip, ie, v)) return false;
        if (v.tag == 0x01u) {  // critical
            if (v.len != 1u) return false;
            const uint32_t bv = __ldg(d + ip + v.hdr);
            if (bv != 0x00u && bv != 0xffu) return false;
            ip += v.hdr + v.len;
            if (!der_read(d, ip, ie, v)) return false;
        }
        if (v.tag != 0x04u || ip + v.hdr + v.len != ie) return false;
        if (!f(oidp, oid, ip + v.hdr, v.len)) return false;
        ep = ie;
    }
    return true;
}

// One revokedCertificates entry at staged position p (its TLV is [p, end)): SEQUENCE { INTEGER, Time, Extensions
// OPTIONAL }, nothing after.
struct CrlEntry {
    uint32_t serial_pos, serial_len;
    int64_t revoked_at;
    uint32_t reason;    // 0xFF when absent
    bool indirect;
};
__device__ __forceinline__ bool parse_entry(const uint8_t* d, uint32_t p, uint32_t end, CrlEntry& e) {
    Tlv s, t;
    if (!der_read(d, p, end, s) || s.tag != 0x30u || p + s.hdr + s.len != end) return false;
    uint32_t q = p + s.hdr;
    if (!der_read(d, q, end, t) || t.tag != 0x02u || t.len == 0u) return false;
    e.serial_pos = q + t.hdr;
    e.serial_len = t.len;
    q += t.hdr + t.len;
    if (!der_read(d, q, end, t) || !der_time(t.tag, d + q + t.hdr, t.len, e.revoked_at)) return false;
    q += t.hdr + t.len;
    e.reason = 0xFFu;
    e.indirect = false;
    if (q == end) return true;
    if (!der_read(d, q, end, t) || t.tag != 0x30u || q + t.hdr + t.len != end) return false;
    return walk_extensions(d, q, end, [&](uint32_t oidp, const Tlv& oid, uint32_t vp, uint32_t vlen) {
        if (oid_is_ce(d, oidp, oid, 0x15u)) {  // reasonCode: ENUMERATED of one octet
            if (vlen != 3u || __ldg(d + vp) != 0x0au || __ldg(d + vp + 1) != 0x01u) return false;
            e.reason = __ldg(d + vp + 2);
        } else if (oid_is_ce(d, oidp, oid, 0x1du)) {  // certificateIssuer
            e.indirect = true;
        }
        return true;
    });
}

__global__ void __launch_bounds__(128) crl_frame_kernel(const uint8_t* __restrict__ stage, const CrlDesc* __restrict__ desc, uint32_t n,
                                                        CrlRes* __restrict__ res) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const CrlDesc cd = desc[k];
    CrlRes r{};
    r.next_update = INT64_MIN;
    r.cs = r.ce = cd.staged;
    r.first = 0xFFFFFFFFu;
    r.status = CTMR_CRL_BAD;
    const uint8_t* d = stage + cd.staged;
    const uint32_t len = cd.len;
    bool ok = false;
    do {
        Tlv cl, tbs, t;
        if (!der_read(d, 0, len, cl) || cl.tag != 0x30u || cl.hdr + cl.len != len) break;
        const uint32_t pos = cl.hdr;
        if (!der_read(d, pos, len, tbs) || tbs.tag != 0x30u) break;
        r.tbs_off = cd.data_off + pos;
        r.tbs_len = tbs.hdr + tbs.len;
        uint32_t tp = pos + tbs.hdr;
        const uint32_t tend = tp + tbs.len;
        if (!der_read(d, tp, tend, t)) break;
        if (t.tag == 0x02u) {  // version: v2 is the only value written
            if (t.len != 1u || __ldg(d + tp + t.hdr) != 1u) break;
            tp += t.hdr + t.len;
            if (!der_read(d, tp, tend, t)) break;
        }
        if (t.tag != 0x30u) break;  // signature AlgorithmIdentifier
        tp += t.hdr + t.len;
        if (!der_read(d, tp, tend, t) || t.tag != 0x30u) break;  // issuer
        r.name_off = cd.data_off + tp;
        r.name_len = t.hdr + t.len;
        if (!der_name(d, tp + t.hdr, tp + t.hdr + t.len, nullptr)) break;
        tp += t.hdr + t.len;
        if (!der_read(d, tp, tend, t) || !der_time(t.tag, d + tp + t.hdr, t.len, r.this_update)) break;
        tp += t.hdr + t.len;
        if (tp < tend) {
            if (!der_read(d, tp, tend, t)) break;
            if (t.tag == 0x17u || t.tag == 0x18u) {  // nextUpdate
                if (!der_time(t.tag, d + tp + t.hdr, t.len, r.next_update)) break;
                tp += t.hdr + t.len;
                if (tp < tend && !der_read(d, tp, tend, t)) break;
            }
        }
        if (tp < tend && t.tag == 0x30u) {  // revokedCertificates
            r.cs = cd.staged + tp + t.hdr;
            r.ce = r.cs + t.len;
            tp += t.hdr + t.len;
            if (tp < tend && !der_read(d, tp, tend, t)) break;
        }
        if (tp < tend && t.tag == 0xa0u) {  // [0] EXPLICIT crlExtensions
            uint32_t flags = 0;
            const bool ext_ok = walk_extensions(d, tp + t.hdr, tp + t.hdr + t.len, [&](uint32_t oidp, const Tlv& oid, uint32_t, uint32_t) {
                if (oid_is_ce(d, oidp, oid, 0x1bu)) flags |= CTMR_CRL_F_DELTA;
                if (oid_is_ce(d, oidp, oid, 0x1cu)) flags |= CTMR_CRL_F_IDP;
                return true;
            });
            if (!ext_ok) break;
            r.flags = flags;
            tp += t.hdr + t.len;
        }
        if (tp != tend) break;
        uint32_t sp = tend;
        if (!der_read(d, sp, len, t) || t.tag != 0x30u) break;  // signatureAlgorithm
        sp += t.hdr + t.len;
        if (!der_read(d, sp, len, t) || t.tag != 0x03u || t.len == 0u) break;  // signatureValue
        if (sp + t.hdr + t.len != len) break;
        ok = true;
    } while (false);
    if (ok) {
        r.status = CTMR_CRL_OK;
    } else {
        r.cs = r.ce = cd.staged;  // nothing to split; keeps the spans ordered for crl_candidates' search
        r.flags = 0;
    }
    res[k] = r;
}

// is p a candidate of the content ending at ce: 30 L 02 .., a well-formed definite length, the TLV inside the content
__device__ __forceinline__ bool candidate_at(const uint8_t* d, uint32_t p, uint32_t ce, uint32_t& next) {
    if (__ldg(d + p) != 0x30u) return false;
    Tlv t;
    if (!der_read(d, p, ce, t) || t.len == 0u || __ldg(d + p + t.hdr) != 0x02u) return false;
    next = p + t.hdr + t.len;
    return true;
}

// the CRL whose content span holds p, or the last CRL whose span starts at or before p (spans are ordered and disjoint)
__device__ __forceinline__ uint32_t crl_of(const CrlRes* res, uint32_t n, uint32_t p) {
    uint32_t lo = 0, hi = n;  // first k with cs > p
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (res[mid].cs <= p) lo = mid + 1; else hi = mid;
    }
    return lo == 0 ? 0u : lo - 1u;
}

// WRITE = false: cnt[t] = candidates among staged bytes [16t, 16t + 16) for every t < groups (0 past the chunk).
// WRITE = true: they go to off[t] ... in byte order, which is (CRL, position) order.
template <bool WRITE>
__global__ void __launch_bounds__(256) crl_candidates_kernel(const uint8_t* __restrict__ stage, uint32_t bytes, uint32_t groups,
                                                             const CrlRes* __restrict__ res, uint32_t n, uint32_t* __restrict__ cnt,
                                                             const uint32_t* __restrict__ off, uint32_t* __restrict__ cpos,
                                                             uint32_t* __restrict__ ccrl, uint32_t* __restrict__ cnext) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= groups) return;
    const uint32_t p0 = t * 16u;
    if (p0 >= bytes) {
        if (!WRITE) cnt[t] = 0;
        return;
    }
    uint32_t k = crl_of(res, n, p0), c = 0, o = WRITE ? off[t] : 0u;
    const uint32_t p1 = min(p0 + 16u, bytes);
    for (uint32_t p = p0; p < p1; ++p) {
        while (k + 1u < n && p >= res[k].ce && p >= res[k + 1u].cs) ++k;
        const CrlRes& r = res[k];
        uint32_t next;
        if (p < r.cs || p >= r.ce || !candidate_at(stage, p, r.ce, next)) continue;
        if (WRITE) {
            cpos[o + c] = p;
            ccrl[o + c] = k;
            cnext[o + c] = next;
        }
        ++c;
    }
    if (!WRITE) cnt[t] = c;
}

// link[i] = the candidate at next(p_i), END at the content's end, NONE otherwise; the candidate at a content span's
// start is its chain's first entry
__global__ void __launch_bounds__(256) crl_link_kernel(const CrlRes* __restrict__ res, const uint32_t* __restrict__ cpos, const uint32_t* __restrict__ ccrl,
                                                       uint32_t m, uint32_t* __restrict__ link, uint32_t* __restrict__ jump, uint8_t* __restrict__ mark) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const CrlRes& r = res[ccrl[i]];
    const uint32_t next = link[i];
    uint32_t to = kNone;
    if (next == r.ce) {
        to = kEnd;
    } else {
        uint32_t lo = i + 1u, hi = m;  // next > p_i: search above i
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (cpos[mid] < next) lo = mid + 1; else hi = mid;
        }
        if (lo < m && cpos[lo] == next) to = lo;
    }
    link[i] = to;
    jump[i] = to;
    mark[i] = cpos[i] == r.cs ? 1 : 0;
}

// Round k of reach doubling: every reached candidate marks jump_k(c), and jump_{k+1} = jump_k o jump_k.  After round k
// the first 2^(k+1) entries of each chain are marked (a mark made earlier in the same round only adds entries further
// down the same chain).  A false candidate whose next lands on the chain is never reached: nothing jumps to it.
__global__ void __launch_bounds__(256) crl_reach_kernel(const uint32_t* __restrict__ jin, uint32_t* __restrict__ jout, uint8_t* mark, uint32_t m) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint32_t j = jin[i];
    const bool real = j < kNone;
    if (real && mark[i]) mark[j] = 1;
    jout[i] = real ? jin[j] : j;
}

// every reached candidate: its link ends the chain (END) or breaks it (NONE), and its entry must parse
__global__ void __launch_bounds__(256) crl_check_kernel(const uint8_t* __restrict__ stage, CrlRes* res, const uint32_t* __restrict__ cpos,
                                                        const uint32_t* __restrict__ ccrl, const uint32_t* __restrict__ link,
                                                        const uint8_t* __restrict__ mark, uint32_t m) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m || !mark[i]) return;
    CrlRes& r = res[ccrl[i]];
    const uint32_t l = link[i];
    if (l == kEnd) atomicOr(&r.done, 1u);
    if (l == kNone) atomicOr(&r.bad, 1u);
    Tlv t;
    der_read(stage, cpos[i], r.ce, t);  // a candidate: well-formed
    CrlEntry e;
    if (!parse_entry(stage, cpos[i], cpos[i] + t.hdr + t.len, e)) atomicOr(&r.bad, 1u);
}

__global__ void __launch_bounds__(128) crl_settle_kernel(const CrlDesc* __restrict__ desc, CrlRes* res, uint32_t n) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    CrlRes& r = res[k];
    if (r.status != CTMR_CRL_OK) return;
    if (r.cs != r.ce && (r.bad || !r.done)) r.status = CTMR_CRL_BAD_ENTRIES;
    else if (desc[k].issuer == CTMR_ISSUER_NONE) r.status = CTMR_CRL_UNKNOWN_ISSUER;
}

__device__ __forceinline__ bool crl_listed(uint32_t status) { return status == CTMR_CRL_OK || status == CTMR_CRL_UNKNOWN_ISSUER; }

__global__ void __launch_bounds__(256) crl_keep_kernel(const CrlRes* __restrict__ res, const uint32_t* __restrict__ ccrl,
                                                       const uint8_t* __restrict__ mark, uint32_t m, uint32_t* __restrict__ keep) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) keep[i] = mark[i] && crl_listed(res[ccrl[i]].status) ? 1u : 0u;
}

__global__ void __launch_bounds__(256) crl_compact_kernel(CrlRes* res, const uint32_t* __restrict__ cpos, const uint32_t* __restrict__ ccrl,
                                                          const uint32_t* __restrict__ keep, const uint32_t* __restrict__ at, uint32_t m,
                                                          uint32_t* __restrict__ epos, uint32_t* __restrict__ ecrl) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m || !keep[i]) return;
    const uint32_t e = at[i], k = ccrl[i];
    epos[e] = cpos[i];
    ecrl[e] = k;
    atomicMin(&res[k].first, e);
    atomicAdd(&res[k].count, 1u);
}

struct EntryOut {
    uint64_t* serial_off;
    uint8_t *serial_len, *reason, *status, *known;
    int64_t *revoked, *hour;
    uint32_t *slot, *sets;
};

__global__ void __launch_bounds__(256) crl_entry_kernel(const uint8_t* __restrict__ stage, const CrlDesc* __restrict__ desc,
                                                        const CrlRes* __restrict__ res, const uint32_t* __restrict__ epos,
                                                        const uint32_t* __restrict__ ecrl, uint32_t ne, EntryOut o) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne) return;
    const uint32_t k = ecrl[e], p = epos[e];
    Tlv t;
    der_read(stage, p, res[k].ce, t);
    CrlEntry ce;
    parse_entry(stage, p, p + t.hdr + t.len, ce);  // checked by crl_check_kernel
    o.serial_off[e] = desc[k].data_off + (ce.serial_pos - desc[k].staged);
    o.serial_len[e] = (uint8_t)min(ce.serial_len, 255u);
    o.revoked[e] = ce.revoked_at;
    o.reason[e] = (uint8_t)ce.reason;
    o.status[e] = ce.indirect ? CTMR_RV_INDIRECT : ce.serial_len > CTMR_MAX_SERIAL ? CTMR_RV_SERIAL_TOO_LONG : CTMR_RV_OK;
}

// an entry's pair as the words w: issuer, then {serial_len, serial[39]} read from the staged CRL (len <= 255: at most 39
// serial bytes are read, all inside the serial)
__device__ __forceinline__ void pair_words(const uint8_t* stage, const CrlDesc& cd, uint64_t serial_off, uint32_t len, uint32_t (&w)[11]) {
    w[0] = cd.issuer;
    const uint8_t* s = stage + cd.staged + (uint32_t)(serial_off - cd.data_off) - 1;  // s[at]: serial byte at - 1
#pragma unroll
    for (uint32_t q = 0; q < 10u; ++q) {  // static register indices
        uint32_t v = q == 0u ? len : 0u;
#pragma unroll
        for (uint32_t b = 0; b < 4u; ++b) {
            const uint32_t at = 4u * q + b;
            if (at >= 1u && at <= len) v |= (uint32_t)__ldg(s + at) << (8u * b);
        }
        w[1 + q] = v;
    }
}

// find-or-insert of the pair w: its slot; equal pairs share one
__device__ __forceinline__ uint32_t set_insert(CrlSetSlot* set, uint64_t mask, const uint32_t (&w)[11]) {
    const uint32_t h = pair_hash(w);
    const uint32_t ready = (h & ~3u) | 2u, pending = (h & ~3u) | 1u;
    uint64_t pos = h & mask;
    for (;;) {
        CrlSetSlot* sl = set + pos;
        uint32_t tg = atomicCAS(&sl->tag, 0u, pending);
        if (tg == 0u) {
#pragma unroll
            for (int i = 0; i < 11; ++i) sl->key[i] = w[i];
            __threadfence();
            atomicExch(&sl->tag, ready);
            break;
        }
        if ((tg & ~3u) == (h & ~3u)) {
            while ((tg & 3u) == 1u) tg = *reinterpret_cast<volatile uint32_t*>(&sl->tag);
            __threadfence();
            bool same = true;
#pragma unroll
            for (int i = 0; i < 11; ++i) same &= *reinterpret_cast<volatile uint32_t*>(&sl->key[i]) == w[i];
            if (same) break;
        }
        pos = (pos + 1) & mask;  // the set has twice the pairs' slots: a free one always exists
    }
    return (uint32_t)pos;
}

__global__ void __launch_bounds__(256) crl_set_insert_kernel(const uint8_t* __restrict__ stage, const CrlDesc* __restrict__ desc,
                                                             const CrlRes* __restrict__ res, const uint32_t* __restrict__ ecrl,
                                                             const uint64_t* __restrict__ serial_off, const uint8_t* __restrict__ serial_len,
                                                             const uint8_t* __restrict__ status, uint32_t ne, CrlSetSlot* set, uint64_t mask,
                                                             uint32_t* __restrict__ slot) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne) return;
    const uint32_t k = ecrl[e];
    const CrlDesc cd = desc[k];
    if (status[e] != CTMR_RV_OK || res[k].status != CTMR_CRL_OK) {
        slot[e] = kNone;
        return;
    }
    uint32_t w[11];
    pair_words(stage, cd, serial_off[e], serial_len[e], w);
    slot[e] = set_insert(set, mask, w);
}

// one pass over the table: every ready key probes the set with its (issuer, serial); a hit records the key's hour
__global__ void __launch_bounds__(256) crl_known_scan_kernel(const KnownSlot* __restrict__ table, uint64_t n_slots, uint32_t epoch,
                                                             const CrlSetSlot* __restrict__ set, uint64_t mask, int32_t* hour,
                                                             uint32_t* count) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slots; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4* sp = reinterpret_cast<const uint4*>(table + i);
        const uint4 q0 = __ldcs(sp), q1 = __ldcs(sp + 1), q2 = __ldcs(sp + 2), q3 = __ldcs(sp + 3);
        if (slot_state(((uint64_t)q0.w << 32) | q0.z, epoch) != kSlotReady) continue;
        const uint32_t w[11] = {q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};
        const uint32_t h = pair_hash(w), ready = (h & ~3u) | 2u;
        uint64_t pos = h & mask;
        for (;;) {
            const CrlSetSlot& sl = set[pos];
            const uint32_t tg = sl.tag;
            if (tg == 0u) break;
            if (tg == ready) {
                bool same = true;
#pragma unroll
                for (int k = 0; k < 11; ++k) same &= sl.key[k] == w[k];
                if (same) {
                    atomicMin(hour + pos, (int32_t)q1.x);
                    atomicAdd(count + pos, 1u);
                    break;
                }
            }
            pos = (pos + 1) & mask;
        }
    }
}

// a group's member 0: another member's answers into its own
__global__ void __launch_bounds__(256) crl_merge_kernel(int32_t* hour, uint32_t* count, const int32_t* __restrict__ rh,
                                                        const uint32_t* __restrict__ rc, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || rc[i] == 0u) return;
    hour[i] = min(hour[i], rh[i]);
    count[i] += rc[i];
}

__global__ void __launch_bounds__(256) crl_finish_kernel(const uint32_t* __restrict__ slot, const int32_t* __restrict__ hour,
                                                         const uint32_t* __restrict__ count, uint32_t ne, EntryOut o) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne) return;
    const uint32_t s = slot[e];
    const uint32_t n = s < kNone ? count[s] : 0u;
    o.known[e] = n ? 1 : 0;
    o.hour[e] = n ? (int64_t)hour[s] : 0;
    o.sets[e] = n;
}

// ---- one process per GPU: every rank's entries against every rank's shard, through the exchange area's inbox regions.
// Region of source s on owner o: px.inbox[o] + s X (parity 0), its record count px.counts[o][s].

// What every rank agreed a source sends in this round (the mailbox row).  The owner never reads more records of a source
// than this, whatever the source's published count says: a source that missed its send (a failure, or a barrier that timed
// out) leaves an earlier round's count behind, and the union set is sized for the agreed total only.
struct CrlRoundCounts {
    unsigned long long n[kMaxWorld];
};

__device__ __forceinline__ uint64_t crl_received(const PeerExchange& px, const CrlRoundCounts& agreed, uint32_t src) {
    unsigned long long a = 0;
#pragma unroll
    for (uint32_t r = 0; r < kMaxWorld; ++r)  // static indices: the counts stay in parameter space, no local copy
        if (r == src) a = agreed.n[r];
    return min(min((unsigned long long)px.X, ld_volatile_u64(px.counts[px.rank] + src)), a);
}

// thread per entry lo + t of the chunk, t < n: its 64-byte record (ctmr_key layout) into rec[t]: index = the entry's
// position in the chunk, issuer, {serial_len, serial}, valid = 1 only for a CTMR_RV_OK entry of a CTMR_CRL_OK CRL; exp_hour
// and pad carry the answer later
__global__ void __launch_bounds__(256) crl_peer_records_kernel(const uint8_t* __restrict__ stage, const CrlDesc* __restrict__ desc,
                                                               const CrlRes* __restrict__ res, const uint32_t* __restrict__ ecrl,
                                                               const uint64_t* __restrict__ serial_off, const uint8_t* __restrict__ serial_len,
                                                               const uint8_t* __restrict__ status, uint32_t lo, uint32_t n,
                                                               ctmr_key* __restrict__ rec) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t e = lo + t;
    const uint32_t k = ecrl[e];
    const CrlDesc cd = desc[k];
    uint32_t w[11];
    pair_words(stage, cd, serial_off[e], serial_len[e], w);
    const uint32_t valid = status[e] == CTMR_RV_OK && res[k].status == CTMR_CRL_OK ? 1u : 0u;
    uint4* dst = reinterpret_cast<uint4*>(rec + t);
    dst[0] = make_uint4(e, 0u, 0u, w[0]);
    dst[1] = make_uint4(w[1], w[2], w[3], w[4]);
    dst[2] = make_uint4(w[5], w[6], w[7], w[8]);
    dst[3] = make_uint4(w[9], w[10], valid, 0u);
}

// Source side, grid (records x 4 / 256, world): records [0, n) into this source's region on every rank, its own among
// them, four lanes per record so that a warp writes 512 contiguous bytes of posted stores; then the count.
__global__ void __launch_bounds__(256) crl_peer_send_kernel(PeerExchange px, const ctmr_key* __restrict__ rec, uint64_t n) {
    const uint32_t owner = blockIdx.y;
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < 4u * n) {
        const uint4 v = reinterpret_cast<const uint4*>(rec)[t];
        reinterpret_cast<uint4*>(px.inbox[owner] + (uint64_t)px.rank * px.X)[t] = v;
    }
    if (t == 0) px.counts[owner][px.rank] = n;  // the barrier after this kernel publishes both
}

// Owner side, grid (the most records of a source / 256, world): every valid record received into the union set; equal
// keys of several sources share a slot.  in_slot[s X + j] = the record's slot, NONE for an invalid one.  The set has at
// least twice the agreed total's slots, so a free one always exists.
__global__ void __launch_bounds__(256) crl_union_insert_kernel(PeerExchange px, CrlRoundCounts agreed, CrlSetSlot* set, uint64_t mask,
                                                               uint32_t* __restrict__ in_slot) {
    const uint32_t src = blockIdx.y;
    const uint64_t m = crl_received(px, agreed, src);
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint4* r = reinterpret_cast<const uint4*>(px.inbox[px.rank] + (uint64_t)src * px.X + j);
    const uint4 q0 = __ldcg(r), q1 = __ldcg(r + 1), q2 = __ldcg(r + 2), q3 = __ldcg(r + 3);
    if (q3.z != 1u) {
        in_slot[(uint64_t)src * px.X + j] = kNone;
        return;
    }
    const uint32_t w[11] = {q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y};
    in_slot[(uint64_t)src * px.X + j] = set_insert(set, mask, w);
}

// Owner side, after the scan of its shard: each received record's answer in place, exp_hour = the lowest hour of this
// shard's sets that hold it and pad = how many (0: none, or an invalid record)
__global__ void __launch_bounds__(256) crl_peer_answer_kernel(PeerExchange px, CrlRoundCounts agreed, const uint32_t* __restrict__ in_slot,
                                                              const int32_t* __restrict__ hour, const uint32_t* __restrict__ count) {
    const uint32_t src = blockIdx.y;
    const uint64_t m = crl_received(px, agreed, src);
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint32_t s = in_slot[(uint64_t)src * px.X + j];
    const uint32_t n = s < kNone ? count[s] : 0u;
    ctmr_key* r = px.inbox[px.rank] + (uint64_t)src * px.X + j;
    r->exp_hour = n ? hour[s] : 0;
    r->pad = n;
}

// Source side, thread per record of the round: the answers of all owners for records [0, n) of this source, read from its
// region on each owner; entry lo + i gets the lowest hour where an owner counted sets, and the sum of the counts
__global__ void __launch_bounds__(256) crl_peer_pull_kernel(PeerExchange px, uint64_t n, uint64_t lo, uint8_t* __restrict__ known,
                                                            int64_t* __restrict__ hour, uint32_t* __restrict__ sets) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int32_t h = INT32_MAX;
    uint32_t total = 0;
    for (uint32_t o = 0; o < px.world; ++o) {
        const ctmr_key* r = px.inbox[o] + (uint64_t)px.rank * px.X + i;
        const uint32_t c = __ldcv(&r->pad);
        if (c) {
            h = min(h, __ldcv(&r->exp_hour));
            total += c;
        }
    }
    known[lo + i] = total ? 1 : 0;
    hour[lo + i] = total ? (int64_t)h : 0;
    sets[lo + i] = total;
}

inline unsigned grid(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

}  // namespace
}  // namespace ctmr

namespace {

constexpr uint64_t kCrlBudgetMax = 256ull << 20;  // staged CRL bytes per chunk
constexpr uint64_t kCrlsPerChunk = 1ull << 16;

// staged CRL bytes per chunk
uint64_t crl_budget(const ctmr_ctx* c) { return ((c->stage_bytes < kCrlBudgetMax ? c->stage_bytes : kCrlBudgetMax) + 15) / 16 * 16; }

// The split's buffers on first use, for chunks of the ctx's budget: built into a local, moved in only when every
// allocation succeeded.
int crl_ensure(ctmr_ctx* c) {
    if (c->crl && c->crl->budget) return CTMR_OK;
    std::unique_ptr<CrlState> s(new (std::nothrow) CrlState());
    if (!s) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    const uint64_t B = crl_budget(c);
    s->budget = B;
    s->cap_crls = kCrlsPerChunk;
    // Candidates of any input: map a candidate p to p + 2 when its length is short (that byte is 02, no candidate) and to
    // p + 1 when it is long (81..84, no candidate).  No two candidates share an image (p short and p + 1 long would need
    // byte p + 2 to be both 02 and 81..84), so at most half the bytes start one -- 30 01 02 repeated reaches a third.
    s->cap_cand = B / 2 + 2;
    s->cap_entries = B / kMinEntry + 1;
    CU(c, create(s->copy_stream));
    for (int i = 0; i < 2; ++i) {
        CU(c, alloc(s->stage[i], B + 64));
        CU(c, cudaMemsetAsync(s->stage[i], 0, B + 64, c->stream));
        CU(c, alloc(s->desc[i], s->cap_crls));
        CU(c, alloc(s->h_desc[i], s->cap_crls));
        CU(c, create(s->uploaded[i]));
        CU(c, create(s->consumed[i]));
    }
    CU(c, alloc(s->res, s->cap_crls));
    CU(c, alloc(s->cnt16, B / 16 + 2));
    CU(c, alloc(s->off16, B / 16 + 2));
    CU(c, alloc(s->cpos, s->cap_cand));
    CU(c, alloc(s->ccrl, s->cap_cand));
    CU(c, alloc(s->link, s->cap_cand));
    CU(c, alloc(s->jump[0], s->cap_cand));
    CU(c, alloc(s->jump[1], s->cap_cand));
    CU(c, alloc(s->mark, s->cap_cand));
    size_t t1 = 0, t2 = 0;
    CU(c, cub::DeviceScan::ExclusiveSum(nullptr, t1, s->cnt16.get(), s->off16.get(), (int)(B / 16 + 2)));
    CU(c, cub::DeviceScan::ExclusiveSum(nullptr, t2, s->jump[0].get(), s->jump[1].get(), (int)s->cap_cand));
    s->temp_bytes = t1 > t2 ? t1 : t2;
    CU(c, alloc(s->temp, s->temp_bytes ? s->temp_bytes : 16));
    const uint64_t E = s->cap_entries;
    CU(c, alloc(s->epos, E)); CU(c, alloc(s->ecrl, E)); CU(c, alloc(s->eslot, E)); CU(c, alloc(s->esets, E));
    CU(c, alloc(s->eserial_off, E));
    CU(c, alloc(s->eserial_len, E)); CU(c, alloc(s->ereason, E)); CU(c, alloc(s->estatus, E)); CU(c, alloc(s->eknown, E));
    CU(c, alloc(s->erevoked, E)); CU(c, alloc(s->ehour, E));
    CU(c, cudaStreamSynchronize(c->stream));
    if (c->crl) {  // a group member's set arrays came first: keep them
        s->set_cap = c->crl->set_cap;
        s->set = std::move(c->crl->set);
        s->set_hour = std::move(c->crl->set_hour);
        s->set_count = std::move(c->crl->set_count);
        s->recv_hour = std::move(c->crl->recv_hour);
        s->recv_count = std::move(c->crl->recv_count);
    }
    c->crl = std::move(s);
    return CTMR_OK;
}

// the set arrays for `slots` pairs (a power of two), all or nothing; `recv`: also the receive side of a group's member 0
int crl_set_ensure(ctmr_ctx* c, uint64_t slots, bool recv) {
    if (!c->crl) {
        c->crl.reset(new (std::nothrow) CrlState());
        if (!c->crl) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    }
    CrlState* s = c->crl.get();
    if (s->set_cap >= slots && (!recv || s->recv_hour)) return CTMR_OK;
    const uint64_t cap = s->set_cap > slots ? s->set_cap : slots;
    DevBuf<CrlSetSlot> set;
    DevBuf<int32_t> hour, rhour;
    DevBuf<uint32_t> count, rcount;
    CU(c, alloc(set, cap));
    CU(c, alloc(hour, cap));
    CU(c, alloc(count, cap));
    if (recv) {
        CU(c, alloc(rhour, cap));
        CU(c, alloc(rcount, cap));
    }
    s->set = std::move(set);
    s->set_hour = std::move(hour);
    s->set_count = std::move(count);
    s->recv_hour = std::move(rhour);
    s->recv_count = std::move(rcount);
    s->set_cap = cap;
    return CTMR_OK;
}

// A rank attached to peers, after crl_ensure: the records of one round (X) and the union set of a round (2 world X
// slots, so that a free slot always exists), all or nothing
int crl_peer_ensure(ctmr_ctx* c) {
    CrlState* s = c->crl.get();
    if (s->records) return CTMR_OK;
    const uint64_t cap = pow2_at_least(2ull * c->px.world * c->px.X);
    DevBuf<ctmr_key> records;
    DevBuf<CrlSetSlot> set;
    DevBuf<int32_t> hour;
    DevBuf<uint32_t> count;
    CU(c, alloc(records, c->px.X));
    CU(c, alloc(set, cap));
    CU(c, alloc(hour, cap));
    CU(c, alloc(count, cap));
    s->union_set = std::move(set);
    s->union_hour = std::move(hour);
    s->union_count = std::move(count);
    s->union_cap = cap;
    s->records = std::move(records);  // last: a state with records has all of it
    return CTMR_OK;
}

struct CrlChunk {
    uint64_t lo = 0, hi = 0;  // CRLs of the batch
    uint64_t bytes = 0;
    uint32_t rounds = 0;      // reach doubling rounds: ceil(log2(most entries one of its CRLs can hold))
};

// Stage chunk `ch` into stage[st] on the copy stream: the CRLs back to back, one copy per run of CRLs that lie back to
// back in the caller's data
int crl_upload(ctmr_ctx* c, const ctmr_crl_batch* b, const std::vector<uint32_t>& issuer, const CrlChunk& ch, int st) {
    CrlState* s = c->crl.get();
    CU(c, cudaStreamWaitEvent(s->copy_stream, s->consumed[st], 0));  // the chunk that last used this stage is done with it
    CU(c, cudaStreamSynchronize(s->copy_stream));                     // h_desc[st] is rewritten below
    uint64_t staged = 0, run_src = 0, run_dst = 0, run_len = 0;
    for (uint64_t k = ch.lo; k < ch.hi; ++k) {
        const uint64_t off = b->crl_off[k], len = b->crl_len[k];
        s->h_desc[st][k - ch.lo] = CrlDesc{off, (uint32_t)staged, (uint32_t)len, issuer[k], 0};
        if (run_len && run_src + run_len == off) {
            run_len += len;
        } else {
            if (run_len) CU(c, cudaMemcpyAsync(s->stage[st] + run_dst, b->data + run_src, run_len, cudaMemcpyHostToDevice, s->copy_stream));
            run_src = off;
            run_dst = staged;
            run_len = len;
        }
        staged += len;
    }
    if (run_len) CU(c, cudaMemcpyAsync(s->stage[st] + run_dst, b->data + run_src, run_len, cudaMemcpyHostToDevice, s->copy_stream));
    // bytes past the chunk: candidates and TLV reads stop at content ends, this keeps the tail defined
    CU(c, cudaMemsetAsync(s->stage[st] + staged, 0, 64, s->copy_stream));
    CU(c, cudaMemcpyAsync(s->desc[st], s->h_desc[st], (ch.hi - ch.lo) * sizeof(CrlDesc), cudaMemcpyHostToDevice, s->copy_stream));
    CU(c, cudaEventRecord(s->uploaded[st], s->copy_stream));
    return CTMR_OK;
}

// A group's member c (its device current) gets a bulk copy of the `slots` slots of member 0's set, on c's stream
int crl_set_copy(ctmr_ctx* c0, ctmr_ctx* c, uint64_t slots) {
    const int rc = crl_set_ensure(c, slots, false);
    if (rc) return rc;
    CU(c, cudaMemcpyPeerAsync(c->crl->set, c->device, c0->crl->set, c0->device, slots * sizeof(CrlSetSlot), c->stream));
    return CTMR_OK;
}

// The split of chunk `ch` in stage[st] on the ctx's stream, up to the compaction: *ne = the chunk's entries (epos, ecrl)
int crl_split(ctmr_ctx* c, const CrlChunk& ch, int st, uint32_t* ne_out) {
    CrlState* s = c->crl.get();
    cudaStream_t q = c->stream;
    const uint32_t n = (uint32_t)(ch.hi - ch.lo);
    const uint32_t bytes = (uint32_t)ch.bytes;
    const uint8_t* stage = s->stage[st];
    CU(c, cudaStreamWaitEvent(q, s->uploaded[st], 0));
    crl_frame_kernel<<<grid(n, 128), 128, 0, q>>>(stage, s->desc[st], n, s->res);
    CU(c, cudaGetLastError());
    const uint32_t groups = bytes / 16u + 2u;  // the last counter is 0: its scan value is the total
    crl_candidates_kernel<false><<<grid(groups, 256), 256, 0, q>>>(stage, bytes, groups, s->res, n, s->cnt16, nullptr, nullptr, nullptr, nullptr);
    CU(c, cudaGetLastError());
    size_t tb = s->temp_bytes;
    CU(c, cub::DeviceScan::ExclusiveSum(s->temp.get(), tb, s->cnt16.get(), s->off16.get(), (int)groups, q));
    crl_candidates_kernel<true><<<grid(groups, 256), 256, 0, q>>>(stage, bytes, groups, s->res, n, nullptr, s->off16, s->cpos, s->ccrl, s->link);
    CU(c, cudaGetLastError());
    uint32_t m_cand = 0;
    CU(c, cudaMemcpyAsync(&m_cand, s->off16 + (groups - 1), 4, cudaMemcpyDeviceToHost, q));
    CU(c, cudaStreamSynchronize(q));
    uint32_t cur = 0;
    if (m_cand) {
        crl_link_kernel<<<grid(m_cand, 256), 256, 0, q>>>(s->res, s->cpos, s->ccrl, m_cand, s->link, s->jump[0], s->mark);
        CU(c, cudaGetLastError());
        for (uint32_t r = 0; r < ch.rounds; ++r, cur ^= 1u) {
            crl_reach_kernel<<<grid(m_cand, 256), 256, 0, q>>>(s->jump[cur], s->jump[cur ^ 1u], s->mark, m_cand);
            CU(c, cudaGetLastError());
        }
        crl_check_kernel<<<grid(m_cand, 256), 256, 0, q>>>(stage, s->res, s->cpos, s->ccrl, s->link, s->mark, m_cand);
        CU(c, cudaGetLastError());
    }
    crl_settle_kernel<<<grid(n, 128), 128, 0, q>>>(s->desc[st], s->res, n);
    CU(c, cudaGetLastError());
    uint32_t ne = 0;
    if (m_cand) {
        crl_keep_kernel<<<grid(m_cand, 256), 256, 0, q>>>(s->res, s->ccrl, s->mark, m_cand, s->jump[0]);
        CU(c, cudaGetLastError());
        tb = s->temp_bytes;
        CU(c, cub::DeviceScan::ExclusiveSum(s->temp.get(), tb, s->jump[0].get(), s->jump[1].get(), (int)m_cand, q));
        crl_compact_kernel<<<grid(m_cand, 256), 256, 0, q>>>(s->res, s->cpos, s->ccrl, s->jump[0], s->jump[1], m_cand, s->epos, s->ecrl);
        CU(c, cudaGetLastError());
        uint32_t last[2] = {0, 0};
        CU(c, cudaMemcpyAsync(&last[0], s->jump[1] + (m_cand - 1), 4, cudaMemcpyDeviceToHost, q));
        CU(c, cudaMemcpyAsync(&last[1], s->jump[0] + (m_cand - 1), 4, cudaMemcpyDeviceToHost, q));
        CU(c, cudaStreamSynchronize(q));
        ne = last[0] + last[1];
    }
    *ne_out = ne;
    return CTMR_OK;
}

// the per-entry outputs of the chunk's ne entries to the caller's entries [at, at + ne), then its per-CRL fields; waits
int crl_copy_back(ctmr_ctx* c, ctmr_crl_out* out, const CrlChunk& ch, uint64_t at, uint32_t ne) {
    CrlState* s = c->crl.get();
    cudaStream_t q = c->stream;
    const uint32_t n = (uint32_t)(ch.hi - ch.lo);
    auto back = [&](void* dst, const void* src, size_t per) -> cudaError_t {
        if (!dst || !ne) return cudaSuccess;
        return cudaMemcpyAsync(static_cast<uint8_t*>(dst) + at * per, src, (size_t)ne * per, cudaMemcpyDeviceToHost, q);
    };
    CU(c, back(out->serial_off, s->eserial_off, 8));
    CU(c, back(out->serial_len, s->eserial_len, 1));
    CU(c, back(out->revoked_at, s->erevoked, 8));
    CU(c, back(out->reason, s->ereason, 1));
    CU(c, back(out->entry_status, s->estatus, 1));
    CU(c, back(out->known, s->eknown, 1));
    CU(c, back(out->known_exp_hour, s->ehour, 8));
    CU(c, back(out->known_sets, s->esets, 4));
    std::vector<CrlRes> res(n);
    CU(c, cudaMemcpyAsync(res.data(), s->res, n * sizeof(CrlRes), cudaMemcpyDeviceToHost, q));
    CU(c, cudaStreamSynchronize(q));
    uint64_t first = at;  // entries are in CRL order: a CRL's first is the count before it, also when it has none
    for (uint32_t k = 0; k < n; ++k) {
        const CrlRes& r = res[k];
        const uint64_t i = ch.lo + k;
        const bool listed = r.status == CTMR_CRL_OK || r.status == CTMR_CRL_UNKNOWN_ISSUER;
        if (out->crl_status) out->crl_status[i] = (uint8_t)r.status;
        if (out->crl_flags) out->crl_flags[i] = (uint8_t)r.flags;
        if (out->this_update) out->this_update[i] = r.this_update;
        if (out->next_update) out->next_update[i] = r.next_update;
        if (out->tbs_off) out->tbs_off[i] = r.tbs_off;
        if (out->tbs_len) out->tbs_len[i] = r.tbs_len;
        if (out->issuer_name_off) out->issuer_name_off[i] = r.name_off;
        if (out->issuer_name_len) out->issuer_name_len[i] = r.name_len;
        if (out->crl_entries) out->crl_entries[i] = listed ? r.count : 0u;
        if (out->crl_first) out->crl_first[i] = first;
        first += listed ? r.count : 0u;
    }
    return CTMR_OK;
}

EntryOut entry_out(CrlState* s) {
    return EntryOut{s->eserial_off, s->eserial_len, s->ereason, s->estatus, s->eknown, s->erevoked, s->ehour, s->eslot, s->esets};
}

// the per-entry outputs of a parsed chunk's ne entries, on c's stream
int crl_entries(ctmr_ctx* c, int st, uint32_t ne) {
    CrlState* s = c->crl.get();
    crl_entry_kernel<<<grid(ne, 256), 256, 0, c->stream>>>(s->stage[st], s->desc[st], s->res, s->epos, s->ecrl, ne, entry_out(s));
    CU(c, cudaGetLastError());
    return CTMR_OK;
}

// The entries of the chunk in stage[st] (ne of them, ne > 0) parsed, and the set of their (issuer, serial) pairs built on
// c's stream; *slots = the set's slots (its whole allocation: every member of a group probes with the same mask).
// `recv`: a group's member 0 also receives the other members' answers.
int crl_set_build(ctmr_ctx* c, int st, uint32_t ne, bool recv, uint64_t* slots) {
    CrlState* s = c->crl.get();
    int rc = crl_entries(c, st, ne);
    if (rc) return rc;
    uint64_t n = 64;
    while (n < 2ull * ne) n <<= 1;
    if ((rc = crl_set_ensure(c, n, recv))) return rc;
    n = s->set_cap;
    CU(c, cudaMemsetAsync(s->set, 0, n * sizeof(CrlSetSlot), c->stream));
    crl_set_insert_kernel<<<grid(ne, 256), 256, 0, c->stream>>>(s->stage[st], s->desc[st], s->res, s->ecrl, s->eserial_off, s->eserial_len,
                                                                 s->estatus, ne, s->set, n - 1, s->eslot);
    CU(c, cudaGetLastError());
    *slots = n;
    return CTMR_OK;
}

// The checks every call makes before any work: the arguments, and each CRL inside data and no larger than a chunk
int crl_check_batch(ctmr_ctx* c, const ctmr_crl_batch* b, const void* out, const std::string& call) {
    if (!b || !out) return fail(c, CTMR_E_INVALID, call + "NULL batch or output");
    if (b->n_crls && (!b->data || !b->crl_off || !b->crl_len || !b->issuer_digest))
        return fail(c, CTMR_E_INVALID, call + "NULL input array");
    const uint64_t B = crl_budget(c);
    for (uint64_t k = 0; k < b->n_crls; ++k) {
        const uint64_t off = b->crl_off[k], len = b->crl_len[k];
        if (off > b->data_bytes || len > b->data_bytes - off)
            return fail(c, CTMR_E_INVALID, call + "CRL " + std::to_string(k) + " lies outside data");
        if (len > B)
            return fail(c, CTMR_E_BATCH_TOO_LARGE, call + "CRL " + std::to_string(k) + " (" + std::to_string(len) +
                                                       " bytes) exceeds the staging budget of " + std::to_string(B) + " bytes");
    }
    return CTMR_OK;
}

// the issuers' dense indices: read from the registry, never registered here
int crl_issuers(ctmr_ctx* c, const ctmr_crl_batch* b, std::vector<uint32_t>& issuer) {
    issuer.assign(b->n_crls, CTMR_ISSUER_NONE);
    for (uint64_t k = 0; k < b->n_crls; ++k) {
        uint32_t idx = 0;
        bool found = false;
        const int rc = lookup_digest(c, b->issuer_digest + 32 * k, false, &idx, &found);
        if (rc) return rc;
        issuer[k] = found ? idx : CTMR_ISSUER_NONE;
    }
    return CTMR_OK;
}

// the batch cut into chunks of whole CRLs of at most the budget's bytes
std::vector<CrlChunk> crl_cut(ctmr_ctx* c, const ctmr_crl_batch* b) {
    const uint64_t B = crl_budget(c);
    std::vector<CrlChunk> chunks;
    for (uint64_t k = 0; k < b->n_crls;) {
        CrlChunk ch;
        ch.lo = k;
        uint64_t most = 0;
        while (k < b->n_crls && k - ch.lo < kCrlsPerChunk && ch.bytes + b->crl_len[k] <= B) {
            ch.bytes += b->crl_len[k];
            most = b->crl_len[k] > most ? b->crl_len[k] : most;
            ++k;
        }
        ch.hi = k;
        const uint64_t chain = most / kMinEntry + 1;  // no chain of well-formed entries is longer
        while ((1ull << ch.rounds) < chain) ++ch.rounds;
        chunks.push_back(ch);
    }
    return chunks;
}

// Every chunk of the batch (n_crls > 0) staged on the copy stream, the next one while chunk(ch, st) works on the current
// one in stage[st] on c's stream.  No upload outlives the call, whatever chunk returns.
int crl_for_chunks(ctmr_ctx* c, const ctmr_crl_batch* b, const std::vector<uint32_t>& issuer,
                   const std::function<int(const CrlChunk&, int)>& chunk) {
    int rc = crl_ensure(c);
    if (rc) return rc;
    const std::vector<CrlChunk> chunks = crl_cut(c, b);
    rc = crl_upload(c, b, issuer, chunks[0], 0);
    for (size_t i = 0; i < chunks.size() && rc == CTMR_OK; ++i) {
        if (i + 1 < chunks.size()) rc = crl_upload(c, b, issuer, chunks[i + 1], (int)((i + 1) & 1));
        if (rc == CTMR_OK) rc = chunk(chunks[i], (int)(i & 1));
    }
    const cudaError_t e = cudaStreamSynchronize(c->crl->copy_stream);
    if (rc == CTMR_OK && e != cudaSuccess) rc = fail(c, CTMR_E_CUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
    return rc;
}

// the CTMR_CRL_* of chunk ch's CRLs, parsed on c, into status[ch.lo, ch.hi); waits for c's stream
int crl_read_status(ctmr_ctx* c, const CrlChunk& ch, std::vector<uint8_t>& status) {
    const uint32_t n = (uint32_t)(ch.hi - ch.lo);
    std::vector<CrlRes> res(n);
    CU(c, cudaMemcpyAsync(res.data(), c->crl->res, n * sizeof(CrlRes), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    for (uint32_t k = 0; k < n; ++k) status[ch.lo + k] = (uint8_t)res[k].status;
    return CTMR_OK;
}

// What a call does with each chunk of its batch, in both forms' drivers (crl_group_chunks, crl_peer_steps):
// ctmr_revoked_known joins the entries and gathers their answers, ctmr_revoked_cascade marks every shard.
struct CrlActions {
    std::function<bool(uint32_t ne)> take;  // the chunk parsed with ne entries: are they joined (false: only counted)
    CrlSetVisit visit;     // a shard against a set: a member's copy of the chunk's set, or a peer rank's union set of a round
    bool answers = false;  // each joined entry's answer is gathered from the visits' hour and count arrays
    std::function<int(const CrlChunk& ch, uint32_t ne)> done;  // after chunk ch (ne entries), its last read of the stage issued
};

// The answers of one ctx or a group, after every member's visit: each other member's (hour, count) into member 0's
// recv_* and merged there, one member at a time in member order, then each entry's answer.  On error *at names the
// member that failed.
int crl_group_answers(ctmr_ctx* const* m, uint32_t W, uint64_t slots, uint32_t ne, ctmr_ctx** at) {
    ctmr_ctx* c0 = m[0];
    CrlState* s0 = c0->crl.get();
    for (uint32_t r = 1; r < W; ++r) {
        ctmr_ctx* c = *at = m[r];
        CU(c, cudaSetDevice(c->device));
        CU(c, cudaMemcpyPeerAsync(s0->recv_hour, c0->device, c->crl->set_hour, c->device, slots * sizeof(int32_t), c->stream));
        CU(c, cudaMemcpyPeerAsync(s0->recv_count, c0->device, c->crl->set_count, c->device, slots * sizeof(uint32_t), c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        *at = c0;
        CU(c0, cudaSetDevice(c0->device));
        crl_merge_kernel<<<grid(slots, 256), 256, 0, c0->stream>>>(s0->set_hour, s0->set_count, s0->recv_hour, s0->recv_count, slots);
        CU(c0, cudaGetLastError());
        CU(c0, cudaStreamSynchronize(c0->stream));
    }
    crl_finish_kernel<<<grid(ne, 256), 256, 0, c0->stream>>>(s0->eslot, s0->set_hour, s0->set_count, ne, entry_out(s0));
    CU(c0, cudaGetLastError());
    return CTMR_OK;
}

// One ctx or a group of W members: member 0 parses each chunk and builds the set of the entries it takes, every other
// member gets a bulk copy of the set (cudaMemcpyPeerAsync), and each member visits its copy on its own stream; with
// answers, crl_group_answers follows.  Synchronous; no upload outlives it.  The first failure goes to `local` and stops
// the call; false: it failed (here, or before).  No atomic crosses a GPU.
bool crl_group_chunks(ctmr_ctx* const* m, uint32_t W, const ctmr_crl_batch* b, const std::vector<uint32_t>& issuer, const CrlActions& a,
                      PeerLocal& local) {
    if (local.code) return false;
    if (b->n_crls == 0) return true;
    ctmr_ctx *c0 = m[0], *at = c0;
    const int rc = crl_for_chunks(c0, b, issuer, [&](const CrlChunk& ch, int st) -> int {
        uint32_t ne = 0;
        uint64_t slots = 0;
        int rc2 = crl_split(c0, ch, st, &ne);
        const bool sets = rc2 == CTMR_OK && a.take(ne) && ne;
        if (sets) rc2 = crl_set_build(c0, st, ne, a.answers && W > 1, &slots);
        if (rc2) return rc2;
        CU(c0, cudaEventRecord(c0->crl->consumed[st], c0->stream));
        if (sets) {
            if (W > 1) CU(c0, cudaStreamSynchronize(c0->stream));  // the other members copy member 0's set
            for (uint32_t r = 0; r < W; ++r) {
                ctmr_ctx* c = at = m[r];
                CU(c, cudaSetDevice(c->device));
                if (r && (rc2 = crl_set_copy(c0, c, slots))) return rc2;
                CrlState* s = c->crl.get();
                if ((rc2 = a.visit(c, CrlSet{s->set, slots - 1, s->set_hour, s->set_count}))) return rc2;
            }
            for (uint32_t r = W; r-- > 1;) {  // the next chunk rewrites member 0's set
                ctmr_ctx* c = at = m[r];
                CU(c, cudaSetDevice(c->device));
                CU(c, cudaStreamSynchronize(c->stream));
            }
            at = c0;
            CU(c0, cudaSetDevice(c0->device));
            if (a.answers && (rc2 = crl_group_answers(m, W, slots, ne, &at))) return rc2;
        }
        return a.done(ch, ne);
    });
    local.fail(at, rc);
    return rc == CTMR_OK;
}

// ---- one process per GPU: the collective call on a ctx attached to peers (include/ctmr.h states the rules) -----------
// Every rank checks its batch and builds its buffers, then agreement 1 posts its chunk count (or that it failed).  For
// each step k below the most chunks any rank has, a rank with a chunk k parses it (one without has no entries),
// agreement 2 posts how many entries it sends, and ceil(the largest count / X) rounds follow:
//     send:  each rank's next <= X entries as records, built from the staged chunk, into its region on EVERY rank (the
//            hour is unknown: no owner routing) + count
//     -- barrier: every region of the round has landed --
//     owner: the valid records received into the union set, one pass over the own shard, each record's answer in place
//     -- barrier: every owner's answers are in --
//     pull:  each rank reads its records' answers from every owner: the lowest hour, the sum of the counts
// One parity of the regions is enough because the rounds are synchronous: a source writes round j + 1 into its regions
// only after its own pull of round j (stream order), and every owner's reads and answers of round j came before the
// second barrier of round j, which the source has passed.  A final agreement makes any later failure every rank's.

// entries [lo, lo + n) of the chunk in stage[st] as records, sent to every rank with the count (n == 0: the count only)
int crl_peer_send(ctmr_ctx* c, int st, uint64_t lo, uint64_t n) {
    CrlState* s = c->crl.get();
    if (n) {
        crl_peer_records_kernel<<<grid(n, 256), 256, 0, c->stream>>>(s->stage[st], s->desc[st], s->res, s->ecrl, s->eserial_off,
                                                                     s->eserial_len, s->estatus, (uint32_t)lo, (uint32_t)n, s->records);
        CU(c, cudaGetLastError());
    }
    crl_peer_send_kernel<<<dim3(grid(4 * (n ? n : 1), 256), c->px.world), 256, 0, c->stream>>>(c->px, s->records, n);
    CU(c, cudaGetLastError());
    return CTMR_OK;
}

// the owner's part of a round: the round's valid records (agreed.n[s] from source s, `total` of them, at most `most` from
// one source) into the union set, the call's visit of the own shard, and with answers each record's answer in place
int crl_peer_owner(ctmr_ctx* c, const CrlRoundCounts& agreed, uint64_t most, uint64_t total, const CrlActions& a) {
    CrlState* s = c->crl.get();
    const dim3 g(grid(most, 256), c->px.world);
    const uint64_t slots = pow2_at_least(2 * total > 64 ? 2 * total : 64);  // <= union_cap: total <= world X
    CU(c, cudaMemsetAsync(s->union_set, 0, slots * sizeof(CrlSetSlot), c->stream));
    crl_union_insert_kernel<<<g, 256, 0, c->stream>>>(c->px, agreed, s->union_set, slots - 1, c->in_slot);
    CU(c, cudaGetLastError());
    const int rc = a.visit(c, CrlSet{s->union_set, slots - 1, s->union_hour, s->union_count});
    if (rc || !a.answers) return rc;
    crl_peer_answer_kernel<<<g, 256, 0, c->stream>>>(c->px, agreed, c->in_slot, s->union_hour, s->union_count);
    CU(c, cudaGetLastError());
    return CTMR_OK;
}

// Round j of a step whose sent entries are row[0..world), this rank's chunk in stage[st]; with answers, the rank pulls
// the answers to the entries it sent.  `work` false (this rank failed): nothing but the two barriers, which every rank
// issues whatever happens, so that a failure never leaves another rank waiting.
int crl_peer_round(ctmr_ctx* c, const uint64_t* row, uint64_t j, bool work, int st, const CrlActions& a) {
    const uint64_t X = c->px.X, lo = j * X;
    const auto in_round = [&](uint64_t n) -> uint64_t { return n > lo ? std::min(X, n - lo) : 0; };
    CrlRoundCounts agreed{};
    uint64_t most = 0, total = 0;
    for (uint32_t r = 0; r < c->px.world; ++r) {
        agreed.n[r] = in_round(row[r]);
        most = std::max<uint64_t>(most, agreed.n[r]);
        total += agreed.n[r];
    }
    const uint64_t mine = agreed.n[c->px.rank];
    int rc = work ? crl_peer_send(c, st, lo, mine) : CTMR_OK;
    int brc = peer_barrier(c, CH_CRL, c->stream);
    if (rc == CTMR_OK) rc = brc;
    if (rc == CTMR_OK && work && total) rc = crl_peer_owner(c, agreed, most, total, a);
    brc = peer_barrier(c, CH_CRL, c->stream);
    if (rc == CTMR_OK) rc = brc;
    if (rc || !work || !mine || !a.answers) return rc;
    CrlState* s = c->crl.get();
    crl_peer_pull_kernel<<<grid(mine, 256), 256, 0, c->stream>>>(c->px, mine, lo, s->eknown, s->ehour, s->esets);
    CU(c, cudaGetLastError());
    return CTMR_OK;
}

// A peer rank's steps after agreement 1 (row: every rank's chunk count), up to the final agreement (crl_peer_finish).  A
// failure of this rank goes to `local`; false: a rank's failure stopped the steps early (every rank saw it in the same
// agreement 2), and the ranks go straight to the final agreement.
bool crl_peer_steps(ctmr_ctx* c, const ctmr_crl_batch* b, const std::vector<uint32_t>& issuer, uint64_t* row, const CrlActions& a,
                    PeerLocal& local) {
    const std::vector<CrlChunk> chunks = crl_cut(c, b);
    const uint32_t W = c->st.peer.world;
    uint64_t steps = 0;
    for (uint32_t r = 0; r < W; ++r) steps = std::max(steps, row[r]);
    CrlState* s = c->crl.get();
    int rc = CTMR_OK;
    if (!chunks.empty() && !local.code && (rc = crl_upload(c, b, issuer, chunks[0], 0))) local.fail(c, rc);
    for (uint64_t k = 0; k < steps; ++k) {
        const int st = (int)(k & 1);
        const bool mine = k < chunks.size() && !local.code;
        uint32_t ne = 0;
        uint64_t send = 0;
        if (mine) {
            rc = k + 1 < chunks.size() ? crl_upload(c, b, issuer, chunks[k + 1], st ^ 1) : CTMR_OK;
            if (rc == CTMR_OK) rc = crl_split(c, chunks[k], st, &ne);
            if (rc == CTMR_OK && a.take(ne) && ne) {
                rc = crl_entries(c, st, ne);
                send = ne;
            }
            if (rc) local.fail(c, rc);
        }
        rc = peer_mailbox(c, peer_word(local.code, send), row);  // agreement 2
        if (rc) {
            local.fail(c, rc);
            return false;
        }
        if (peer_row_failed(row, W) < W) return false;  // every rank saw the same row: all go to the final agreement
        uint64_t most = 0;
        for (uint32_t r = 0; r < W; ++r) most = std::max(most, row[r]);
        for (uint64_t j = 0; j * c->px.X < most; ++j)  // the rounds build their records from the staged chunk
            if ((rc = crl_peer_round(c, row, j, !local.code, st, a))) local.fail(c, rc);
        if (!mine || local.code) continue;
        if (cudaEventRecord(s->consumed[st], c->stream) != cudaSuccess) {  // the rounds' last read of stage[st] is issued
            local.fail(c, fail(c, CTMR_E_CUDA, "cudaEventRecord failed"));
            continue;
        }
        if ((rc = a.done(chunks[k], ne))) local.fail(c, rc);
    }
    return true;
}

// every chunk of the batch through the form's driver: one ctx or a group, or a peer rank after agreement 1
bool crl_chunks(ctmr_ctx* const* m, uint32_t W, bool peer, const ctmr_crl_batch* b, const std::vector<uint32_t>& issuer, uint64_t* row,
                const CrlActions& a, PeerLocal& local) {
    return peer ? crl_peer_steps(m[0], b, issuer, row, a, local) : crl_group_chunks(m, W, b, issuer, a, local);
}

// ---- the call ---------------------------------------------------------------------------------------------------------
// One driver answers the call on the members this process holds: a group's W members, one ctx (W == 1), or one rank of
// a group of processes (W == 1; the call is collective, include/ctmr.h states the rules).  Only these steps differ:
//   checks   one ctx or a group: a failure returns at once, and n_entries is 0 once the checks pass.  A peer rank:
//            n_entries is 0 first; the checks and every buffer of the call travel in agreement 1 with its chunk count.
//   answers  one ctx or a group: crl_group_answers.  A peer rank: each owner answers the records it received in a round
//            (crl_peer_answer), and each source pulls its records' answers from every owner (crl_peer_pull).
//   finish   one ctx or a group: its first failure, with the failing member's text.  A peer rank: crl_peer_finish.
// The entry_cap rule holds in every form: once the entries do not fit, later chunks are only counted, and a peer rank
// still answers the other ranks' records.
int revoked_known(ctmr_ctx* const* m, uint32_t W, ctmr_group* g, const ctmr_crl_batch* b, ctmr_crl_out* out) {
    ctmr_ctx* c0 = m[0];
    const bool peer = peer_call(c0);
    const char* call = "ctmr_revoked_known: ";
    CU(c0, cudaSetDevice(c0->device));
    if (peer && out) out->n_entries = 0;
    std::vector<uint32_t> issuer;
    uint64_t n_chunks = 0, row[kMaxWorld] = {};
    int rc = crl_prepare(c0, b, out, call, issuer, &n_chunks);
    if (peer) rc = peer_agree(c0, rc, n_chunks, row, call, "collective call failed");  // agreement 1
    if (rc) return group_fail(g, c0, rc);
    out->n_entries = 0;
    uint64_t base = 0;  // entries placed so far
    bool count_only = false;
    PeerLocal local;
    CrlActions a;
    a.take = [&](uint32_t ne) {
        if (count_only || base + ne > out->entry_cap) count_only = true;
        return !count_only;
    };
    a.visit = [](ctmr_ctx* c, const CrlSet& set) -> int {  // every key whose pair is in the set takes the lowest hour and counts
        CU(c, cudaMemsetAsync(set.hour, 0x7f, (set.mask + 1) * sizeof(int32_t), c->stream));
        CU(c, cudaMemsetAsync(set.count, 0, (set.mask + 1) * sizeof(uint32_t), c->stream));
        crl_known_scan_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->st.table, c->st.table_mask + 1, c->st.epoch, set.slots, set.mask, set.hour,
                                                                          set.count);
        CU(c, cudaGetLastError());
        return CTMR_OK;
    };
    a.answers = true;
    a.done = [&](const CrlChunk& ch, uint32_t ne) {  // per-entry outputs straight into the caller's arrays
        const int rc2 = count_only ? CTMR_OK : crl_copy_back(c0, out, ch, base, ne);
        base += ne;
        return rc2;
    };
    crl_chunks(m, W, peer, b, issuer, row, a, local);
    rc = peer ? crl_peer_finish(c0, local, 0, row, call) : local.code;
    if (rc) {
        if (g) g->err = local.err;  // the failing member's text is the group's
        return rc;
    }
    out->n_entries = base;
    if (count_only)
        return group_fail(g, c0, fail(c0, CTMR_E_BATCH_TOO_LARGE, std::string(call) + "entry_cap " + std::to_string(out->entry_cap) + " < " +
                                                               std::to_string(base) + " entries"));
    return CTMR_OK;
}

}  // namespace

// ---- the chunk path as ctmr_revoked_cascade and ctmr_revoked_stash use it (ctmr_cascade.cu) ---------------------------
namespace ctmr_host {

int crl_prepare(ctmr_ctx* c, const ctmr_crl_batch* b, const void* out, const char* call, std::vector<uint32_t>& issuer,
                uint64_t* n_chunks) {
    *n_chunks = 0;
    int rc = crl_check_batch(c, b, out, call);
    if (rc == CTMR_OK) rc = crl_issuers(c, b, issuer);
    if (rc || !peer_call(c)) return rc;
    rc = crl_ensure(c);
    if (rc == CTMR_OK) rc = crl_peer_ensure(c);
    if (rc == CTMR_OK) *n_chunks = crl_cut(c, b).size();
    return rc;
}

bool crl_each_set(ctmr_ctx* const* m, uint32_t W, bool peer, const ctmr_crl_batch* b, const std::vector<uint32_t>& issuer, uint64_t* row,
                  const CrlSetVisit& visit, std::vector<uint8_t>& status, PeerLocal& local) {
    CrlActions a;
    a.take = [](uint32_t) { return true; };
    a.visit = visit;
    a.done = [&](const CrlChunk& ch, uint32_t) { return crl_read_status(m[0], ch, status); };
    return crl_chunks(m, W, peer, b, issuer, row, a, local);
}

int crl_peer_finish(ctmr_ctx* c, PeerLocal& local, uint64_t payload, uint64_t* row, const char* call) {
    const cudaStream_t drain[] = {c->crl->copy_stream, c->stream};
    drain_streams(c, drain, 2);  // no upload may read the caller's data after the call
    int rc = CTMR_OK;
    if (!local.code && (rc = ctmr_check_device(c, nullptr))) local.fail(c, rc);  // a barrier of a round that timed out
    if (local.code) c->err = local.err;
    return peer_agree(c, local.code, payload, row, call, "collective call failed");  // the final agreement
}

}  // namespace ctmr_host

extern "C" {

int ctmr_revoked_known(ctmr_ctx* c, const ctmr_crl_batch* batch, ctmr_crl_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group) return fail(c, CTMR_E_INVALID, "ctmr_revoked_known: a member of a group; use ctmr_group_revoked_known");
    ctmr_ctx* m[1] = {c};
    return revoked_known(m, 1, nullptr, batch, out);
}

int ctmr_group_revoked_known(ctmr_group* g, const ctmr_crl_batch* batch, ctmr_crl_out* out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const int rc = revoked_known(g->m.data(), (uint32_t)g->m.size(), g, batch, out);
    cudaSetDevice(g->m[0]->device);
    return rc;
}

}  // extern "C"
