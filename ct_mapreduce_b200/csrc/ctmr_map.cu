// ctmr_map.cu -- the map half of the CT-entry hot path: hand-written sm_90a kernels.
//
// K_map        (map_stream_kernel) lane-per-certificate map: DER walk + certIsFilteredOut + SHA-256(leaf DER).
//              Each lane streams ITS certificate through a private two-chunk shared-memory ring filled by
//              asynchronous 16-byte global->shared copies (cp.async.cg -> SASS LDGSTS, per-thread commit / wait groups: no
//              barrier is shared between lanes), so certificate bytes never occupy registers while the INT pipe runs the
//              64-round compression; the resumable walker (ctmr_stream.cuh) eats from the same ring.  Epilogue: filter,
//              outputs, key record, and the key's route -- fused find-or-insert into this GPU's table when it owns the set,
//              else an append to the owner GPU's inbox over NVLink (route_append).
//              (cmd/ct-fetch/ct-fetch.go:44-70,198-213, storage/types.go:171-178,339-346; fingerprint =
//              crypto/sha256.Sum256(cert.Raw).)
// K_map_light  (map_light_kernel) the same outputs without the fingerprint: thread per certificate, loads through L1.
// length bucketing (len_hist / len_scan / len_scatter): processing order with equally long records per warp.
// sha_ceiling_kernel: the register-only SHA-256 microbenchmark the roofline is quoted against.
// The reduce half (K_insert / K_resolve / K_pairs, string identities, the owner and source passes of the multi-GPU key
// exchange, the issuer registry, the peer barrier) lives in ctmr_reduce.cu.
#include "ctmr_common.cuh"
#include "ctmr_stream.cuh"

namespace ctmr {

// Appends the finished 64-byte key record `kr` (local memory) of an entry owned by another GPU to that owner's inbox:
// lanes of the warp that route to the same owner take consecutive positions from ONE atomic on a cursor in LOCAL
// memory, so the records of a (warp, owner) group form one contiguous run of posted NVLink writes.  rev[] remembers
// which entry sits at which inbox position (the result bits come back by position).  Called by every lane that is
// inside the caller's active region, remote or not.
__device__ __forceinline__ void route_append(const RouteOut& r, bool remote, uint32_t owner, const uint4* kr, uint32_t entry) {
    if (r.world <= 1u) return;
    const uint32_t rmask = __ballot_sync(__activemask(), remote);
    if (!remote) return;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t peers = __match_any_sync(rmask, owner);
    const uint32_t leader = (uint32_t)__ffs(peers) - 1u;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(r.cursor + owner, (unsigned long long)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    const uint64_t i = base + __popc(peers & ((1u << lane) - 1u));
    if (i >= r.X) return;  // cannot happen: the host checks entries-per-round <= X
    const uint4 q0 = kr[0], q1 = kr[1], q2 = kr[2], q3 = kr[3];
    uint4* dst = reinterpret_cast<uint4*>(r.inbox[owner] + i);
    dst[0] = q0; dst[1] = q1; dst[2] = q2; dst[3] = q3;
    r.rev[(uint64_t)owner * r.X + i] = entry;
}

// ------------------------------------------------------------------------------------------------
// K_map_light: the map WITHOUT the whole-certificate fingerprint (CTMR_F_NO_FINGERPRINT, i.e. the
// reference's own semantics: it never hashes the leaf, SURVEY.md §0 M3).  With no SHA-256 there is
// nothing to stream: the walker touches ~1/3 of a certificate's 32-byte sectors (TBS header,
// names, validity, the extension headers, the trailing signature header) and skips the key,
// the padding and the signature.  So: no shared memory, one thread per certificate, byte loads
// through L1 (the full 256 KB is available as cache), 32 resident warps per SM to hide the pointer
// chase.  The streaming kernel, which must stage every byte, is slower on this path.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kLightPrefetchLines = 2;  // leading 128-byte lines of a record prefetched to L2

// 6 resident CTAs per SM (40 registers, a few bytes of spills) ran faster than 4 CTAs (56 registers) when measured before the
// port; 8 CTAs (32 registers) spill too much
__global__ void __launch_bounds__(256, 6) map_light_kernel(const __grid_constant__ MapParams p) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool act = e < p.n;
    uint32_t status = CTMR_ST_PARSE_ERR;
    if (act) {
        const uint64_t off = p.offsets[e], end = p.lens ? off + p.lens[e] : p.offsets[e + 1];
        const bool bad_span = end < off || end > p.blob_bytes || end - off > 0x7fffffffull;
        const uint32_t L = bad_span ? 0u : (uint32_t)(end - off);
        const uint8_t* d = p.blob + off;
        if (L) {
            // The walk is a pointer chase (latency bound, not bandwidth bound): start the lines it is going to need
            // first -- header, serial, names, validity -- before the first dependent load, so that they arrive in
            // parallel.  Two lines measured best before the port; a prefetch of the tail (signature header) did not pay.
            const uint8_t* base = reinterpret_cast<const uint8_t*>(reinterpret_cast<uint64_t>(d) & ~127ull);
            const uint32_t lines = (uint32_t)((d - base) + L + 127u) >> 7;
            const uint32_t nl = min(kLightPrefetchLines, lines);
            for (uint32_t i = 0; i < nl; ++i) asm volatile("prefetch.global.L2 [%0];" ::"l"(base + 128u * i));
        }
        ParsedCert pc;
        uint32_t issuer = CTMR_ISSUER_NONE;
        int64_t exp_hour = 0;
        if (!bad_span && parse_cert(d, L, pc)) {
            status = CTMR_ST_OK;
            exp_hour = pc.not_after >= 0 ? pc.not_after / 3600 : -((-pc.not_after + 3599) / 3600);
            if ((pc.flags & (PC_BC_VALID | PC_IS_CA)) == (PC_BC_VALID | PC_IS_CA)) {
                status = CTMR_ST_FILTER_CA;
            } else if (!p.filter.log_expired &&
                       (pc.not_after < p.now_sec || (pc.not_after == p.now_sec && p.now_frac_nonzero))) {
                status = CTMR_ST_FILTER_EXPIRED;
            } else if (p.filter.filter_nonempty) {
                bool skip = true;
                const uint32_t cnl = (pc.flags & PC_HAS_CN) ? pc.cn_len : 0u;
                for (uint32_t q = 0; q < p.filter.n_prefix && skip; ++q) {
                    const uint32_t po = p.filter.off[q], pl = p.filter.off[q + 1] - po;
                    if (pl > cnl) continue;
                    bool eq = true;
                    for (uint32_t i = 0; i < pl; ++i)
                        if (__ldg(d + pc.cn_off + i) != p.filter.bytes[po + i]) { eq = false; break; }
                    if (eq) skip = false;
                }
                if (skip) status = CTMR_ST_FILTER_CN;
            }
            if (status == CTMR_ST_OK) {
                uint32_t k = p.issuer_idx ? p.issuer_idx[e] : CTMR_ISSUER_NONE;
                if (k != CTMR_ISSUER_NONE && p.issuer_map) k = k < p.issuer_map_len ? p.issuer_map[k] : CTMR_ISSUER_NONE;
                issuer = k;
                if (k == CTMR_ISSUER_NONE) status = CTMR_ST_NO_ISSUER;
                else if (k == CTMR_ISSUER_BAD) status = CTMR_ST_ISSUER_PARSE_ERR;
                else if (pc.serial_len > CTMR_MAX_SERIAL) status = CTMR_ST_SERIAL_TOO_LONG;
            }
        } else {
            pc.serial_off = pc.serial_len = 0;
            pc.issuer_off = pc.issuer_len = pc.crldp_off = pc.crldp_len = 0;
        }
        if (p.status) p.status[e] = (uint8_t)status;
        if (p.exp_hour) p.exp_hour[e] = exp_hour;
        if (p.serial_off) p.serial_off[e] = pc.serial_off;
        if (p.serial_len) p.serial_len[e] = pc.serial_len;
        if (p.issuer_name_off) {
            const bool okp = status != CTMR_ST_PARSE_ERR;
            p.issuer_name_off[e] = okp ? pc.issuer_off : 0u;
            p.issuer_name_len[e] = okp ? pc.issuer_len : 0u;
            p.crldp_off[e] = okp ? pc.crldp_off : 0u;
            p.crldp_len[e] = okp ? pc.crldp_len : 0u;
        }
        if (p.keys) {
            const bool valid = status == CTMR_ST_OK;
            uint32_t body[12];
#pragma unroll
            for (int i = 0; i < 12; ++i) body[i] = 0;
            if (valid) {
                body[0] = (uint32_t)(int32_t)exp_hour;
                body[1] = issuer;
                body[2] = pc.serial_len;
#pragma unroll 1
                for (uint32_t i = 0; i < pc.serial_len; ++i) {  // {len, serial[39]} packed little-endian from byte 8
                    const uint32_t at = i + 1u;
                    const uint32_t b = __ldg(d + pc.serial_off + i) << (8u * (at & 3u));
                    switch (at >> 2) {  // static register indices
                    case 0: body[2] |= b; break; case 1: body[3] |= b; break; case 2: body[4] |= b; break;
                    case 3: body[5] |= b; break; case 4: body[6] |= b; break; case 5: body[7] |= b; break;
                    case 6: body[8] |= b; break; case 7: body[9] |= b; break; case 8: body[10] |= b; break;
                    default: body[11] |= b; break;
                    }
                }
            }
            const uint64_t gi = p.first_index + e;
            uint4* kr = reinterpret_cast<uint4*>(p.keys + e);
            kr[0] = make_uint4((uint32_t)gi, (uint32_t)(gi >> 32), body[0], body[1]);
            kr[1] = make_uint4(body[2], body[3], body[4], body[5]);
            kr[2] = make_uint4(body[6], body[7], body[8], body[9]);
            kr[3] = make_uint4(body[10], body[11], valid ? 1u : 0u, 0u);
            if (p.slot_of) {
                const uint32_t owner = (valid && p.route.world > 1u) ? key_owner((int32_t)body[0], body[1], p.route.world) : p.route.rank;
                const bool remote = valid && owner != p.route.rank;
                p.slot_of[e] = (valid && !remote) ? known_insert<false>(p.table, p.table_mask, p.epoch, p.error_flag, body, ~gi) : 0xFFFFFFFFu;
                route_append(p.route, remote, owner, kr, (uint32_t)e);
            }
        }
    }
    if (p.status_counts) {
        const uint32_t amask = __ballot_sync(0xffffffffu, act);
        if (act) {
            const uint32_t peers = __match_any_sync(amask, status);
            if ((threadIdx.x & 31u) == (uint32_t)__ffs(peers) - 1u)
                atomicAdd(p.status_counts + status, (unsigned long long)__popc(peers));
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K_map v2: single-pass streaming map.  The DER walker (ctmr_stream.cuh) and the SHA-256 loop both
// eat from the same per-lane shared-memory ring of two chunks; global memory is touched once per
// byte, by asynchronous copies only, and every byte is copied once (ring_step in ctmr_common.cuh:
// the next chunk is copied after the walk, so the walker can still look back into the previous one).
// Staging: per-lane cp.async 16-byte copies (LDGSTS) + commit/wait groups -- no barrier at all.
// ------------------------------------------------------------------------------------------------
// Timing experiments (tools/kmap_split.py compiles this file into libraries of its own with one or both set; libctmr.so
// is built with neither): CTMR_KMAP_SKIP_WALK never calls the walker and stands a key made of the entry number in for
// the serial, CTMR_KMAP_SKIP_HASH folds each block's 16 words into the state with XORs instead of compressing them.
// Either makes the outputs wrong on purpose.
#ifndef CTMR_KMAP_SKIP_WALK
#define CTMR_KMAP_SKIP_WALK 0
#endif
#ifndef CTMR_KMAP_SKIP_HASH
#define CTMR_KMAP_SKIP_HASH 0
#endif
__global__ void __launch_bounds__(StreamCfg::kWarps * 32, StreamCfg::kCtasPerSm) map_stream_kernel(const __grid_constant__ MapParams p) {
    using Cfg = StreamCfg;
    constexpr int WARPS = Cfg::kWarps, CHUNK = Cfg::kChunk;
    static_assert(Cfg::kRing == (int)kRingBytes && CHUNK >= (int)kWalkNeed + 16, "ring geometry");
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint8_t* my_ring = smem + (size_t)warp * Cfg::kWarpBytes + (size_t)lane * Cfg::kLaneBytes;
    const uint32_t ring = smem_u32(my_ring);

    const uint64_t ngroups = (p.n + 31) >> 5;
    const bool want_sha = p.sha256 != nullptr;
    for (uint64_t g = (uint64_t)blockIdx.x * WARPS + warp; g < ngroups; g += (uint64_t)gridDim.x * WARPS) {
        const uint64_t pos = g * 32 + lane;
        const bool act = pos < p.n;
        // length-bucketed assignment: the 32 records of a warp have (nearly) the same number of chunks
        const uint64_t e = act ? (p.order ? (uint64_t)p.order[pos] : pos) : 0;
        uint64_t off = 0, end = 0;
        if (act) {
            off = p.offsets[e];
            end = p.lens ? off + p.lens[e] : p.offsets[e + 1];
        }
        const bool bad_span = !act || end < off || end > p.blob_bytes || end - off > 0x7fffffffull;
        const uint32_t L = bad_span ? 0u : (uint32_t)(end - off);
        const uint8_t* d = p.blob + off;
        const uint64_t addr = reinterpret_cast<uint64_t>(d);
        const uint32_t m = (uint32_t)(addr & 15u);
        const uint8_t* src_base = reinterpret_cast<const uint8_t*>(addr & ~15ull);
        const uint32_t nfull = L >> 6;
        const uint32_t nb = want_sha && act ? nfull + 1u + ((L & 63u) >= 56u ? 1u : 0u) : 0u;
        const uint32_t ndata = act ? (L + CHUNK - 1) / CHUNK : 0u;
        uint32_t nch = (nb + Cfg::kBlocksPerChunk - 1) / Cfg::kBlocksPerChunk;
        nch = nch > ndata ? nch : ndata;                    // without SHA the walker alone drives the stream
        if (act && nch == 0u) nch = 1u;                     // empty record: one step so that the walker reports the error
        const uint32_t iters = warp_max_u32(nch);
        const uint32_t yend = L ? (m + L + 15u) >> 4 : 0u;  // source granules holding record bytes

        // source granules [y0, y1) to their ring slots (the range never crosses the ring's end); the ring's
        // first granule also goes to the mirror behind the ring
        auto copy = [&](uint32_t y0, uint32_t y1) {
            const uint8_t* src = src_base + 16u * y0;
            const uint32_t dst = ring + ((16u * y0) & (Cfg::kRing - 1u));
            if (y0 < y1 && dst == ring) cp_async16(ring + Cfg::kRing, src);
#pragma unroll 1
            for (uint32_t j = 0; j < 16u * (y1 - y0); j += 16u) cp_async16(dst + j, src + j);
        };
        {
            const RingCopy r0 = ring_chunk_copy(0u, m, yend);
            copy(r0.y0, r0.y1);
            cp_async_commit();
        }

        Walker w;
        w.init();
        uint32_t* key_words = (p.keys && act) ? reinterpret_cast<uint32_t*>(p.keys + e) + 4 : nullptr;
        const GlobalBytes far{d};
        Sha256State st;
        st.init();
        const uint32_t sel = 0x0123u + 0x1111u * (m & 3u);
        const uint32_t one = p.one;

        for (uint32_t c = 0; c < iters; ++c) {
            cp_async_wait<0>();  // chunk c has landed
            if (c < nch) {
                // ---- map: resume the TLV walk over the newly staged bytes
                auto walk = [&] {
                    if (!CTMR_KMAP_SKIP_WALK && act && w.st < W_DONE) {
                        const uint32_t avail = min((c + 1u) * CHUNK, L);
                        walk_advance(w, SmemWindow{ring, m}, far, bad_span ? 0u : avail, L, p.filter, key_words);
                    }
                };
                // ---- fingerprint: the chunk's 64-byte blocks, whose words start at ring offset (c*CHUNK + m) mod kRing
                auto hash = [&] {
#pragma unroll 1
                    for (uint32_t bb = 0; bb < (uint32_t)Cfg::kBlocksPerChunk; ++bb) {
                        const uint32_t b = c * Cfg::kBlocksPerChunk + bb;
                        if (b >= nb) break;
                        const uint32_t* sw = reinterpret_cast<const uint32_t*>(my_ring) + (((c & 1u) * CHUNK + m + 64u * bb) >> 2);
                        uint32_t x[17], wd[16];
#pragma unroll
                        for (int i = 0; i < 17; ++i) x[i] = sw[i];
#pragma unroll
                        for (int i = 0; i < 16; ++i) wd[i] = __byte_perm(x[i], x[i + 1], sel);
                        if (b >= nfull) {
#pragma unroll
                            for (int i = 0; i < 16; ++i) wd[i] = sha256_pad_word(wd[i], b * 64u + 4u * i, L);
                            if (b == nb - 1u) {
                                wd[14] = L >> 29;
                                wd[15] = L << 3;
                            }
                        }
#if CTMR_KMAP_SKIP_HASH
#pragma unroll
                        for (int i = 0; i < 16; ++i) st.h[i & 7] ^= wd[i];
#else
                        sha256_compress_rolled(st, wd, one);
#endif
                    }
                };
                ring_step(c, m, yend, walk, copy, hash);
                cp_async_commit();
            }
        }
        cp_async_wait<0>();  // nothing is in flight when the ring takes the warp's next records
#if CTMR_KMAP_SKIP_WALK
        if (act && !bad_span) {
            w.st = W_DONE;
            if (key_words) {
                key_words[0] = 4u | ((uint32_t)e << 8);
                key_words[1] = (uint32_t)e >> 24;
                for (int i = 2; i < 10; ++i) key_words[i] = 0u;
            }
        }
#endif

        // ---- certIsFilteredOut + Store preconditions, in the reference's order
        if (act) {
            uint32_t status = CTMR_ST_PARSE_ERR, issuer = CTMR_ISSUER_NONE;
            int64_t exp_hour = 0;
            uint32_t serial_off = 0, serial_len = 0;
            if (w.st == W_DONE) {
                status = CTMR_ST_OK;
                serial_off = w.serial_off;
                serial_len = w.serial_len;
                exp_hour = w.not_after >= 0 ? w.not_after / 3600 : -((-w.not_after + 3599) / 3600);
                if ((w.flags & (WF_BC_VALID | WF_IS_CA)) == (WF_BC_VALID | WF_IS_CA)) {
                    status = CTMR_ST_FILTER_CA;
                } else if (!p.filter.log_expired &&
                           (w.not_after < p.now_sec || (w.not_after == p.now_sec && p.now_frac_nonzero))) {
                    status = CTMR_ST_FILTER_EXPIRED;
                } else if (p.filter.filter_nonempty) {
                    // CommonName "" (no CN attribute) matches only an empty prefix
                    bool keep = (w.flags & WF_HAS_CN) ? (w.flags & WF_CN_MATCH) != 0 : false;
                    if (!(w.flags & WF_HAS_CN))
                        for (uint32_t q = 0; q < p.filter.n_prefix; ++q) keep |= p.filter.off[q + 1] == p.filter.off[q];
                    if (!keep) status = CTMR_ST_FILTER_CN;
                }
                if (status == CTMR_ST_OK) {
                    uint32_t k = p.issuer_idx ? p.issuer_idx[e] : CTMR_ISSUER_NONE;
                    if (k != CTMR_ISSUER_NONE && p.issuer_map) k = k < p.issuer_map_len ? p.issuer_map[k] : CTMR_ISSUER_NONE;
                    issuer = k;
                    if (k == CTMR_ISSUER_NONE) status = CTMR_ST_NO_ISSUER;
                    else if (k == CTMR_ISSUER_BAD) status = CTMR_ST_ISSUER_PARSE_ERR;
                    else if (serial_len > CTMR_MAX_SERIAL) status = CTMR_ST_SERIAL_TOO_LONG;
                }
            }
            if (p.status) p.status[e] = (uint8_t)status;
            if (p.exp_hour) p.exp_hour[e] = exp_hour;
            if (p.serial_off) p.serial_off[e] = serial_off;
            if (p.serial_len) p.serial_len[e] = serial_len;
            if (p.issuer_name_off) {  // spans of the strings IssuerMetadata.Accumulate looks at (SURVEY §8(f)-1)
                const bool okp = w.st == W_DONE;
                p.issuer_name_off[e] = okp ? w.name_off : 0u;
                p.issuer_name_len[e] = okp ? w.name_len : 0u;
                p.crldp_off[e] = okp ? w.crldp_off : 0u;
                p.crldp_len[e] = okp ? w.crldp_len : 0u;
            }
            if (p.keys) {
                const bool valid = status == CTMR_ST_OK;
                const uint64_t gi = p.first_index + e;
                uint4* kr = reinterpret_cast<uint4*>(p.keys + e);
                kr[0] = make_uint4((uint32_t)gi, (uint32_t)(gi >> 32), (uint32_t)(int32_t)exp_hour, valid ? issuer : 0u);
                *reinterpret_cast<uint2*>(reinterpret_cast<uint32_t*>(kr) + 14) = make_uint2(valid ? 1u : 0u, 0u);
                if (p.slot_of) {
                    // fused K_insert (single-GPU path): the probe's random HBM accesses hide under the
                    // INT-bound SHA work of the other warps instead of costing a latency-bound pass
                    uint32_t slot = 0xFFFFFFFFu;
                    const uint32_t owner = (valid && p.route.world > 1u) ? key_owner((int32_t)exp_hour, issuer, p.route.world) : p.route.rank;
                    const bool remote = valid && owner != p.route.rank;
                    if (valid && !remote) {
                        const uint4 k1 = kr[1], k2 = kr[2];  // the serial words the walker stored (L2-resident)
                        const uint2 k3 = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint32_t*>(kr) + 12);
                        const uint32_t body[12] = {(uint32_t)(int32_t)exp_hour, issuer, k1.x, k1.y, k1.z, k1.w,
                                                   k2.x, k2.y, k2.z, k2.w, k3.x, k3.y};
                        slot = known_insert<false>(p.table, p.table_mask, p.epoch, p.error_flag, body, ~gi);
                    }
                    p.slot_of[e] = slot;
                    route_append(p.route, remote, owner, kr, (uint32_t)e);  // keys owned elsewhere: into the owner's inbox over NVLink
                }
            }
            if (want_sha) {
                uint4* o = reinterpret_cast<uint4*>(p.sha256 + e * 32);
                o[0] = make_uint4(__byte_perm(st.h[0], 0, 0x0123), __byte_perm(st.h[1], 0, 0x0123),
                                  __byte_perm(st.h[2], 0, 0x0123), __byte_perm(st.h[3], 0, 0x0123));
                o[1] = make_uint4(__byte_perm(st.h[4], 0, 0x0123), __byte_perm(st.h[5], 0, 0x0123),
                                  __byte_perm(st.h[6], 0, 0x0123), __byte_perm(st.h[7], 0, 0x0123));
            }
            if (p.status_counts) {
                const uint32_t peers = __match_any_sync(__activemask(), status);
                if ((uint32_t)lane == (uint32_t)__ffs(peers) - 1u)
                    atomicAdd(p.status_counts + status, (unsigned long long)__popc(peers));
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Length bucketing: a counting sort of the batch's entries by their number of streaming chunks,
// longest first.  K_map then gives each warp 32 records of (nearly) equal length, so a warp no
// longer waits for its longest record (this matters on mixed 512 B..8 KB input), and the
// longest records are started first (LPT order) so the grid drains evenly.  Three tiny kernels:
// histogram over 256 buckets, 256-entry scan, scatter.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kLenBuckets = 256;
// K_map's three resident CTAs hold 61,440 of an SM's 65,536 registers.  A 128-thread block of up to 32 registers fits
// into the rest, a 256-thread block does not: it would wait until a K_map CTA of the round running on the other stream
// retires, and K_map's next launch would wait behind it.
constexpr uint32_t kLenThreads = 128;

__device__ __forceinline__ uint32_t len_bucket(const uint64_t* __restrict__ offsets, const uint32_t* __restrict__ lens, uint64_t e,
                                               uint64_t blob_bytes) {
    const uint64_t off = offsets[e], end = lens ? off + lens[e] : offsets[e + 1];
    const uint64_t L = (end < off || end > blob_bytes) ? 0 : end - off;
    const uint64_t chunks = (L + 127) >> 7;
    const uint32_t b = chunks >= kLenBuckets ? kLenBuckets - 1 : (uint32_t)chunks;
    return (kLenBuckets - 1) - b;  // bucket 0 = longest
}

__global__ void __launch_bounds__(kLenThreads) len_hist_kernel(const uint64_t* __restrict__ offsets, const uint32_t* __restrict__ lens, uint64_t n, uint64_t blob_bytes,
                                                       unsigned int* __restrict__ hist) {
    __shared__ unsigned int sh[kLenBuckets];
    for (uint32_t b = threadIdx.x; b < kLenBuckets; b += blockDim.x) sh[b] = 0;
    __syncthreads();
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x)
        atomicAdd(&sh[len_bucket(offsets, lens, e, blob_bytes)], 1u);
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < kLenBuckets; b += blockDim.x)
        if (sh[b]) atomicAdd(&hist[b], sh[b]);
}

// exclusive scan of the 256 bucket counts by ONE WARP (8 buckets per lane + a shuffle scan): this tiny kernel sits on
// K_map's stream in front of every launch, where a single-thread loop sat on the critical path
__global__ void len_scan_kernel(unsigned int* hist_then_cursor) {
    const uint32_t lane = threadIdx.x;
    unsigned int v[8], sum = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        v[i] = hist_then_cursor[lane * 8 + i];
        sum += v[i];
    }
    unsigned int incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned int up = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= (uint32_t)d) incl += up;
    }
    unsigned int acc = incl - sum;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        hist_then_cursor[lane * 8 + i] = acc;
        acc += v[i];
    }
}

__global__ void __launch_bounds__(kLenThreads) len_scatter_kernel(const uint64_t* __restrict__ offsets, const uint32_t* __restrict__ lens, uint64_t n, uint64_t blob_bytes,
                                                          unsigned int* __restrict__ cursor, uint32_t* __restrict__ order) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = e < n;
    const uint32_t b = in ? len_bucket(offsets, lens, e, blob_bytes) : 0xFFFFFFFFu;
    const uint32_t peers = __match_any_sync(0xffffffffu, b);
    if (in) {
        const uint32_t leader = (uint32_t)__ffs(peers) - 1u;
        unsigned int base = 0;
        if ((threadIdx.x & 31u) == leader) base = atomicAdd(&cursor[b], (unsigned int)__popc(peers));
        base = __shfl_sync(peers, base, leader);
        order[base + __popc(peers & ((1u << (threadIdx.x & 31u)) - 1u))] = (uint32_t)e;
    }
}

cudaError_t launch_len_order(const uint64_t* offsets, const uint32_t* lens, uint64_t n, uint64_t blob_bytes, unsigned int* hist256, uint32_t* order,
                             int sm_count, cudaStream_t s) {
    if (!n) return cudaSuccess;
    cudaError_t err = cudaMemsetAsync(hist256, 0, kLenBuckets * sizeof(unsigned int), s);
    if (err != cudaSuccess) return err;
    const unsigned hb = (unsigned)((n + kLenThreads * 8 - 1) / (kLenThreads * 8));
    const unsigned cap = (unsigned)sm_count * 8u;
    len_hist_kernel<<<hb < cap ? (hb ? hb : 1u) : cap, kLenThreads, 0, s>>>(offsets, lens, n, blob_bytes, hist256);
    len_scan_kernel<<<1, 32, 0, s>>>(hist256);
    len_scatter_kernel<<<(unsigned)((n + kLenThreads - 1) / kLenThreads), kLenThreads, 0, s>>>(offsets, lens, n, blob_bytes, hist256, order);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Register-only SHA-256 microbenchmark (SURVEY.md §7 H2: "measure the INT ceiling ... rather than
// trusting the estimate").  Same compression function as K_map, no memory traffic at all: every
// lane chains `iters` compressions on register-resident message words.  Its rate is the practical
// ceiling of the fingerprint on this part; bench.py --sha-ceiling reports it beside K_map's rate.
// ------------------------------------------------------------------------------------------------
template <int ROLLED>
__global__ void __launch_bounds__(256) sha_ceiling_kernel(uint32_t iters, uint32_t one, uint32_t* __restrict__ sink) {
    extern __shared__ uint8_t occupancy_pad[];  // only sized to pin the number of resident CTAs per SM
    Sha256State st;
    st.init();
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i] = (blockIdx.x * blockDim.x + threadIdx.x) * 0x9E3779B9u + i;
    for (uint32_t it = 0; it < iters; ++it) {
        uint32_t m[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) m[i] = w[i] ^ st.h[i & 7];  // data-dependent: nothing can be hoisted
        if (ROLLED) sha256_compress_rolled(st, m, one);
        else sha256_compress(st, m, one);
    }
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc ^= st.h[i];
    if (acc == 0x12345678u) sink[0] = acc;  // keeps the chain alive without a store per thread
}

cudaError_t launch_sha_ceiling(uint32_t iters, int rolled, int ctas_per_sm, int sm_count, uint32_t* sink, cudaStream_t s) {
    // 256-thread CTAs; dynamic shared memory chosen so that exactly ctas_per_sm CTAs fit per SM
    const int smem = ctas_per_sm >= 8 ? 0 : (int)((227 * 1024) / ctas_per_sm - 2048);
    auto kern = rolled ? sha_ceiling_kernel<1> : sha_ceiling_kernel<0>;
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (err != cudaSuccess) return err;
    kern<<<sm_count * ctas_per_sm, 256, smem, s>>>(iters, 1u, sink);
    return cudaGetLastError();
}

cudaError_t launch_map(const MapParams& p, int sm_count, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    if (p.sha256 == nullptr) {  // no fingerprint requested: nothing to stream
        map_light_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, s>>>(p);
        return cudaGetLastError();
    }
    using Cfg = StreamCfg;
    cudaError_t err = cudaFuncSetAttribute(map_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmem);
    if (err != cudaSuccess) return err;
    // kCtasPerSm rings need the largest shared-memory carve-out
    err = cudaFuncSetAttribute(map_stream_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    if (err != cudaSuccess) return err;
    // persistent grid: kCtasPerSm CTAs on every SM, fewer when the batch has fewer warp groups
    const uint64_t ngroups = (p.n + 31) / 32;
    uint64_t ctas = (uint64_t)sm_count * Cfg::kCtasPerSm;
    const uint64_t need = (ngroups + Cfg::kWarps - 1) / Cfg::kWarps;
    if (need < ctas) ctas = need ? need : 1;
    map_stream_kernel<<<(unsigned)ctas, Cfg::kWarps * 32, Cfg::kSmem, s>>>(p);
    return cudaGetLastError();
}

}  // namespace ctmr
