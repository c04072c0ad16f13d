// ctmr_map_alt.cu -- MEASURED ALTERNATIVES of K_map, kept selectable (CTMR_MAP_VARIANT=1|3) because the
// verdicts in DESIGN.md "Measured and rejected" come from them and they pass the same parity suite:
//   v1  DER walk on global memory (LDG.U8) + per-lane TMA bulk copies for the SHA-256 stream
//   v3  streaming kernel with per-lane dynamic scheduling (loader cursor two slots ahead)
#include "ctmr_common.cuh"
#include "ctmr_stream.cuh"

namespace ctmr {

// ------------------------------------------------------------------------------------------------
// K_map
// ------------------------------------------------------------------------------------------------
template <int WARPS, int CHUNK>
struct MapCfg {
    static constexpr int kSlot = CHUNK + 16;                 // +16: a record may start anywhere in a 16-byte line
    static constexpr int kWarpBytes = 2 * 32 * kSlot;        // two stages x 32 lanes
    static constexpr int kBlocksPerChunk = CHUNK / 64;
    static constexpr size_t kSmem = (size_t)WARPS * kWarpBytes + (size_t)WARPS * 2 * sizeof(uint64_t);
};

template <int WARPS, int CHUNK>
__global__ void __launch_bounds__(WARPS * 32) map_kernel(const __grid_constant__ MapParams p) {
    using Cfg = MapCfg<WARPS, CHUNK>;
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* my_slots = smem + (size_t)warp * Cfg::kWarpBytes + (size_t)lane * Cfg::kSlot;  // stage s at + s*32*kSlot
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)WARPS * Cfg::kWarpBytes) + warp * 2;
    const uint32_t bar0 = smem_u32(&bars[0]), bar1 = smem_u32(&bars[1]);
    const uint32_t slot0 = smem_u32(my_slots), slot1 = slot0 + 32 * Cfg::kSlot;
    if (lane == 0) {
        mbar_init(bar0, 32);
        mbar_init(bar1, 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    uint32_t parity = 0;  // bit s: phase parity the next wait on stage s expects

    const uint64_t ngroups = (p.n + 31) >> 5;
    const bool want_sha = p.sha256 != nullptr;
    for (uint64_t g = (uint64_t)blockIdx.x * WARPS + warp; g < ngroups; g += (uint64_t)gridDim.x * WARPS) {
        const uint64_t e = g * 32 + lane;
        const bool act = e < p.n;
        uint64_t off = 0, end = 0;
        if (act) {
            off = p.offsets[e];
            end = p.offsets[e + 1];
        }
        // memory safety against malformed offset tables: an unusable record hashes as empty
        bool bad_span = !act || end < off || end > p.blob_bytes || end - off > 0x7fffffffull;
        const uint32_t L = bad_span ? 0u : (uint32_t)(end - off);
        const uint8_t* d = p.blob + off;

        // ---- streaming plan for the fingerprint
        const uint64_t addr = reinterpret_cast<uint64_t>(d);
        const uint32_t m = (uint32_t)(addr & 15u);
        const uint8_t* src_base = reinterpret_cast<const uint8_t*>(addr & ~15ull);
        const uint32_t nfull = L >> 6;
        const uint32_t nb = want_sha && act ? nfull + 1u + ((L & 63u) >= 56u ? 1u : 0u) : 0u;  // padded blocks
        const uint32_t ndata = want_sha && act ? (L + CHUNK - 1) / CHUNK : 0u;                  // chunks with data
        const uint32_t nch = (nb + Cfg::kBlocksPerChunk - 1) / Cfg::kBlocksPerChunk;
        uint32_t iters = warp_max_u32(nch);
        iters = iters < 2u ? 2u : iters;

        auto issue = [&](uint32_t c) {
            const uint32_t bar = (c & 1u) ? bar1 : bar0;
            if (c < ndata) {
                const uint32_t db = min((uint32_t)CHUNK, L - c * CHUNK);
                const uint32_t bytes = (m + db + 15u) & ~15u;
                mbar_arrive_expect_tx(bar, bytes);
                bulk_g2s((c & 1u) ? slot1 : slot0, src_base + (size_t)c * CHUNK, bytes, bar);
            } else {
                mbar_arrive(bar);
            }
        };
        if (want_sha) {  // both stages in flight while this lane walks the TLV tree
            issue(0);
            issue(1);
        }

        // ---- map: x509 field extraction + certIsFilteredOut
        ParsedCert pc;
        uint32_t status = CTMR_ST_PARSE_ERR;
        uint32_t issuer = CTMR_ISSUER_NONE;
        int64_t exp_hour = 0;
        if (act) {
            const bool ok = !bad_span && parse_cert(d, L, pc);
            if (ok) {
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
                        for (uint32_t i = 0; i < pl; ++i) {
                            if (__ldg(d + pc.cn_off + i) != p.filter.bytes[po + i]) {
                                eq = false;
                                break;
                            }
                        }
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
            }
            if (p.status) p.status[e] = (uint8_t)status;
            if (p.exp_hour) p.exp_hour[e] = exp_hour;
            if (p.serial_off) p.serial_off[e] = pc.serial_off;
            if (p.serial_len) p.serial_len[e] = pc.serial_len;
            if (p.keys) {
                // 64-byte key record, written as four 16-byte stores
                uint32_t kw[10];
#pragma unroll
                for (int i = 0; i < 10; ++i) kw[i] = 0;
                const bool valid = status == CTMR_ST_OK;
                if (valid) {
                    kw[0] = pc.serial_len;
#pragma unroll
                    for (int i = 0; i < (int)CTMR_MAX_SERIAL; ++i) {
                        if ((uint32_t)i < pc.serial_len)
                            kw[(i + 1) >> 2] |= (uint32_t)__ldg(d + pc.serial_off + i) << (8 * ((i + 1) & 3));
                    }
                }
                const uint64_t gi = p.first_index + e;
                uint4* kr = reinterpret_cast<uint4*>(p.keys + e);
                kr[0] = make_uint4((uint32_t)gi, (uint32_t)(gi >> 32), (uint32_t)(int32_t)exp_hour, valid ? issuer : 0u);
                kr[1] = make_uint4(kw[0], kw[1], kw[2], kw[3]);
                kr[2] = make_uint4(kw[4], kw[5], kw[6], kw[7]);
                kr[3] = make_uint4(kw[8], kw[9], valid ? 1u : 0u, 0u);
            }
        }
        if (p.status_counts) {  // certIsFilteredOut.* / insertCTWorker.Inserted counters, one atomic per value per warp
            const uint32_t amask = __ballot_sync(0xffffffffu, act);
            if (act) {
                const uint32_t peers = __match_any_sync(amask, status);
                if ((uint32_t)lane == (uint32_t)__ffs(peers) - 1u)
                    atomicAdd(p.status_counts + status, (unsigned long long)__popc(peers));
            }
        }

        // ---- fingerprint: SHA-256 over the record, streamed chunk by chunk through shared memory
        if (want_sha) {
            Sha256State st;
            st.init();
            const uint32_t sel = 0x0123u + 0x1111u * (m & 3u);  // PRMT: big-endian word starting at byte (m & 3)
            for (uint32_t c = 0; c < iters; ++c) {
                const uint32_t s = c & 1u;
                mbar_wait(s ? bar1 : bar0, (parity >> s) & 1u);
                parity ^= 1u << s;
                if (c < nch) {
                    const uint8_t* slot = my_slots + (size_t)s * 32 * Cfg::kSlot;
#pragma unroll 1
                    for (uint32_t bb = 0; bb < (uint32_t)Cfg::kBlocksPerChunk; ++bb) {
                        const uint32_t b = c * Cfg::kBlocksPerChunk + bb;
                        if (b >= nb) break;
                        const uint32_t* sw = reinterpret_cast<const uint32_t*>(slot) + ((m + 64u * bb) >> 2);
                        uint32_t x[17], w[16];
#pragma unroll
                        for (int i = 0; i < 17; ++i) x[i] = sw[i];
#pragma unroll
                        for (int i = 0; i < 16; ++i) w[i] = __byte_perm(x[i], x[i + 1], sel);
                        if (b >= nfull) {  // trailing block(s): 0x80, zeros, 64-bit bit length
#pragma unroll
                            for (int i = 0; i < 16; ++i) w[i] = sha256_pad_word(w[i], b * 64u + 4u * i, L);
                            if (b == nb - 1u) {
                                w[14] = L >> 29;
                                w[15] = L << 3;
                            }
                        }
                        sha256_compress(st, w, p.one);
                    }
                }
                if (c + 2u < iters) issue(c + 2u);
            }
            if (act) {
                uint4* o = reinterpret_cast<uint4*>(p.sha256 + e * 32);
                o[0] = make_uint4(__byte_perm(st.h[0], 0, 0x0123), __byte_perm(st.h[1], 0, 0x0123),
                                  __byte_perm(st.h[2], 0, 0x0123), __byte_perm(st.h[3], 0, 0x0123));
                o[1] = make_uint4(__byte_perm(st.h[4], 0, 0x0123), __byte_perm(st.h[5], 0, 0x0123),
                                  __byte_perm(st.h[6], 0, 0x0123), __byte_perm(st.h[7], 0, 0x0123));
            }
        }
    }
}

template <int WARPS, int CHUNK>
static cudaError_t launch_map_t(const MapParams& p, int sm_count, int ctas_per_sm, cudaStream_t s) {
    using Cfg = MapCfg<WARPS, CHUNK>;
    auto kern = map_kernel<WARPS, CHUNK>;
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmem);
    if (err != cudaSuccess) return err;
    const uint64_t ngroups = (p.n + 31) / 32;
    uint64_t ctas = (uint64_t)sm_count * ctas_per_sm;  // persistent: a multiple of the SM count
    const uint64_t need = (ngroups + WARPS - 1) / WARPS;
    if (need < ctas) ctas = need ? need : 1;
    kern<<<(unsigned)ctas, WARPS * 32, Cfg::kSmem, s>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_map_v1(const MapParams& p, int sm_count, cudaStream_t s) {
    static const int warps = env_int("CTMR_MAP_WARPS", 4);
    static const int cps = env_int("CTMR_MAP_CTAS_PER_SM", 0);
    if (warps == 8) return launch_map_t<8, 256>(p, sm_count, cps ? cps : 1, s);
    return launch_map_t<4, 256>(p, sm_count, cps ? cps : 3, s);
}

// ------------------------------------------------------------------------------------------------
// K_map v3: the streaming map with PER-LANE dynamic scheduling.
//
// In v2 a warp takes 32 consecutive records and runs until its longest record is done, so on
// mixed-size input (BASELINE configs[4]: 512 B..8 KB) lanes idle for most of the time (measured
// before the port at less than half the uniform-size rate).  Here every lane owns an endless stream of "slots"
// (one slot = one CHUNK of one record); a loader cursor runs exactly two slots ahead of the consumer
// cursor and crosses record boundaries on its own, so the first chunks of a lane's NEXT record are
// already in flight while it finishes the current one.  Records are handed out from a warp-local
// queue (ballot + prefix popcount) that is refilled in spans from one global atomic counter.
// cp.async only: completion is tracked per thread (wait_group), no barrier is shared by lanes.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kDynSpan = 128;  // records a warp takes from the global counter at a time

struct DynCert {  // what a lane needs to know about a record
    uint32_t e;     // entry index inside the batch
    uint32_t L;     // length (0 for an unusable span)
    uint64_t addr;  // address of byte 0
};

template <int WARPS, int CHUNK, int ROLLED>
__global__ void __launch_bounds__(WARPS * 32) map_dyn_kernel(const __grid_constant__ MapParams p,
                                                             unsigned long long* __restrict__ work_counter) {
    using Cfg = StreamCfg<WARPS, CHUNK, 0>;
    constexpr uint32_t OV = Cfg::kOverlap;
    constexpr uint32_t BPC = Cfg::kBlocksPerChunk;
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t slot_base = smem_u32(smem + (size_t)warp * Cfg::kWarpBytes + (size_t)lane * Cfg::kSlot);
    const uint32_t stage_stride = 32 * Cfg::kSlot;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const bool want_sha = p.sha256 != nullptr;
    const uint32_t one = p.one;

    // warp-uniform work queue
    uint64_t q_next = 0, q_end = 0;
    bool global_done = false;

    // per-lane cursors
    DynCert cur{0, 0, 0}, nxt{0, 0, 0};
    bool have_cur = false, have_nxt = false, drained = false;
    uint32_t c = 0, cur_nch = 0;                    // consumer: slot index inside cur, slots of cur
    uint32_t ld_c = 0, ld_nch = 0, ld_L = 0;        // loader: slot index inside its record, slots, length
    uint64_t ld_addr = 0;
    uint32_t lag = 0, stage_c = 0, stage_l = 0;     // slots issued - consumed; stage of next consume / next issue
    uint32_t tags = 0;                              // bit s: the slot staged in stage s belongs to a record (else: a bubble)
    Walker w;
    w.init();
    Sha256State st;
    st.init();

    auto slots_of = [&](uint32_t L) -> uint32_t {
        const uint32_t nb = want_sha ? (L >> 6) + 1u + ((L & 63u) >= 56u ? 1u : 0u) : 0u;
        uint32_t n = (nb + BPC - 1) / BPC;
        const uint32_t nd = (L + CHUNK - 1) / CHUNK;
        n = n > nd ? n : nd;
        return n < 2u ? 2u : n;  // >= 2 slots per record: the loader is never more than one record ahead
    };

    for (;;) {
        // ---- (a) hand out records to lanes whose loader has run off the end of its record
        const bool wants = !drained && !have_nxt && ld_c == ld_nch;
        const uint32_t want_mask = __ballot_sync(0xffffffffu, wants);
        if (want_mask) {
            if (q_next >= q_end && !global_done) {
                unsigned long long s0 = 0;
                if (lane == 0) s0 = atomicAdd(work_counter, (unsigned long long)kDynSpan);
                s0 = __shfl_sync(0xffffffffu, s0, 0);
                if (s0 >= p.n) {
                    global_done = true;
                } else {
                    q_next = s0;
                    q_end = s0 + kDynSpan < p.n ? s0 + kDynSpan : p.n;
                }
            }
            const uint32_t avail = (uint32_t)(q_end - q_next);
            const uint32_t rank = __popc(want_mask & lt_mask);
            if (wants) {
                if (rank < avail) {
                    const uint64_t e = q_next + rank;
                    const uint64_t off = p.offsets[e], end = p.offsets[e + 1];
                    const bool bad = end < off || end > p.blob_bytes || end - off > 0x7fffffffull;
                    nxt.e = (uint32_t)e;
                    nxt.L = bad ? 0u : (uint32_t)(end - off);
                    nxt.addr = reinterpret_cast<uint64_t>(p.blob + (bad ? 0 : off));
                    have_nxt = true;
                    ld_c = 0;
                    ld_L = nxt.L;
                    ld_nch = slots_of(nxt.L);
                    ld_addr = nxt.addr;
                } else if (global_done) {
                    drained = true;  // nothing left anywhere: this lane's loader idles from now on
                }
            }
            const uint32_t taken = (uint32_t)__popc(want_mask);
            q_next += taken < avail ? taken : avail;
        }
        if (!__ballot_sync(0xffffffffu, have_cur || have_nxt || !drained)) break;

        // ---- (b) consumer: slot `c` of the current record, once two slots are in flight behind it
        if (lag == 2u) {
            cp_async_wait<1>();
            const bool real = (tags >> stage_c) & 1u;
            if (real && !have_cur) {  // first slot of the record the loader started two slots ago: it becomes current
                cur = nxt;
                have_cur = true;
                have_nxt = false;
                cur_nch = slots_of(cur.L);
                w.init();
                st.init();
            }
            if (real) {
                const uint32_t L = cur.L;
                const uint32_t m = (uint32_t)(cur.addr & 15u);
                const uint32_t sbase = slot_base + stage_c * stage_stride;
                if (w.st < W_DONE) {
                    const uint32_t avail = min((c + 1u) * CHUNK, L);
                    const SmemWindow rd{sbase + m + OV - c * CHUNK};
                    const GlobalBytes far{reinterpret_cast<const uint8_t*>(cur.addr)};
                    uint32_t* key_words = p.keys ? reinterpret_cast<uint32_t*>(p.keys + cur.e) + 4 : nullptr;
                    walk_advance(w, rd, far, avail, L, p.filter, key_words);
                }
                if (want_sha) {
                    const uint32_t nfull = L >> 6;
                    const uint32_t nb = nfull + 1u + ((L & 63u) >= 56u ? 1u : 0u);
                    const uint32_t sel = 0x0123u + 0x1111u * (m & 3u);
#pragma unroll 1
                    for (uint32_t bb = 0; bb < BPC; ++bb) {
                        const uint32_t b = c * BPC + bb;
                        if (b >= nb) break;
                        const uint32_t wa = sbase + ((m + OV + 64u * bb) & ~3u);
                        uint32_t x[17], wd[16];
#pragma unroll
                        for (int i = 0; i < 17; ++i) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(x[i]) : "r"(wa + 4u * i));
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
                        if (ROLLED) sha256_compress_rolled(st, wd, one);
                        else sha256_compress(st, wd, one);
                    }
                }
                ++c;
                if (c == cur_nch) {
                    // ---- record finished: certIsFilteredOut + Store preconditions, outputs
                    const uint64_t e = cur.e;
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
                    if (p.keys) {
                        const bool valid = status == CTMR_ST_OK;
                        const uint64_t gi = p.first_index + e;
                        uint4* kr = reinterpret_cast<uint4*>(p.keys + e);
                        kr[0] = make_uint4((uint32_t)gi, (uint32_t)(gi >> 32), (uint32_t)(int32_t)exp_hour, valid ? issuer : 0u);
                        *reinterpret_cast<uint2*>(reinterpret_cast<uint32_t*>(kr) + 14) = make_uint2(valid ? 1u : 0u, 0u);
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
                    have_cur = false;
                    c = 0;
                }
            }
            stage_c ^= 1u;
            --lag;
        }

        // ---- (c) loader: one slot per iteration into the stage the consumer has just left (or the pipeline fill)
        {
            uint32_t bytes = 0, dst = slot_base + stage_l * stage_stride;
            const uint8_t* src = nullptr;
            tags &= ~(1u << stage_l);
            if (ld_c < ld_nch) {
                tags |= 1u << stage_l;
                const uint32_t nd = (ld_L + CHUNK - 1) / CHUNK;
                if (ld_c < nd) {
                    const uint32_t m = (uint32_t)(ld_addr & 15u);
                    const uint32_t db = min((uint32_t)CHUNK, ld_L - ld_c * CHUNK);
                    const uint8_t* base = reinterpret_cast<const uint8_t*>(ld_addr & ~15ull);
                    if (ld_c == 0u) {
                        bytes = (m + db + 15u) & ~15u;
                        dst += OV;
                        src = base;
                    } else {
                        bytes = (m + OV + db + 15u) & ~15u;
                        src = base + (size_t)ld_c * CHUNK - OV;
                    }
                }
                ++ld_c;
            }
#pragma unroll 1
            for (uint32_t j = 0; j < bytes; j += 16u) cp_async16(dst + j, src + j);
            cp_async_commit();
            stage_l ^= 1u;
            ++lag;
        }
    }
    cp_async_wait<0>();
}

template <int WARPS, int CHUNK, int ROLLED>
static cudaError_t launch_dyn_t(const MapParams& p, int sm_count, int ctas_per_sm, unsigned long long* counter, cudaStream_t s) {
    using Cfg = StreamCfg<WARPS, CHUNK, 0>;
    auto kern = map_dyn_kernel<WARPS, CHUNK, ROLLED>;
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmem);
    if (err != cudaSuccess) return err;
    err = cudaMemsetAsync(counter, 0, sizeof(unsigned long long), s);
    if (err != cudaSuccess) return err;
    const uint64_t nspans = (p.n + kDynSpan - 1) / kDynSpan;
    uint64_t ctas = (uint64_t)sm_count * ctas_per_sm;
    const uint64_t need = (nspans + WARPS - 1) / WARPS;
    if (need < ctas) ctas = need ? need : 1;
    kern<<<(unsigned)ctas, WARPS * 32, Cfg::kSmem, s>>>(p, counter);
    return cudaGetLastError();
}

cudaError_t launch_map_v3(const MapParams& p, int sm_count, cudaStream_t s) {
    static const int chunk = env_int("CTMR_MAP_CHUNK", 128);
    static const int cps = env_int("CTMR_MAP_CTAS_PER_SM", 0);
    if (!p.work_counter) return cudaErrorInvalidValue;
    if (chunk == 256) return launch_dyn_t<8, 256, 1>(p, sm_count, cps ? cps : 1, p.work_counter, s);
    return launch_dyn_t<8, 128, 1>(p, sm_count, cps ? cps : 2, p.work_counter, s);
}

}  // namespace ctmr
