// ctmr_cascade.cu -- ctmr_revoked_cascade / ctmr_group_revoked_cascade: CRLite's filter cascade of the covered issuers'
// revoked (R) and not revoked (S) live key records, built next to the table (include/ctmr.h states the contract, DESIGN.md
// "Revoked cascade" the design).
//
// The CRLs go through ctmr_crl.cu's chunk path up to the chunk's (issuer, serial) set (crl_each_set); then
//   cascade_mark     grid-stride over the table per chunk: a live ready key whose pair is in the set sets its slot's bit
//   cascade_split    grid-stride over the table once: live ready keys of covered issuers; revoked ones -> the R list,
//                    the others are counted (S)
//   cascade_insert   thread per included record: k_l SHA-256s of one or two blocks, atomicOr into the level's bits
//   cascade_test     thread per excluded record (level 1: grid-stride over the table for S): hashes until the first
//                    clear bit; a record the level contains goes to the next include list
// The host reads one count per level, sizes the next level and reads each finished level back.
// ctmr_revoked_stash / ctmr_group_revoked_stash share the work up to the split (cascade_front), then
//   stash_query      thread per R record: the published filter's query; the records it misses go to the host
// ctmr_revoked_verify / ctmr_group_revoked_verify share cascade_front too, mark the stashes' set with cascade_mark, then
//   verify_table     grid-stride over the table, one hash per lane per step: the filter's query of every covered live
//                    record the stashes do not list; counts, and the slots of the records answered wrongly
//   verify_gather    thread per listed record: the slot, for the host
#include <algorithm>
#include <cmath>
#include <initializer_list>
#include <string>
#include <unordered_map>
#include <unordered_set>

#include "ctmr_common.cuh"
#include "ctmr_ctx.cuh"

namespace ctmr {
namespace {

constexpr uint32_t kCascadeThreads = 256;  // the message columns in shared memory are laid out for this block size
constexpr uint32_t kNoList = 0xFFFFFFFFu;

// What every cascade kernel reads: the table, the registry's digests and the covered issuers, the salt, and the level.
struct CascadeParams {
    const KnownSlot* table;
    uint64_t n_slots;
    uint32_t epoch;
    const uint8_t* dig;        // [n_issuers][32] by dense index
    const uint32_t* covered;   // bit per dense index
    uint32_t n_issuers;
    uint32_t salt_len;
    int64_t now;
    uint32_t salt[8];          // little-endian words: byte j is salt[j >> 2] >> 8 (j & 3)
    uint32_t level, k, m;
    uint32_t one;              // always 1: sha256_compress's multiplier ptxas cannot fold
};

__device__ __forceinline__ bool slot_live_ready(uint4 q0, uint4 q1, uint32_t epoch, int64_t now) {
    return slot_state(((uint64_t)q0.w << 32) | q0.z, epoch) == kSlotReady && (int64_t)(int32_t)q1.x * 3600 > now;
}

__device__ __forceinline__ bool issuer_covered(const CascadeParams& p, uint32_t issuer) {
    return issuer < p.n_issuers && (__ldg(p.covered + (issuer >> 5)) >> (issuer & 31u) & 1u);
}

// One thread's message, salt || LE32(i) || u8(l) || digest || serial, padded, in its column of the block's shared
// memory: word w of thread t at col[w * kCascadeThreads], so that the 32 lanes of a warp touch 32 banks.
struct CascadeMsg {
    uint32_t* col;
    uint32_t len;  // message bytes: salt_len + 37 + serial_len <= 108, two blocks at most

    __device__ __forceinline__ void put(uint32_t b, uint32_t v) {
        reinterpret_cast<uint8_t*>(col + (b >> 2) * kCascadeThreads)[b & 3u] = (uint8_t)v;
    }

    // the message of the key in the slot body words b[0..12) (exp_hour, issuer, {serial_len, serial[39]}) at level l; the
    // four bytes of i are written by hash()
    __device__ __forceinline__ void build(const CascadeParams& p, const uint32_t (&b)[12]) {
#pragma unroll
        for (uint32_t w = 0; w < 32u; ++w) col[w * kCascadeThreads] = 0u;
        const uint32_t sl = p.salt_len;
#pragma unroll
        for (uint32_t j = 0; j < 32u; ++j)
            if (j < sl) put(j, p.salt[j >> 2] >> (8u * (j & 3u)));
        put(sl + 4u, p.level);
        const uint4* d = reinterpret_cast<const uint4*>(p.dig + 32ull * b[1]);
        const uint4 d0 = __ldg(d), d1 = __ldg(d + 1);
        const uint32_t dw[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
        for (uint32_t j = 0; j < 32u; ++j) put(sl + 5u + j, dw[j >> 2] >> (8u * (j & 3u)));
        const uint32_t n = b[2] & 0xFFu;  // serial byte j is body byte 9 + j
#pragma unroll
        for (uint32_t j = 0; j < (uint32_t)CTMR_MAX_SERIAL; ++j)
            if (j < n) put(sl + 37u + j, b[(9u + j) >> 2] >> (8u * ((9u + j) & 3u)));
        len = sl + 37u + n;
        put(len, 0x80u);
    }

    // b_i before the modulus: LE32 of the first four digest bytes
    __device__ __forceinline__ uint32_t hash(const CascadeParams& p, uint32_t i) {
        const uint32_t sl = p.salt_len;
#pragma unroll
        for (uint32_t j = 0; j < 4u; ++j) put(sl + j, i >> (8u * j));
        const uint32_t nb = len + 9u <= 64u ? 1u : 2u;
        Sha256State s;
        s.init();
        for (uint32_t blk = 0; blk < nb; ++blk) {
            uint32_t w[16];
#pragma unroll
            for (uint32_t j = 0; j < 16u; ++j) w[j] = __byte_perm(col[(16u * blk + j) * kCascadeThreads], 0u, 0x0123u);
            if (blk + 1u == nb) w[15] = len * 8u;
            sha256_compress(s, w, p.one);
        }
        return __byte_perm(s.h[0], 0u, 0x0123u);
    }
};

__device__ __forceinline__ void load_body(const KnownSlot* table, uint64_t slot, uint32_t (&b)[12]) {
    const uint4* sp = reinterpret_cast<const uint4*>(table + slot) + 1;
    const uint4 q1 = __ldg(sp), q2 = __ldg(sp + 1), q3 = __ldg(sp + 2);
    const uint32_t v[12] = {q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};
#pragma unroll
    for (int j = 0; j < 12; ++j) b[j] = v[j];
}

// does the level (bits, p.k functions, p.m bits) contain the key of the message?
__device__ __forceinline__ bool contains(const CascadeParams& p, CascadeMsg& msg, const uint32_t* __restrict__ bits) {
    for (uint32_t i = 0; i < p.k; ++i) {
        const uint32_t b = msg.hash(p, i) % p.m;
        if (!(__ldg(bits + (b >> 5)) >> (b & 31u) & 1u)) return false;
    }
    return true;
}

__device__ __forceinline__ void append(uint32_t slot, uint32_t* list, uint64_t cap, unsigned long long* counter) {
    const unsigned long long at = atomicAdd(counter, 1ull);
    if (at < cap) list[at] = slot;  // past cap only the count advances: the host grows the list and runs again
}

// per chunk: every live ready key whose (issuer, serial) is in the set marks its slot revoked
__global__ void __launch_bounds__(256) cascade_mark_kernel(const KnownSlot* __restrict__ table, uint64_t n_slots, uint32_t epoch, int64_t now,
                                                           const CrlSetSlot* __restrict__ set, uint64_t mask, uint32_t* revoked) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slots; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4* sp = reinterpret_cast<const uint4*>(table + i);
        const uint4 q0 = __ldcs(sp), q1 = __ldcs(sp + 1);
        if (!slot_live_ready(q0, q1, epoch, now)) continue;
        const uint4 q2 = __ldcs(sp + 2), q3 = __ldcs(sp + 3);
        const uint32_t w[11] = {q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};
        const uint32_t h = pair_hash(w), ready = (h & ~3u) | 2u;
        for (uint64_t pos = h & mask;; pos = (pos + 1) & mask) {
            const CrlSetSlot& sl = set[pos];
            const uint32_t tg = sl.tag;
            if (tg == 0u) break;
            if (tg != ready) continue;
            bool same = true;
#pragma unroll
            for (int k = 0; k < 11; ++k) same &= sl.key[k] == w[k];
            if (same) {
                atomicOr(revoked + (i >> 5), 1u << (i & 31u));
                break;
            }
        }
    }
}

// once, after the last chunk: the live ready keys of covered issuers; revoked ones go to the R list, the others are
// counted.  counters[0]: |R| of this shard, counters[1]: |S|.
__global__ void __launch_bounds__(256) cascade_split_kernel(CascadeParams p, const uint32_t* __restrict__ revoked, uint32_t* rlist,
                                                            uint64_t cap, unsigned long long* counters) {
    unsigned long long valid = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n_slots; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4* sp = reinterpret_cast<const uint4*>(p.table + i);
        const uint4 q0 = __ldcs(sp), q1 = __ldcs(sp + 1);
        if (!slot_live_ready(q0, q1, p.epoch, p.now) || !issuer_covered(p, q1.y)) continue;
        if (__ldg(revoked + (i >> 5)) >> (i & 31u) & 1u) append((uint32_t)i, rlist, cap, counters);
        else ++valid;
    }
    valid = __reduce_add_sync(0xffffffffu, (uint32_t)valid);
    if ((threadIdx.x & 31u) == 0u && valid) atomicAdd(counters + 1, valid);
}

// thread per included record: its k_l bits into the level
__global__ void __launch_bounds__(kCascadeThreads) cascade_insert_kernel(CascadeParams p, const uint32_t* __restrict__ list, uint64_t n,
                                                                         uint32_t* bits) {
    __shared__ uint32_t smem[32 * kCascadeThreads];
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint32_t b[12];
    load_body(p.table, list[t], b);
    CascadeMsg msg{smem + threadIdx.x, 0u};
    msg.build(p, b);
    for (uint32_t i = 0; i < p.k; ++i) {
        const uint32_t j = msg.hash(p, i) % p.m;
        atomicOr(bits + (j >> 5), 1u << (j & 31u));
    }
}

// thread per excluded record of a list: the records the level contains go to the next include list
__global__ void __launch_bounds__(kCascadeThreads) cascade_test_kernel(CascadeParams p, const uint32_t* __restrict__ list, uint64_t n,
                                                                       const uint32_t* __restrict__ bits, uint32_t* next, uint64_t cap,
                                                                       unsigned long long* counter) {
    __shared__ uint32_t smem[32 * kCascadeThreads];
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t slot = list[t];
    uint32_t b[12];
    load_body(p.table, slot, b);
    CascadeMsg msg{smem + threadIdx.x, 0u};
    msg.build(p, b);
    if (contains(p, msg, bits)) append(slot, next, cap, counter);
}

// level 1's test: grid-stride over the table for S (live ready keys of covered issuers, not revoked)
__global__ void __launch_bounds__(kCascadeThreads) cascade_test_table_kernel(CascadeParams p, const uint32_t* __restrict__ revoked,
                                                                             const uint32_t* __restrict__ bits, uint32_t* next, uint64_t cap,
                                                                             unsigned long long* counter) {
    __shared__ uint32_t smem[32 * kCascadeThreads];
    CascadeMsg msg{smem + threadIdx.x, 0u};
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n_slots; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4* sp = reinterpret_cast<const uint4*>(p.table + i);
        const uint4 q0 = __ldcs(sp), q1 = __ldcs(sp + 1);
        if (!slot_live_ready(q0, q1, p.epoch, p.now) || !issuer_covered(p, q1.y)) continue;
        if (__ldg(revoked + (i >> 5)) >> (i & 31u) & 1u) continue;
        uint32_t b[12];
        load_body(p.table, i, b);
        msg.build(p, b);
        if (contains(p, msg, bits)) append((uint32_t)i, next, cap, counter);
    }
}

// a group's member 0: another member's partial level into its own
__global__ void __launch_bounds__(256) cascade_or_kernel(uint32_t* bits, const uint32_t* __restrict__ other, uint64_t words) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < words) bits[i] |= other[i];
}

// One process per GPU, a slice of the OR all-reduce.  Source side, grid (n / 256, world): words [0, n) of the rank's
// bits into its region on every rank, its own among them (posted stores; the barrier after publishes them).
__global__ void __launch_bounds__(256) cascade_peer_send_kernel(PeerExchange px, const uint32_t* __restrict__ bits, uint64_t n) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) reinterpret_cast<uint32_t*>(px.inbox[blockIdx.y] + (uint64_t)px.rank * px.X)[j] = bits[j];
}

// Owner side, thread per word: the OR of every source's region, its own included, into words [0, n) of the rank's bits
__global__ void __launch_bounds__(256) cascade_peer_or_kernel(PeerExchange px, uint32_t* bits, uint64_t n) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    uint32_t v = 0;
    for (uint32_t s = 0; s < px.world; ++s) v |= __ldcg(reinterpret_cast<const uint32_t*>(px.inbox[px.rank] + (uint64_t)s * px.X) + j);
    bits[j] = v;
}

// The published filter's query of the key whose message msg holds, one hash at a time (p: the filter's salt; levels[l]:
// level l + 1's first word in `words`, m and k).  The message is built once and only its level byte changes between
// levels.  A walk is at (l, i, lv): function i of level l + 1, lv = levels[l].
struct FilterWalk {
    uint32_t l, i;
    StashLevel lv;

    __device__ __forceinline__ void start(const CascadeParams& p, CascadeMsg& msg, const StashLevel* __restrict__ levels) {
        l = i = 0;
        lv = levels[0];
        msg.put(p.salt_len + 4u, 1u);
    }

    // the walk's next hash; true when the key is answered, with *revoked
    __device__ __forceinline__ bool step(const CascadeParams& p, CascadeMsg& msg, const uint32_t* __restrict__ words,
                                         const StashLevel* __restrict__ levels, uint32_t n_levels, bool* revoked) {
        const uint32_t b = msg.hash(p, i) % lv.m;
        if (!(__ldg(words + lv.word + (b >> 5)) >> (b & 31u) & 1u)) {  // stopped at level l + 1: revoked iff that is even
            *revoked = l & 1u;
            return true;
        }
        if (++i < lv.k) return false;
        i = 0;
        if (++l == n_levels) {  // contained in all: revoked iff n_levels is odd
            *revoked = n_levels & 1u;
            return true;
        }
        lv = levels[l];
        msg.put(p.salt_len + 4u, l + 1u);
        return false;
    }
};

__device__ __forceinline__ bool filter_revoked(const CascadeParams& p, CascadeMsg& msg, const uint32_t* __restrict__ words,
                                               const StashLevel* __restrict__ levels, uint32_t n_levels) {
    FilterWalk w;
    w.start(p, msg, levels);
    bool revoked = false;
    while (!w.step(p, msg, words, levels, n_levels, &revoked)) {
    }
    return revoked;
}

// ctmr_revoked_stash, thread per record of the R list: the published filter's query.  A record the filter calls revoked
// is counted in counters[1]; the key body words 1..11 of any other go to `bodies`, which holds n of them, at counters[0].
__global__ void __launch_bounds__(kCascadeThreads) stash_query_kernel(CascadeParams p, const uint32_t* __restrict__ list, uint64_t n,
                                                                      const uint32_t* __restrict__ words, const StashLevel* __restrict__ levels,
                                                                      uint32_t n_levels, uint32_t* bodies, unsigned long long* counters) {
    __shared__ uint32_t smem[32 * kCascadeThreads];
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint32_t b[12];
    load_body(p.table, list[t], b);
    CascadeMsg msg{smem + threadIdx.x, 0u};
    msg.build(p, b);
    if (filter_revoked(p, msg, words, levels, n_levels)) {
        atomicAdd(counters + 1, 1ull);
        return;
    }
    uint32_t* o = bodies + 11ull * atomicAdd(counters, 1ull);
#pragma unroll
    for (int j = 0; j < 11; ++j) o[j] = b[1 + j];
}

// ctmr_revoked_verify: the filter and the verify call's inputs of a member
struct VerifyArgs {
    const uint32_t* revoked;  // slot bits: R
    const uint32_t* listed;   // slot bits: a stash lists the slot's pair
    const uint32_t* words;
    const StashLevel* levels;
    uint32_t n_levels;
    uint64_t covered_below;
    uint32_t* list;           // slots of the listed records [cap]
    uint64_t cap;
    unsigned long long* counters;  // [9]
};

__device__ __forceinline__ bool slot_bit(const uint32_t* __restrict__ bits, uint32_t i) { return __ldg(bits + (i >> 5)) >> (i & 31u) & 1u; }

// The answer `ans` of the covered live record in `slot`: its count into the block's counters and, when it is listed,
// its slot into the list
__device__ __forceinline__ void verify_finish(const CascadeParams& p, const VerifyArgs& a, uint32_t slot, bool ans,
                                              unsigned long long* counts) {
    const bool rev = slot_bit(a.revoked, slot);
    const bool before = ~__ldg(&p.table[slot].inv_first) < a.covered_below;
    atomicAdd(counts + (before ? 0u : 4u) + (rev ? (ans ? 0u : 1u) : (ans ? 3u : 2u)), 1ull);
    if (before && rev != ans) append(slot, a.list, a.cap, a.counters + 8);
}

constexpr uint32_t kVerifyBlocksPerSm = 4;  // 64 registers, no spills (DESIGN.md "Revoked verify")

// One pass over the table, scheduled by hash rather than by record.  Each lane holds one covered live record and its
// place in the filter walk (FilterWalk), and every step of the loop computes one SHA-256 per lane.  A lane
// whose record is answered (a clear bit, or every level walked) takes the next record from its warp's queue in shared
// memory at the next step; the warp refills the queue 32 slots at a time whenever it holds fewer records than idle
// lanes.  So a lane never waits for the longest walk of its warp, and the R records, whose walks are the long ones, cost
// their own hashes only.  Records a stash lists are answered revoked at the scan, with no hash.  counters[0..8) += the
// counts, counters[8]: records listed (past cap only the count advances).
__global__ void __launch_bounds__(kCascadeThreads, kVerifyBlocksPerSm) verify_table_kernel(CascadeParams p, VerifyArgs a) {
    __shared__ uint32_t smem[32 * kCascadeThreads];
    __shared__ uint32_t queue[kCascadeThreads / 32][64];
    __shared__ unsigned long long counts[8];
    if (threadIdx.x < 8u) counts[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u, lower = (1u << lane) - 1u;
    uint32_t* q = queue[threadIdx.x >> 5];
    CascadeMsg msg{smem + threadIdx.x, 0u};
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u);
    uint32_t nq = 0, slot = 0;
    bool have = false;
    FilterWalk walk{};
    for (;;) {
        const uint32_t idle = __ballot_sync(0xffffffffu, !have);
        const uint32_t want = __popc(idle);
        while (nq < want && base < p.n_slots) {  // nq < 64 afterwards
            const uint64_t s = base + lane;
            bool cand = false;
            if (s < p.n_slots) {
                const uint4* sp = reinterpret_cast<const uint4*>(p.table + s);
                const uint4 q0 = __ldg(sp), q1 = __ldg(sp + 1);  // the body is read again soon: no evict-first hint
                cand = slot_live_ready(q0, q1, p.epoch, p.now) && issuer_covered(p, q1.y);
                if (cand && slot_bit(a.listed, (uint32_t)s)) {
                    verify_finish(p, a, (uint32_t)s, true, counts);
                    cand = false;
                }
            }
            const uint32_t bal = __ballot_sync(0xffffffffu, cand);
            if (cand) q[nq + __popc(bal & lower)] = (uint32_t)s;
            nq += __popc(bal);
            base += stride;
        }
        __syncwarp();
        if (!have) {
            const uint32_t r = __popc(idle & lower);
            if (r < nq) {
                slot = q[nq - 1u - r];
                have = true;
                uint32_t b[12];
                load_body(p.table, slot, b);
                msg.build(p, b);
                walk.start(p, msg, a.levels);
            }
        }
        nq -= min(want, nq);
        __syncwarp();
        if (!__any_sync(0xffffffffu, have)) break;  // no record left in the warp's slots
        bool revoked;
        if (have && walk.step(p, msg, a.words, a.levels, a.n_levels, &revoked)) {
            verify_finish(p, a, slot, revoked, counts);
            have = false;
        }
    }
    __syncthreads();
    if (threadIdx.x < 8u && counts[threadIdx.x]) atomicAdd(a.counters + threadIdx.x, counts[threadIdx.x]);
}

// thread per listed record: the whole slot, its tag replaced by 1 for an S record and 0 for an R record
__global__ void __launch_bounds__(256) verify_gather_kernel(const KnownSlot* __restrict__ table, const uint32_t* __restrict__ list, uint64_t n,
                                                            const uint32_t* __restrict__ revoked, KnownSlot* out) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t s = list[t];
    KnownSlot r = table[s];
    r.tag = slot_bit(revoked, s) ? 0ull : 1ull;
    out[t] = r;
}

// One process per GPU, a slice of the list exchange: records [0, n) of the rank's listed records into its region on
// every rank (grid (n * 4 / 256, world); posted stores, the barrier after publishes them)
__global__ void __launch_bounds__(256) verify_peer_send_kernel(PeerExchange px, const uint4* __restrict__ recs, uint64_t n) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < 4 * n) reinterpret_cast<uint4*>(px.inbox[blockIdx.y] + (uint64_t)px.rank * px.X)[j] = recs[j];
}

inline unsigned grid(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

}  // namespace
}  // namespace ctmr

namespace {

constexpr uint32_t kMaxSalt = 32;
constexpr uint32_t kMaxLevels = 255;

// The scratch of a member (CascadeState): the slot bits, the digests and the covered bitmap and the counters first,
// then lists of list_cap and level bits of bit_words (recv: also the merge's receive side), each grown when too small.
// Every allocation is built into a local and moved in only when all of them succeeded.
int cascade_ensure(ctmr_ctx* c, uint64_t list_cap, uint64_t bit_words, bool recv) {
    const uint64_t slot_words = (c->st.table_mask + 1 + 31) / 32;
    const uint32_t issuer_cap = c->st.max_issuers;
    CascadeState* have = c->cascade.get();
    const bool base = !have || have->slot_words < slot_words || have->issuer_cap < issuer_cap;
    const bool lists = !have || have->list_cap < list_cap;
    const bool bits = !have || have->bit_words < bit_words;
    const bool rcv = recv && (!have || have->recv_words < bit_words);
    if (!base && !lists && !bits && !rcv) return CTMR_OK;
    DevBuf<uint32_t> revoked, covered, list[3], lbits, lrecv;
    DevBuf<uint8_t> dig;
    DevBuf<unsigned long long> counters;
    if (base) {
        CU(c, alloc(revoked, slot_words));
        CU(c, alloc(dig, (uint64_t)issuer_cap * 32 + 32));
        CU(c, alloc(covered, issuer_cap / 32 + 1));
        CU(c, alloc(counters, 2));
    }
    const uint64_t lc = std::max<uint64_t>(list_cap, have ? have->list_cap : 0);
    if (lists)
        for (auto& l : list) CU(c, alloc(l, std::max<uint64_t>(lc, 1)));
    const uint64_t bw = std::max<uint64_t>(bit_words, have ? have->bit_words : 0);
    if (bits) CU(c, alloc(lbits, std::max<uint64_t>(bw, 1)));
    if (rcv) CU(c, alloc(lrecv, std::max<uint64_t>(bw, 1)));
    if (!have) {
        c->cascade.reset(new (std::nothrow) CascadeState());
        if (!c->cascade) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    }
    CascadeState* s = c->cascade.get();
    if (base) {
        s->revoked = std::move(revoked);
        s->dig = std::move(dig);
        s->covered = std::move(covered);
        s->counters = std::move(counters);
        s->slot_words = slot_words;
        s->issuer_cap = issuer_cap;
    }
    if (lists) {
        for (int i = 0; i < 3; ++i) s->list[i] = std::move(list[i]);
        s->list_cap = lc;
    }
    if (bits) {
        s->bits = std::move(lbits);
        s->bit_words = bw;
    }
    if (rcv) {
        s->recv = std::move(lrecv);
        s->recv_words = bw;
    }
    return CTMR_OK;
}

// The sizing of include/ctmr.h, host IEEE double in exactly that order
struct LevelSize {
    uint32_t k;
    double m;
};
LevelSize level_size(uint64_t n, double p) {
    const double k = std::max(1.0, std::ceil(std::log(1 / p) / std::log(2)));
    const double m = std::max(8.0, std::ceil(-k * (double)n / std::log(1 - std::pow(p, 1.0 / k))));
    return LevelSize{(uint32_t)k, m};
}

// One member's records at a level: its include list (kNoList at level 1: the R list is list 0) and test list (kNoList at
// level 1: S is read from the table), how many of each, and where the records the level contains go.
struct MemberLevel {
    uint32_t inc = 0, exc = kNoList, out = 1;
    uint64_t n_inc = 0, n_exc = 0;
};

// The work of a build on its W members.  The first failure goes to `local`, and run() skips every step after it (a peer
// rank's exchanges still run).
struct Cascade {
    ctmr_ctx* const* m;
    uint32_t W;
    bool peer;  // one rank of a group of processes (W == 1)
    CascadeParams p{};
    std::vector<MemberLevel> ml;
    uint64_t R = 0, S = 0;
    PeerLocal local;

    // f() on member c unless the call has failed; a failure of f is c's
    template <class F>
    void run(ctmr_ctx* c, F&& f) {
        if (!local.code) local.fail(c, f());
    }

    // member r's R list (list 0) and counts; the list grown first to `cap`
    int split(uint32_t r, uint64_t cap, uint64_t* nr, uint64_t* ns) {
        ctmr_ctx* c = m[r];
        CU(c, cudaSetDevice(c->device));
        int rc = cascade_ensure(c, cap, 0, false);
        if (rc) return rc;
        CascadeState* s = c->cascade.get();
        CascadeParams q = params(c);
        CU(c, cudaMemsetAsync(s->counters, 0, 2 * sizeof(unsigned long long), c->stream));
        cascade_split_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(q, s->revoked, s->list[0], s->list_cap, s->counters);
        CU(c, cudaGetLastError());
        unsigned long long h[2] = {0, 0};
        CU(c, cudaMemcpyAsync(h, s->counters, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        *nr = h[0];
        *ns = h[1];
        return CTMR_OK;
    }

    CascadeParams params(ctmr_ctx* c) const {
        CascadeParams q = p;
        q.table = c->st.table;
        q.n_slots = c->st.table_mask + 1;
        q.epoch = c->st.epoch;
        q.dig = c->cascade->dig;
        q.covered = c->cascade->covered;
        return q;
    }

    // member r's test of level p.level: F into its out list; *f = how many
    int test(uint32_t r, uint64_t* f) {
        ctmr_ctx* c = m[r];
        CU(c, cudaSetDevice(c->device));
        CascadeState* s = c->cascade.get();
        const MemberLevel& l = ml[r];
        const CascadeParams q = params(c);
        CU(c, cudaMemsetAsync(s->counters, 0, sizeof(unsigned long long), c->stream));
        if (l.exc == kNoList) {
            cascade_test_table_kernel<<<c->sm_count * 8, kCascadeThreads, 0, c->stream>>>(q, s->revoked, s->bits, s->list[l.out], s->list_cap,
                                                                                         s->counters);
        } else if (l.n_exc) {
            cascade_test_kernel<<<grid(l.n_exc, kCascadeThreads), kCascadeThreads, 0, c->stream>>>(q, s->list[l.exc], l.n_exc, s->bits,
                                                                                                  s->list[l.out], s->list_cap, s->counters);
        }
        CU(c, cudaGetLastError());
        unsigned long long h = 0;
        CU(c, cudaMemcpyAsync(&h, s->counters, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        *f = h;
        return CTMR_OK;
    }

    // member r's included records into its partial bits of level p.level, `words` of them
    int insert(uint32_t r, uint64_t words) {
        ctmr_ctx* c = m[r];
        CU(c, cudaSetDevice(c->device));
        const int rc = cascade_ensure(c, 0, words, r == 0 && W > 1);
        if (rc) return rc;
        CascadeState* s = c->cascade.get();
        CU(c, cudaMemsetAsync(s->bits, 0, words * 4, c->stream));
        if (ml[r].n_inc) {
            cascade_insert_kernel<<<grid(ml[r].n_inc, kCascadeThreads), kCascadeThreads, 0, c->stream>>>(params(c), s->list[ml[r].inc],
                                                                                                        ml[r].n_inc, s->bits);
            CU(c, cudaGetLastError());
        }
        return CTMR_OK;
    }

    // a group's level (W > 1): member 0 pulls every other member's partial bits and ORs them into its own, then copies
    // the merged level back to every member
    void merge(uint64_t words) {
        if (W == 1 || local.code) return;
        ctmr_ctx *c0 = m[0], *at = c0;
        CascadeState* s0 = c0->cascade.get();
        const int rc = [&]() -> int {
            for (uint32_t r = 1; r < W; ++r) {
                ctmr_ctx* c = at = m[r];
                CU(c, cudaSetDevice(c->device));
                CU(c, cudaStreamSynchronize(c->stream));
                at = c0;
                CU(c0, cudaSetDevice(c0->device));
                CU(c0, cudaMemcpyPeerAsync(s0->recv, c0->device, c->cascade->bits, c->device, words * 4, c0->stream));
                cascade_or_kernel<<<grid(words, 256), 256, 0, c0->stream>>>(s0->bits, s0->recv, words);
                CU(c0, cudaGetLastError());
            }
            CU(c0, cudaStreamSynchronize(c0->stream));
            for (uint32_t r = 1; r < W; ++r) {
                ctmr_ctx* c = at = m[r];
                CU(c, cudaSetDevice(c->device));
                CU(c, cudaMemcpyPeerAsync(c->cascade->bits, c->device, s0->bits, c0->device, words * 4, c->stream));
            }
            return CTMR_OK;
        }();
        local.fail(at, rc);
    }
};

int launched(ctmr_ctx* c) {
    CU(c, cudaGetLastError());
    return CTMR_OK;
}

int set_device(ctmr_ctx* c) {
    CU(c, cudaSetDevice(c->device));
    return CTMR_OK;
}

// the OR all-reduce of words [0, words) of every rank's bits, slice by slice; `work` false (this rank failed): the
// barriers only
int cascade_peer_or(ctmr_ctx* c, uint32_t* bits, uint64_t words, bool work) {
    const uint64_t per = c->px.X * (sizeof(ctmr_key) / sizeof(uint32_t));
    int rc = CTMR_OK;
    for (uint64_t lo = 0; lo < words; lo += per) {
        const uint64_t n = std::min(per, words - lo);
        work = work && rc == CTMR_OK;
        if (work) {
            cascade_peer_send_kernel<<<dim3(grid(n, 256), c->px.world), 256, 0, c->stream>>>(c->px, bits + lo, n);
            rc = launched(c);
        }
        int brc = peer_barrier(c, CH_CRL, c->stream);  // every region of the slice has landed
        if (rc == CTMR_OK) rc = brc;
        if (rc == CTMR_OK && work) {
            cascade_peer_or_kernel<<<grid(n, 256), 256, 0, c->stream>>>(c->px, bits + lo, n);
            rc = launched(c);
        }
        brc = peer_barrier(c, CH_CRL, c->stream);  // every rank has read the slice: the regions are free again
        if (rc == CTMR_OK) rc = brc;
    }
    return rc;
}

// One mailbox exchange of this rank's payload, or of its failure.  false: some rank failed (every rank reads the same
// row and goes to the final agreement); else *sum = the sum of the payloads, and row_out (if given) every rank's.
bool peer_sum(ctmr_ctx* c, PeerLocal& local, uint64_t mine, uint64_t* sum, uint64_t* row_out = nullptr) {
    uint64_t row[kMaxWorld] = {};
    const int rc = peer_mailbox(c, peer_word(local.code, mine), row);
    if (rc) {
        local.fail(c, rc);
        return false;
    }
    const uint32_t W = c->st.peer.world;
    if (peer_row_failed(row, W) < W) return false;
    *sum = 0;
    for (uint32_t r = 0; r < W; ++r) *sum += row[r];
    if (row_out) std::copy(row, row + W, row_out);
    return true;
}

struct ByteSpan {
    const void* p;
    uint64_t n;
};

// The arguments that define the outputs (`what` names them) must be rank 0's on every rank: one mailbox word each, 63
// bits of FNV-1a over the spans' bytes back to back
int peer_same_args(ctmr_ctx* c, std::initializer_list<ByteSpan> args, const char* call, const char* what) {
    uint64_t h = 14695981039346656037ull;
    for (const ByteSpan& s : args)
        for (uint64_t j = 0; j < s.n; ++j) h = (h ^ static_cast<const uint8_t*>(s.p)[j]) * 1099511628211ull;
    h >>= 1;
    uint64_t row[kMaxWorld] = {};
    int rc = peer_mailbox(c, h, row);
    if (rc == CTMR_OK) rc = ctmr_check_device(c, nullptr);  // a barrier that timed out
    if (rc) return rc;
    if (h != row[0]) return fail(c, CTMR_E_INVALID, std::string(call) + what + " differs from rank 0's");
    for (uint32_t r = 1; r < c->st.peer.world; ++r)
        if (row[r] != row[0])
            return fail(c, CTMR_E_PEER_FAILED, std::string(call) + "rank " + std::to_string(r) + "'s " + what + " differs from rank 0's");
    return CTMR_OK;
}

// a count summed over the members, or over the ranks; false: the build stops (it failed here, or on a peer rank)
bool cascade_total(Cascade& cs, const std::vector<uint64_t>& v, uint64_t* sum) {
    if (cs.peer) return peer_sum(cs.m[0], cs.local, v[0], sum);
    *sum = 0;
    for (const uint64_t x : v) *sum += x;
    return !cs.local.code;
}

// The front half of the cascade, which the stash shares: every member's scratch (slot bits cleared, the registry's
// digests), the mark, the coverage and the split.  cs.p holds n_issuers, now and the salt; issuer[] is each CRL's dense
// issuer, row agreement 1's row (peer ranks).  Afterwards crl_status[] holds each CRL's status, *n_covered the covered
// issuers, cs.R and cs.S the sizes, and each member's R list is list 0 (ml[r].n_inc records; n_exc: its |S|).  false:
// the build stops (it failed here, or on a peer rank).
bool cascade_front(Cascade& cs, const ctmr_crl_batch* b, const std::vector<uint32_t>& issuer, uint64_t* row,
                   std::vector<uint8_t>& crl_status, uint32_t* n_covered) {
    ctmr_ctx* const* m = cs.m;
    ctmr_ctx* c0 = m[0];
    const uint32_t W = cs.W, n_issuers = cs.p.n_issuers;
    const bool peer = cs.peer;
    const int64_t now = cs.p.now;
    const uint64_t IW = c0->st.max_issuers / 32 + 1;  // words of the seen bitmap, and of the bad one after it
    PeerLocal& local = cs.local;

    // every member's scratch, its slot bits cleared, the registry's digests
    for (uint32_t r = 0; r < W; ++r)
        cs.run(m[r], [&, c = m[r]]() -> int {
            CU(c, cudaSetDevice(c->device));
            const int rc2 = cascade_ensure(c, 0, 0, false);
            if (rc2) return rc2;
            CascadeState* s = c->cascade.get();
            CU(c, cudaMemsetAsync(s->revoked, 0, s->slot_words * 4, c->stream));
            if (n_issuers) CU(c, cudaMemcpyAsync(s->dig, c0->digests.data(), (size_t)n_issuers * 32, cudaMemcpyHostToDevice, c->stream));
            CU(c, cudaStreamSynchronize(c->stream));
            return CTMR_OK;
        });

    // mark: every member's shard against each chunk's set, or a peer rank's against each round's union set
    const CrlSetVisit mark = [&](ctmr_ctx* c, const CrlSet& set) -> int {
        cascade_mark_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->st.table, c->st.table_mask + 1, c->st.epoch, now, set.slots, set.mask,
                                                                    c->cascade->revoked);
        return launched(c);
    };
    if (!crl_each_set(m, W, peer, b, issuer, row, mark, crl_status, local)) return false;

    // coverage: every CRL of an issuer in the batch is CTMR_CRL_OK
    std::vector<uint32_t> sb(2 * IW, 0);  // seen, then bad
    for (uint64_t k = 0; k < b->n_crls; ++k) {
        const uint32_t i = issuer[k];
        if (i >= n_issuers) continue;
        sb[i >> 5] |= 1u << (i & 31);
        if (crl_status[k] != CTMR_CRL_OK) sb[IW + (i >> 5)] |= 1u << (i & 31);
    }
    if (peer) {
        uint32_t* bits = c0->cascade->bits;
        cs.run(c0, [&]() -> int {
            CU(c0, cudaMemcpyAsync(bits, sb.data(), sb.size() * 4, cudaMemcpyHostToDevice, c0->stream));
            return CTMR_OK;
        });
        local.fail(c0, cascade_peer_or(c0, bits, 2 * IW, !local.code));
        cs.run(c0, [&]() -> int {
            CU(c0, cudaMemcpyAsync(sb.data(), bits, sb.size() * 4, cudaMemcpyDeviceToHost, c0->stream));
            CU(c0, cudaStreamSynchronize(c0->stream));
            return CTMR_OK;
        });
    }
    std::vector<uint32_t> covered(n_issuers / 32 + 1, 0);
    for (uint32_t i = 0; i < n_issuers; ++i)
        if ((sb[i >> 5] & ~sb[IW + (i >> 5)]) >> (i & 31) & 1u) {
            covered[i >> 5] |= 1u << (i & 31);
            ++*n_covered;
        }

    // R and S: each member's R list and counts
    std::vector<uint64_t> nr(W, 0), ns(W, 0);
    for (uint32_t r = 0; r < W; ++r)
        cs.run(m[r], [&, c = m[r]]() -> int {
            CU(c, cudaSetDevice(c->device));
            CU(c, cudaMemcpyAsync(c->cascade->covered, covered.data(), covered.size() * 4, cudaMemcpyHostToDevice, c->stream));
            int rc2 = cs.split(r, c->cascade->list_cap, &nr[r], &ns[r]);
            if (rc2 == CTMR_OK && nr[r] > c->cascade->list_cap) rc2 = cs.split(r, nr[r], &nr[r], &ns[r]);
            return rc2;
        });
    if (!cascade_total(cs, nr, &cs.R) || !cascade_total(cs, ns, &cs.S)) return false;
    for (uint32_t r = 0; r < W; ++r) {
        cs.ml[r].n_inc = nr[r];
        cs.ml[r].n_exc = ns[r];
    }
    return true;
}

// ---- the call ---------------------------------------------------------------------------------------------------------
// One driver builds the cascade on the members this process holds: a group's W members, one ctx (W == 1), or one rank
// of a group of processes (W == 1; the call is collective, include/ctmr.h states the rules).  The phases run in the same
// order in every form, and only these steps differ:
//   checks    one ctx or a group: the arguments and crl_prepare, and a failure returns at once.  A peer rank: the same
//             checks and every allocation of the call, carried in agreement 1 with the rank's chunk count; then one more
//             mailbox word, a hash of (now, salt), which must equal rank 0's.
//   mark      one call, crl_each_set, which takes the form.  One ctx or a group: member 0 builds each chunk's set, and
//             every member marks its shard against its copy of it.  A peer rank: the steps and rounds of the collective
//             ctmr_revoked_known; in each round the rank marks its shard against the union set of every rank's valid
//             records of the round.
//   coverage  seen and bad bitmaps over dense indices from the CRLs' statuses (peer ranks: each from its own CRLs, then
//             OR-reduced over the ranks); covered = seen & ~bad
//   counts    |R|, |S| and |F_l| are sums over the members, or mailbox sums over the ranks
//   merge     each member inserts its own include list into partial bits; a group's member 0 pulls them, ORs them
//             (cascade_or) and copies the merged level back; peer ranks OR-reduce them on every rank (cascade_peer_or)
//   finish    one ctx or a group: the cap check.  A peer rank: crl_peer_finish, whose final agreement makes a failure on
//             any rank every rank's, and then a cap too small on any rank every rank's CTMR_E_BATCH_TOO_LARGE.
// The OR all-reduce goes through the parity-0 region of source `rank` on every rank, 16 X words a slice: the rank's words
// of the slice into that region on every rank, a barrier, the OR of the world regions into the rank's bits, a barrier.
// One ctx or a group stops at its first failure.  A peer rank that failed after agreement 1 does no more work, but every
// decision is made from agreed sizes or from a mailbox row that every rank reads alike, so it still issues every barrier
// and exchange the others do.
int revoked_cascade(ctmr_ctx* const* m, uint32_t W, ctmr_group* g, const ctmr_crl_batch* b, int64_t now, const uint8_t* salt,
                    uint32_t salt_len, ctmr_cascade_out* out) {
    ctmr_ctx* c0 = m[0];
    const bool peer = peer_call(c0);
    const char* call = "ctmr_revoked_cascade: ";
    int rc = set_device(c0);
    if (rc) return group_fail(g, c0, rc);
    if (peer && out) out->bytes = 0;
    const uint64_t IW = c0->st.max_issuers / 32 + 1;  // words of the seen bitmap, and of the bad one after it
    std::vector<uint32_t> issuer;
    uint64_t n_chunks = 0, row[kMaxWorld] = {};
    rc = salt_len > kMaxSalt ? fail(c0, CTMR_E_INVALID, "ctmr_revoked_cascade: salt_len > 32")
             : salt_len && !salt ? fail(c0, CTMR_E_INVALID, "ctmr_revoked_cascade: NULL salt")
                                 : CTMR_OK;
    if (rc == CTMR_OK) rc = crl_prepare(c0, b, out, call, issuer, &n_chunks);
    if (rc == CTMR_OK && peer) rc = cascade_ensure(c0, 0, 2 * IW, false);
    if (rc == CTMR_OK) rc = refresh_digests(c0);
    if (peer && (rc = peer_agree(c0, rc, n_chunks, row, call, "collective call failed")) == CTMR_OK) {  // agreement 1
        const uint8_t sl = (uint8_t)salt_len;
        rc = peer_same_args(c0, {{&now, 8}, {&sl, 1}, {salt, salt_len}}, call, "now_unix_sec or salt");
    }
    if (rc) return group_fail(g, c0, rc);

    Cascade cs{m, W, peer};
    cs.p.n_issuers = (uint32_t)c0->digests.size();
    cs.p.salt_len = salt_len;
    cs.p.now = now;
    for (uint32_t j = 0; j < salt_len; ++j) cs.p.salt[j >> 2] |= (uint32_t)salt[j] << (8 * (j & 3));
    cs.p.one = 1;
    cs.ml.assign(W, MemberLevel{});
    PeerLocal& local = cs.local;

    std::vector<uint8_t> crl_status(b->n_crls, CTMR_CRL_OK);
    std::vector<uint8_t> img;
    uint32_t n_covered = 0, level = 0;
    const auto build = [&]() {  // every return is one that all peer ranks take together, to the finish
        if (!cascade_front(cs, b, issuer, row, crl_status, &n_covered)) return;

        // the levels, each merged and read back into the image behind the header
        img = {2, 0, 0, (uint8_t)salt_len};
        img.insert(img.end(), salt, salt + salt_len);
        uint64_t n_inc = cs.R;
        std::vector<uint64_t> fr(W, 0);  // each member's F_l
        for (;;) {
            if (++level > kMaxLevels) {
                local.fail(c0, fail(c0, CTMR_E_INVALID, "ctmr_revoked_cascade: more than 255 levels; build with another salt"));
                return;
            }
            const double p = level == 1 ? (cs.R == 0 || cs.S == 0 ? 0.5 : std::min(0.5, (double)cs.R / (std::sqrt(2.0) * (double)cs.S))) : 0.5;
            const LevelSize ls = level_size(n_inc, p);
            if (ls.m >= 4294967296.0) {
                out->bytes = 0;
                local.fail(c0, fail(c0, CTMR_E_BATCH_TOO_LARGE, "ctmr_revoked_cascade: level " + std::to_string(level) + " needs 2^32 bits or more"));
                return;
            }
            const uint32_t mbits = (uint32_t)ls.m;
            const uint64_t words = ((uint64_t)mbits + 31) / 32;
            cs.p.level = level;
            cs.p.k = ls.k;
            cs.p.m = mbits;
            for (uint32_t r = 0; r < W; ++r) cs.run(m[r], [&] { return cs.insert(r, words); });
            if (peer) local.fail(c0, cascade_peer_or(c0, c0->cascade->bits, words, !local.code));
            else cs.merge(words);
            for (uint32_t r = 0; r < W; ++r)
                cs.run(m[r], [&]() -> int {
                    int rc2 = cs.test(r, &fr[r]);
                    if (rc2 == CTMR_OK && fr[r] > m[r]->cascade->list_cap) {  // level 1 only: F_1 outgrew the lists, which hold R; make room and run again
                        uint64_t nr2 = 0, ns2 = 0;
                        rc2 = cs.split(r, fr[r], &nr2, &ns2);
                        if (rc2 == CTMR_OK) rc2 = cs.test(r, &fr[r]);
                    }
                    return rc2;
                });
            uint64_t F = 0;
            if (!cascade_total(cs, fr, &F)) return;
            const uint64_t nbytes = ((uint64_t)mbits + 7) / 8;
            const size_t at = img.size();
            img.resize(at + 10 + nbytes);
            img[at] = 2;
            std::memcpy(&img[at + 1], &mbits, 4);
            std::memcpy(&img[at + 5], &ls.k, 4);
            img[at + 9] = (uint8_t)level;
            cs.run(c0, [&]() -> int {
                CU(c0, cudaSetDevice(c0->device));
                CU(c0, cudaMemcpyAsync(&img[at + 10], c0->cascade->bits, nbytes, cudaMemcpyDeviceToHost, c0->stream));
                CU(c0, cudaStreamSynchronize(c0->stream));
                return CTMR_OK;
            });
            if (F == 0 || (local.code && !peer)) return;  // one ctx or a group stops at its first failure
            for (uint32_t r = 0; r < W; ++r) {  // I_{l+1} = F_l, E_{l+1} = I_l
                MemberLevel& l = cs.ml[r];
                const uint32_t free_list = l.exc == kNoList ? 3 - l.inc - l.out : l.exc;
                l.exc = l.inc;
                l.n_exc = l.n_inc;
                l.inc = l.out;
                l.n_inc = fr[r];
                l.out = free_list;
            }
            n_inc = F;
        }
    };
    build();

    const bool short_cap = img.size() > out->cap || !out->buf;
    rc = peer ? crl_peer_finish(c0, local, short_cap ? 1 : 0, row, call) : local.code;
    if (rc) {
        if (g) g->err = local.err;  // the failing member's text is the group's
        return rc;
    }
    if (!peer) row[0] = short_cap;  // as the only rank
    out->bytes = img.size();
    const uint32_t world = peer ? c0->st.peer.world : 1, me = peer ? c0->px.rank : 0;
    for (uint32_t r = 0; r < world; ++r)
        if (row[r])
            return group_fail(g, c0, fail(c0, CTMR_E_BATCH_TOO_LARGE, r == me ? "ctmr_revoked_cascade: cap " + std::to_string(out->cap) + " < " + std::to_string(img.size()) + " bytes"
                                                                             : "ctmr_revoked_cascade: rank " + std::to_string(r) + "'s cap < " + std::to_string(img.size()) + " bytes"));
    std::memcpy(out->buf, img.data(), img.size());
    if (out->crl_status) std::memcpy(out->crl_status, crl_status.data(), crl_status.size());
    out->issuers = n_covered;
    out->levels = level;
    out->revoked = cs.R;
    out->valid = cs.S;
    return CTMR_OK;
}

// ---- the stash ------------------------------------------------------------------------------------------------------
constexpr uint32_t kMaxStashK = 64;  // a bound on each thread's hashes per level; the build's k is far below it

// A published filter checked against include/ctmr.h's layout: its salt, and each level's bits laid out again in words
// from a 16-byte boundary (bit j stays (byte[j >> 3] >> (j & 7)) & 1: words are little-endian), with its level table.
struct StashFilter {
    uint32_t salt_len = 0;
    const uint8_t* salt = nullptr;
    std::vector<StashLevel> levels;
    std::vector<uint32_t> words;
};

// nullptr, or what is wrong with the filter
const char* stash_filter(const uint8_t* f, uint64_t n, StashFilter& out) {
    if (n < 4) return "filter shorter than its header";
    if (f[0] != 2 || f[1] != 0) return "filter version is not 2";
    if (f[2] != 0) return "filter is inverted";
    out.salt_len = f[3];
    out.salt = f + 4;
    if (out.salt_len > kMaxSalt) return "filter salt_len > 32";
    if (n - 4 < out.salt_len) return "filter truncated in its salt";
    for (uint64_t o = 4 + out.salt_len; o < n;) {
        if (n - o < 10) return "filter truncated in a level header";
        uint32_t m, k;
        std::memcpy(&m, f + o + 1, 4);
        std::memcpy(&k, f + o + 5, 4);
        if (f[o] != 2) return "filter level hash is not 2";
        if (k < 1 || k > kMaxStashK) return "filter level k is not in [1, 64]";
        if (m < 8) return "filter level m < 8";
        if (f[o + 9] != out.levels.size() + 1) return "filter level number is not its position";
        const uint64_t nbytes = ((uint64_t)m + 7) / 8;
        o += 10;
        if (n - o < nbytes) return "filter truncated in a level's bits";
        if ((m & 7u) && f[o + nbytes - 1] >> (m & 7u)) return "filter level has unused high bits set";
        const uint64_t at = out.words.size();
        out.levels.push_back(StashLevel{at, m, k});
        out.words.resize(at + ((nbytes + 15) / 16) * 4, 0u);
        std::memcpy(out.words.data() + at, f + o, nbytes);
        o += nbytes;
    }
    return out.levels.empty() ? "filter has no level" : nullptr;
}

// nullptr, or what is wrong with the stashes; every listed (digest || serial) into `listed`
const char* stash_parse(const uint8_t* s, uint64_t n, std::unordered_set<std::string>& listed) {
    for (uint64_t o = 0; o < n;) {
        if (n - o < 37) return "stash truncated in a unit header";
        uint32_t cnt;
        std::memcpy(&cnt, s + o, 4);
        if (s[o + 4] != 32) return "stash unit hash length is not 32";
        const char* dig = reinterpret_cast<const char*>(s + o + 5);
        o += 37;
        for (uint32_t e = 0; e < cnt; ++e) {
            if (o >= n || n - o - 1 < s[o]) return "stash truncated in an entry";
            std::string key(dig, 32);
            key.append(reinterpret_cast<const char*>(s + o + 1), s[o]);
            listed.insert(std::move(key));
            o += 1 + s[o];
        }
    }
    return nullptr;
}

// all or nothing, like cascade_ensure: the filter words, the level table and the bodies of `records` R records
int stash_ensure(ctmr_ctx* c, uint64_t words, uint64_t levels, uint64_t records) {
    StashState* have = c->stash.get();
    const bool w = !have || have->word_cap < words;
    const bool l = !have || have->level_cap < levels;
    const bool bd = !have || have->body_cap < records;
    if (!w && !l && !bd) return CTMR_OK;
    DevBuf<uint32_t> nw, nb;
    DevBuf<StashLevel> nl;
    if (w) CU(c, alloc(nw, std::max<uint64_t>(words, 1)));
    if (l) CU(c, alloc(nl, std::max<uint64_t>(levels, 1)));
    if (bd) CU(c, alloc(nb, 11 * std::max<uint64_t>(records, 1)));
    if (!have) {
        c->stash.reset(new (std::nothrow) StashState());
        if (!c->stash) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    }
    StashState* s = c->stash.get();
    if (w) {
        s->words = std::move(nw);
        s->word_cap = words;
    }
    if (l) {
        s->levels = std::move(nl);
        s->level_cap = levels;
    }
    if (bd) {
        s->bodies = std::move(nb);
        s->body_cap = records;
    }
    return CTMR_OK;
}

// member r's query of its R list (list 0 after cascade_front) against the filter: the records it calls revoked are
// counted in *in_filter, the others' (digest || serial) appended to `cand`
int stash_query(Cascade& cs, uint32_t r, const StashFilter& f, uint64_t* in_filter, std::vector<std::string>& cand) {
    ctmr_ctx* c = cs.m[r];
    const uint64_t n = cs.ml[r].n_inc;
    if (n == 0) return CTMR_OK;
    CU(c, cudaSetDevice(c->device));
    const int rc = stash_ensure(c, f.words.size(), f.levels.size(), n);
    if (rc) return rc;
    StashState* s = c->stash.get();
    CascadeState* cst = c->cascade.get();
    CU(c, cudaMemcpyAsync(s->words, f.words.data(), f.words.size() * 4, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(s->levels, f.levels.data(), f.levels.size() * sizeof(StashLevel), cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemsetAsync(cst->counters, 0, 2 * sizeof(unsigned long long), c->stream));
    stash_query_kernel<<<grid(n, kCascadeThreads), kCascadeThreads, 0, c->stream>>>(cs.params(c), cst->list[0], n, s->words, s->levels,
                                                                                  (uint32_t)f.levels.size(), s->bodies, cst->counters);
    CU(c, cudaGetLastError());
    unsigned long long h[2] = {0, 0};
    CU(c, cudaMemcpyAsync(h, cst->counters, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    std::vector<uint32_t> body(11 * h[0]);
    if (h[0]) {
        CU(c, cudaMemcpyAsync(body.data(), s->bodies, body.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
    }
    *in_filter += h[1];
    const auto& dig = cs.m[0]->digests;
    for (uint64_t i = 0; i < h[0]; ++i) {
        const uint32_t* b = &body[11 * i];  // issuer, then serial_len and serial[39] from byte 4
        const uint8_t* sb = reinterpret_cast<const uint8_t*>(b + 1);
        std::string key(reinterpret_cast<const char*>(dig[b[0]].data()), 32);
        key.append(reinterpret_cast<const char*>(sb + 1), sb[0]);
        cand.push_back(std::move(key));
    }
    return CTMR_OK;
}

// ctmr_revoked_stash on one ctx or a group: the checks, cascade_front, each member's query, and on the host the drop of
// the pairs the earlier stashes list, the sort and the serialization (include/ctmr.h states the rules)
int revoked_stash(ctmr_ctx* const* m, uint32_t W, ctmr_group* g, const ctmr_crl_batch* b, int64_t now, const uint8_t* filter,
                  uint64_t filter_bytes, const uint8_t* stashes, uint64_t stash_bytes, ctmr_stash_out* out) {
    ctmr_ctx* c0 = m[0];
    const char* call = "ctmr_revoked_stash: ";
    int rc = set_device(c0);
    if (rc) return group_fail(g, c0, rc);
    std::vector<uint32_t> issuer;
    uint64_t n_chunks = 0;  // a peer rank's: the stash is refused there
    StashFilter f;
    std::unordered_set<std::string> listed;
    const char* bad = !filter && filter_bytes ? "NULL filter" : !stashes && stash_bytes ? "NULL stashes" : nullptr;
    if (!bad) bad = stash_filter(filter, filter_bytes, f);
    if (!bad) bad = stash_parse(stashes, stash_bytes, listed);
    rc = bad ? fail(c0, CTMR_E_INVALID, std::string(call) + bad) : crl_prepare(c0, b, out, call, issuer, &n_chunks);
    if (rc == CTMR_OK) rc = refresh_digests(c0);
    if (rc) return group_fail(g, c0, rc);

    Cascade cs{m, W, false};
    cs.p.n_issuers = (uint32_t)c0->digests.size();
    cs.p.salt_len = f.salt_len;
    cs.p.now = now;
    for (uint32_t j = 0; j < f.salt_len; ++j) cs.p.salt[j >> 2] |= (uint32_t)f.salt[j] << (8 * (j & 3));
    cs.p.one = 1;
    cs.ml.assign(W, MemberLevel{});
    std::vector<uint8_t> crl_status(b->n_crls, CTMR_CRL_OK);
    uint32_t n_covered = 0;
    uint64_t in_filter = 0;
    std::vector<std::string> cand;
    if (cascade_front(cs, b, issuer, nullptr, crl_status, &n_covered))
        for (uint32_t r = 0; r < W; ++r) cs.run(m[r], [&] { return stash_query(cs, r, f, &in_filter, cand); });
    if (cs.local.code) {
        if (g) g->err = cs.local.err;  // the failing member's text is the group's
        return cs.local.code;
    }

    // the new records: those no earlier stash lists; then their distinct pairs by digest, then serial
    uint64_t in_stashes = 0;
    std::vector<std::string> fresh;
    for (std::string& k : cand) {
        if (listed.count(k)) ++in_stashes;
        else fresh.push_back(std::move(k));
    }
    std::sort(fresh.begin(), fresh.end());  // std::string orders bytes as unsigned, a prefix first
    fresh.erase(std::unique(fresh.begin(), fresh.end()), fresh.end());
    std::vector<uint8_t> img;
    uint32_t units = 0;
    for (size_t i = 0; i < fresh.size();) {
        size_t j = i;
        while (j < fresh.size() && fresh[j].compare(0, 32, fresh[i], 0, 32) == 0) ++j;
        const uint32_t cnt = (uint32_t)(j - i);
        const size_t at = img.size();
        img.resize(at + 37);
        std::memcpy(&img[at], &cnt, 4);
        img[at + 4] = 32;
        std::memcpy(&img[at + 5], fresh[i].data(), 32);
        for (; i < j; ++i) {
            img.push_back((uint8_t)(fresh[i].size() - 32));
            img.insert(img.end(), fresh[i].begin() + 32, fresh[i].end());
        }
        ++units;
    }

    out->bytes = img.size();
    if (img.size() > out->cap || (!out->buf && !img.empty()))
        return group_fail(g, c0, fail(c0, CTMR_E_BATCH_TOO_LARGE, "ctmr_revoked_stash: cap " + std::to_string(out->cap) + " < " + std::to_string(img.size()) + " bytes"));
    if (!img.empty()) std::memcpy(out->buf, img.data(), img.size());
    if (out->crl_status) std::memcpy(out->crl_status, crl_status.data(), crl_status.size());
    out->issuers = n_covered;
    out->stash_issuers = units;
    out->revoked = cs.R;
    out->in_filter = in_filter;
    out->in_stashes = in_stashes;
    out->serials = fresh.size();
    return CTMR_OK;
}

// ---- the verify -----------------------------------------------------------------------------------------------------
// all or nothing, like cascade_ensure: the listed bits and the counters, a set of set_slots slots and room for `records`
// listed records
int verify_ensure(ctmr_ctx* c, uint64_t set_slots, uint64_t records) {
    const uint64_t slot_words = (c->st.table_mask + 1 + 31) / 32;
    VerifyState* have = c->verify.get();
    const bool base = !have || have->slot_words < slot_words;
    const bool st = !have || have->set_cap < set_slots;
    const bool rs = !have || have->rec_cap < records;
    if (!base && !st && !rs) return CTMR_OK;
    DevBuf<uint32_t> listed;
    DevBuf<unsigned long long> counters;
    DevBuf<CrlSetSlot> set;
    DevBuf<KnownSlot> recs;
    if (base) {
        CU(c, alloc(listed, slot_words));
        CU(c, alloc(counters, 9));
    }
    if (st) CU(c, alloc(set, std::max<uint64_t>(set_slots, 1)));
    if (rs) CU(c, alloc(recs, std::max<uint64_t>(records, 1)));
    if (!have) {
        c->verify.reset(new (std::nothrow) VerifyState());
        if (!c->verify) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    }
    VerifyState* s = c->verify.get();
    if (base) {
        s->listed = std::move(listed);
        s->counters = std::move(counters);
        s->slot_words = slot_words;
    }
    if (st) {
        s->set = std::move(set);
        s->set_cap = std::max<uint64_t>(set_slots, 1);
    }
    if (rs) {
        s->recs = std::move(recs);
        s->rec_cap = std::max<uint64_t>(records, 1);
    }
    return CTMR_OK;
}

// The stashes' pairs as the slots of a CrlSet (the join's key words, pair_hash, linear probing, at least twice the
// pairs' slots): every listed (digest || serial) whose digest is registered and whose serial a key can hold.  Empty when
// there is none.
std::vector<CrlSetSlot> verify_stash_set(const std::vector<std::array<uint8_t, 32>>& digests, const std::unordered_set<std::string>& listed) {
    std::unordered_map<std::string, uint32_t> dense;
    for (uint32_t i = 0; i < digests.size(); ++i) dense.emplace(std::string(reinterpret_cast<const char*>(digests[i].data()), 32), i);
    std::vector<std::array<uint32_t, 11>> keys;
    for (const std::string& x : listed) {
        const auto it = dense.find(x.substr(0, 32));
        if (x.size() - 32 > CTMR_MAX_SERIAL || it == dense.end()) continue;  // never matches
        std::array<uint32_t, 11> w{};
        w[0] = it->second;
        uint8_t* sb = reinterpret_cast<uint8_t*>(w.data() + 1);  // serial_len, then the serial, zero padded
        sb[0] = (uint8_t)(x.size() - 32);
        std::memcpy(sb + 1, x.data() + 32, x.size() - 32);
        keys.push_back(w);
    }
    if (keys.empty()) return {};
    uint64_t n = 64;
    while (n < 2 * keys.size()) n <<= 1;
    std::vector<CrlSetSlot> set(n, CrlSetSlot{});
    for (const auto& k : keys) {
        uint32_t w[11];
        std::copy(k.begin(), k.end(), w);
        const uint32_t h = pair_hash(w);
        uint64_t pos = h & (n - 1);
        while (set[pos].tag) pos = (pos + 1) & (n - 1);  // the pairs are distinct
        set[pos].tag = (h & ~3u) | 2u;
        std::copy(w, w + 11, set[pos].key);
    }
    return set;
}

// member r's verify after cascade_front: the stashes' set marked into the listed bits, the pass over the shard (run
// again with longer lists when its listed records outgrew them), counts[0..8) = its counts, and its listed records
// gathered into VerifyState::recs and appended to `recs`
int verify_member(Cascade& cs, uint32_t r, const StashFilter& f, const std::vector<CrlSetSlot>& set, uint64_t covered_below,
                  uint64_t* counts, std::vector<KnownSlot>& recs) {
    ctmr_ctx* c = cs.m[r];
    CU(c, cudaSetDevice(c->device));
    int rc = stash_ensure(c, f.words.size(), f.levels.size(), 0);
    if (rc == CTMR_OK) rc = verify_ensure(c, set.size(), 0);
    if (rc) return rc;
    StashState* s = c->stash.get();
    VerifyState* v = c->verify.get();
    CascadeState* cst = c->cascade.get();
    const CascadeParams q = cs.params(c);
    CU(c, cudaMemcpyAsync(s->words, f.words.data(), f.words.size() * 4, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(s->levels, f.levels.data(), f.levels.size() * sizeof(StashLevel), cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemsetAsync(v->listed, 0, v->slot_words * 4, c->stream));
    if (!set.empty()) {
        CU(c, cudaMemcpyAsync(v->set, set.data(), set.size() * sizeof(CrlSetSlot), cudaMemcpyHostToDevice, c->stream));
        cascade_mark_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(q.table, q.n_slots, q.epoch, q.now, v->set, set.size() - 1, v->listed);
        CU(c, cudaGetLastError());
    }
    unsigned long long h[9] = {};
    for (;;) {
        const VerifyArgs a{cst->revoked, v->listed, s->words, s->levels, (uint32_t)f.levels.size(), covered_below, cst->list[1], cst->list_cap,
                           v->counters};
        CU(c, cudaMemsetAsync(v->counters, 0, sizeof(h), c->stream));
        verify_table_kernel<<<c->sm_count * kVerifyBlocksPerSm, kCascadeThreads, 0, c->stream>>>(q, a);
        CU(c, cudaGetLastError());
        CU(c, cudaMemcpyAsync(h, v->counters, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        if (h[8] <= cst->list_cap) break;
        if ((rc = cascade_ensure(c, h[8], 0, false))) return rc;
    }
    std::copy(h, h + 8, counts);
    if (h[8] == 0) return CTMR_OK;
    if ((rc = verify_ensure(c, 0, h[8]))) return rc;
    verify_gather_kernel<<<grid(h[8], 256), 256, 0, c->stream>>>(q.table, cst->list[1], h[8], cst->revoked, v->recs);
    CU(c, cudaGetLastError());
    const size_t at = recs.size();
    recs.resize(at + h[8]);
    CU(c, cudaMemcpyAsync(recs.data() + at, v->recs, h[8] * sizeof(KnownSlot), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return CTMR_OK;
}

// Peer ranks: every other rank's listed records (n[s] of rank s, agreed) appended to `recs`, slice by slice through the
// parity-0 regions: the rank's X records of the slice into its region on every rank, a barrier, the other ranks' regions
// to the host, a barrier.  `work` false (this rank failed): the barriers only.
int verify_peer_gather(ctmr_ctx* c, const uint64_t* n, std::vector<KnownSlot>& recs, bool work) {
    const PeerExchange& px = c->px;
    uint64_t most = 0;
    for (uint32_t r = 0; r < px.world; ++r) most = std::max(most, n[r]);
    int rc = CTMR_OK;
    for (uint64_t lo = 0; lo < most; lo += px.X) {
        work = work && rc == CTMR_OK;
        if (work && n[px.rank] > lo) {
            const uint64_t k = std::min(px.X, n[px.rank] - lo);
            verify_peer_send_kernel<<<dim3(grid(4 * k, 256), px.world), 256, 0, c->stream>>>(
                px, reinterpret_cast<const uint4*>(c->verify->recs.get() + lo), k);
            rc = launched(c);
        }
        int brc = peer_barrier(c, CH_CRL, c->stream);  // every region of the slice has landed
        if (rc == CTMR_OK) rc = brc;
        if (rc == CTMR_OK && work)
            rc = [&]() -> int {
                for (uint32_t s = 0; s < px.world; ++s) {
                    if (s == px.rank || n[s] <= lo) continue;
                    const uint64_t k = std::min(px.X, n[s] - lo);
                    const size_t at = recs.size();
                    recs.resize(at + k);
                    CU(c, cudaMemcpyAsync(recs.data() + at, px.inbox[px.rank] + (uint64_t)s * px.X, k * sizeof(KnownSlot), cudaMemcpyDeviceToHost,
                                          c->stream));
                }
                CU(c, cudaStreamSynchronize(c->stream));
                return CTMR_OK;
            }();
        brc = peer_barrier(c, CH_CRL, c->stream);  // every rank has read the slice: the regions are free again
        if (rc == CTMR_OK) rc = brc;
    }
    return rc;
}

// One driver for one ctx, a group and one rank of a group of processes, in revoked_cascade's phases: its checks (with the
// stash's checks of the filter and the stashes) and agreements (the hash covers now, covered_below, the filter and the
// stashes), cascade_front, then every member's verify_member.  The counts are sums over the members, or mailbox sums
// over the ranks; the listed records are every member's, or every rank's after verify_peer_gather, and every rank sorts
// the same union.  The finish is the cascade's, with the list cap in place of the byte cap.
int revoked_verify(ctmr_ctx* const* m, uint32_t W, ctmr_group* g, const ctmr_crl_batch* b, int64_t now, const uint8_t* filter,
                   uint64_t filter_bytes, const uint8_t* stashes, uint64_t stash_bytes, uint64_t covered_below, ctmr_verify_out* out) {
    ctmr_ctx* c0 = m[0];
    const bool peer = peer_call(c0);
    const char* call = "ctmr_revoked_verify: ";
    int rc = set_device(c0);
    if (rc) return group_fail(g, c0, rc);
    if (peer && out) out->n_list = 0;
    const uint64_t IW = c0->st.max_issuers / 32 + 1;  // words of the seen bitmap, and of the bad one after it
    std::vector<uint32_t> issuer;
    uint64_t n_chunks = 0, row[kMaxWorld] = {};
    StashFilter f;
    std::unordered_set<std::string> listed;
    const char* bad = !filter && filter_bytes ? "NULL filter" : !stashes && stash_bytes ? "NULL stashes" : nullptr;
    if (!bad) bad = stash_filter(filter, filter_bytes, f);
    if (!bad) bad = stash_parse(stashes, stash_bytes, listed);
    rc = bad ? fail(c0, CTMR_E_INVALID, std::string(call) + bad) : crl_prepare(c0, b, out, call, issuer, &n_chunks);
    if (rc == CTMR_OK && peer) rc = cascade_ensure(c0, 0, 2 * IW, false);
    if (rc == CTMR_OK) rc = refresh_digests(c0);
    if (peer && (rc = peer_agree(c0, rc, n_chunks, row, call, "collective call failed")) == CTMR_OK)  // agreement 1
        rc = peer_same_args(c0, {{&now, 8}, {&covered_below, 8}, {&filter_bytes, 8}, {filter, filter_bytes}, {&stash_bytes, 8}, {stashes, stash_bytes}},
                            call, "now_unix_sec, covered_below, filter or stashes");
    if (rc) return group_fail(g, c0, rc);

    Cascade cs{m, W, peer};
    cs.p.n_issuers = (uint32_t)c0->digests.size();
    cs.p.salt_len = f.salt_len;
    cs.p.now = now;
    for (uint32_t j = 0; j < f.salt_len; ++j) cs.p.salt[j >> 2] |= (uint32_t)f.salt[j] << (8 * (j & 3));
    cs.p.one = 1;
    cs.ml.assign(W, MemberLevel{});
    PeerLocal& local = cs.local;
    std::vector<uint8_t> crl_status(b->n_crls, CTMR_CRL_OK);
    uint32_t n_covered = 0;
    uint64_t counts[8] = {};
    std::vector<KnownSlot> recs;
    const auto verify = [&]() {  // every return is one that all peer ranks take together, to the finish
        if (!cascade_front(cs, b, issuer, row, crl_status, &n_covered)) return;
        const std::vector<CrlSetSlot> set = verify_stash_set(c0->digests, listed);
        std::vector<uint64_t> mc(8 * W, 0);
        for (uint32_t r = 0; r < W; ++r) cs.run(m[r], [&] { return verify_member(cs, r, f, set, covered_below, &mc[8 * r], recs); });
        if (!peer) {
            for (uint32_t j = 0; j < 8 * W; ++j) counts[j & 7] += mc[j];
            return;
        }
        for (uint32_t j = 0; j < 8; ++j)
            if (!peer_sum(c0, local, mc[j], &counts[j])) return;
        uint64_t total = 0, n[kMaxWorld] = {};
        if (!peer_sum(c0, local, recs.size(), &total, n)) return;
        local.fail(c0, verify_peer_gather(c0, n, recs, !local.code));
    };
    verify();

    const uint64_t n_list = recs.size();
    const bool short_cap = n_list > out->list_cap || (!out->list && n_list);
    rc = peer ? crl_peer_finish(c0, local, short_cap ? 1 : 0, row, call) : local.code;
    if (rc) {
        if (g) g->err = local.err;  // the failing member's text is the group's
        return rc;
    }
    if (!peer) row[0] = short_cap;  // as the only rank
    out->n_list = n_list;
    const uint32_t world = peer ? c0->st.peer.world : 1, me = peer ? c0->px.rank : 0;
    for (uint32_t r = 0; r < world; ++r)
        if (row[r])
            return group_fail(g, c0, fail(c0, CTMR_E_BATCH_TOO_LARGE, r == me ? "ctmr_revoked_verify: list_cap " + std::to_string(out->list_cap) + " < " + std::to_string(n_list) + " records"
                                                                             : "ctmr_revoked_verify: rank " + std::to_string(r) + "'s list_cap < " + std::to_string(n_list) + " records"));
    std::vector<ctmr_verify_miss> list(n_list);
    for (uint64_t i = 0; i < n_list; ++i) {
        const KnownSlot& k = recs[i];
        const uint8_t* kb = reinterpret_cast<const uint8_t*>(k.body);  // exp_hour, issuer, serial_len, serial
        ctmr_verify_miss& e = list[i];
        std::memset(&e, 0, sizeof(e));
        std::memcpy(e.digest, c0->digests[k.body[1]].data(), 32);
        e.exp_hour = (int32_t)k.body[0];
        e.first_index = ~k.inv_first;
        e.serial_len = kb[8];
        std::memcpy(e.serial, kb + 9, CTMR_MAX_SERIAL);
        e.blocked = (uint8_t)k.tag;
    }
    std::sort(list.begin(), list.end(), [](const ctmr_verify_miss& a, const ctmr_verify_miss& z) {
        if (const int d = std::memcmp(a.digest, z.digest, 32)) return d < 0;
        if (const int s = std::memcmp(a.serial, z.serial, std::min(a.serial_len, z.serial_len))) return s < 0;
        if (a.serial_len != z.serial_len) return a.serial_len < z.serial_len;
        return a.exp_hour < z.exp_hour;
    });
    if (n_list) std::memcpy(out->list, list.data(), n_list * sizeof(ctmr_verify_miss));
    if (out->crl_status) std::memcpy(out->crl_status, crl_status.data(), crl_status.size());
    out->issuers = n_covered;
    out->levels = (uint32_t)f.levels.size();
    out->before = ctmr_verify_counts{counts[0], counts[1], counts[2], counts[3]};
    out->since = ctmr_verify_counts{counts[4], counts[5], counts[6], counts[7]};
    return CTMR_OK;
}

}  // namespace

extern "C" {

int ctmr_revoked_cascade(ctmr_ctx* c, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* salt, uint32_t salt_len,
                         ctmr_cascade_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group) return fail(c, CTMR_E_INVALID, "ctmr_revoked_cascade: a member of a group; use ctmr_group_revoked_cascade");
    ctmr_ctx* m[1] = {c};
    return revoked_cascade(m, 1, nullptr, batch, now_unix_sec, salt, salt_len, out);
}

int ctmr_group_revoked_cascade(ctmr_group* g, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* salt, uint32_t salt_len,
                               ctmr_cascade_out* out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const int rc = revoked_cascade(g->m.data(), (uint32_t)g->m.size(), g, batch, now_unix_sec, salt, salt_len, out);
    cudaSetDevice(g->m[0]->device);
    return rc;
}

int ctmr_revoked_stash(ctmr_ctx* c, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* filter, uint64_t filter_bytes,
                       const uint8_t* stashes, uint64_t stash_bytes, ctmr_stash_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group) return fail(c, CTMR_E_INVALID, "ctmr_revoked_stash: a member of a group; use ctmr_group_revoked_stash");
    if (peer_call(c)) return fail(c, CTMR_E_INVALID, "ctmr_revoked_stash: not a collective call; load the ranks' checkpoint parts into one ctx or a group");
    ctmr_ctx* m[1] = {c};
    return revoked_stash(m, 1, nullptr, batch, now_unix_sec, filter, filter_bytes, stashes, stash_bytes, out);
}

int ctmr_group_revoked_stash(ctmr_group* g, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* filter, uint64_t filter_bytes,
                             const uint8_t* stashes, uint64_t stash_bytes, ctmr_stash_out* out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const int rc = revoked_stash(g->m.data(), (uint32_t)g->m.size(), g, batch, now_unix_sec, filter, filter_bytes, stashes, stash_bytes, out);
    cudaSetDevice(g->m[0]->device);
    return rc;
}

int ctmr_revoked_verify(ctmr_ctx* c, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* filter, uint64_t filter_bytes,
                        const uint8_t* stashes, uint64_t stash_bytes, uint64_t covered_below, ctmr_verify_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group) return fail(c, CTMR_E_INVALID, "ctmr_revoked_verify: a member of a group; use ctmr_group_revoked_verify");
    ctmr_ctx* m[1] = {c};
    return revoked_verify(m, 1, nullptr, batch, now_unix_sec, filter, filter_bytes, stashes, stash_bytes, covered_below, out);
}

int ctmr_group_revoked_verify(ctmr_group* g, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* filter, uint64_t filter_bytes,
                              const uint8_t* stashes, uint64_t stash_bytes, uint64_t covered_below, ctmr_verify_out* out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const int rc = revoked_verify(g->m.data(), (uint32_t)g->m.size(), g, batch, now_unix_sec, filter, filter_bytes, stashes, stash_bytes,
                                  covered_below, out);
    cudaSetDevice(g->m[0]->device);
    return rc;
}

}  // extern "C"
