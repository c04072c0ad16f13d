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
#include <cmath>

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
    const uint8_t* dig;        // [n_issuers][32] by dense index
    const uint32_t* covered;   // bit per dense index
    uint32_t n_issuers;
    uint32_t salt_len;
    int64_t now;
    uint32_t salt[8];          // little-endian words: byte j is salt[j >> 2] >> 8 (j & 3)
    uint32_t level, k, m;
    uint32_t one;              // always 1: sha256_compress's multiplier ptxas cannot fold
};

__device__ __forceinline__ bool slot_live_ready(uint4 q0, uint4 q1, int64_t now) {
    return (q0.z & 3u) == 2u && (int64_t)(int32_t)q1.x * 3600 > now;
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
__global__ void __launch_bounds__(256) cascade_mark_kernel(const KnownSlot* __restrict__ table, uint64_t n_slots, int64_t now,
                                                           const CrlSetSlot* __restrict__ set, uint64_t mask, uint32_t* revoked) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slots; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4* sp = reinterpret_cast<const uint4*>(table + i);
        const uint4 q0 = __ldcs(sp), q1 = __ldcs(sp + 1);
        if (!slot_live_ready(q0, q1, now)) continue;
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
        if (!slot_live_ready(q0, q1, p.now) || !issuer_covered(p, q1.y)) continue;
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
        if (!slot_live_ready(q0, q1, p.now) || !issuer_covered(p, q1.y)) continue;
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

// CU for the code that serves a group too: the failing ctx's error text also becomes the group's
#define CUG(g, ctx, call)                                                                                                      \
    do {                                                                                                                       \
        const cudaError_t e_ = (call);                                                                                         \
        if (e_ != cudaSuccess)                                                                                                 \
            return group_fail((g), (ctx), fail((ctx), e_ == cudaErrorMemoryAllocation ? CTMR_E_NOMEM : CTMR_E_CUDA,             \
                                               std::string(#call) + ": " + cudaGetErrorString(e_)));                           \
    } while (0)

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

struct Cascade {
    ctmr_ctx* const* m;
    uint32_t W;
    ctmr_group* g;
    CascadeParams p{};
    std::vector<MemberLevel> ml;
    uint64_t R = 0, S = 0;

    int gfail(ctmr_ctx* c, int rc) { return group_fail(g, c, rc); }

    // member r's R list (list 0) and counts; the list grown first to `cap`
    int split(uint32_t r, uint64_t cap, uint64_t* nr, uint64_t* ns) {
        ctmr_ctx* c = m[r];
        CUG(g, c, cudaSetDevice(c->device));
        int rc = cascade_ensure(c, cap, 0, false);
        if (rc) return rc;
        CascadeState* s = c->cascade.get();
        CascadeParams q = params(c);
        CUG(g, c, cudaMemsetAsync(s->counters, 0, 2 * sizeof(unsigned long long), c->stream));
        cascade_split_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(q, s->revoked, s->list[0], s->list_cap, s->counters);
        CUG(g, c, cudaGetLastError());
        unsigned long long h[2] = {0, 0};
        CUG(g, c, cudaMemcpyAsync(h, s->counters, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
        CUG(g, c, cudaStreamSynchronize(c->stream));
        *nr = h[0];
        *ns = h[1];
        return CTMR_OK;
    }

    CascadeParams params(ctmr_ctx* c) const {
        CascadeParams q = p;
        q.table = c->st.table;
        q.n_slots = c->st.table_mask + 1;
        q.dig = c->cascade->dig;
        q.covered = c->cascade->covered;
        return q;
    }

    // member r's test of level p.level: F into its out list; *f = how many
    int test(uint32_t r, uint64_t* f) {
        ctmr_ctx* c = m[r];
        CUG(g, c, cudaSetDevice(c->device));
        CascadeState* s = c->cascade.get();
        const MemberLevel& l = ml[r];
        const CascadeParams q = params(c);
        CUG(g, c, cudaMemsetAsync(s->counters, 0, sizeof(unsigned long long), c->stream));
        if (l.exc == kNoList) {
            cascade_test_table_kernel<<<c->sm_count * 8, kCascadeThreads, 0, c->stream>>>(q, s->revoked, s->bits, s->list[l.out], s->list_cap,
                                                                                         s->counters);
        } else if (l.n_exc) {
            cascade_test_kernel<<<grid(l.n_exc, kCascadeThreads), kCascadeThreads, 0, c->stream>>>(q, s->list[l.exc], l.n_exc, s->bits,
                                                                                                  s->list[l.out], s->list_cap, s->counters);
        }
        CUG(g, c, cudaGetLastError());
        unsigned long long h = 0;
        CUG(g, c, cudaMemcpyAsync(&h, s->counters, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
        CUG(g, c, cudaStreamSynchronize(c->stream));
        *f = h;
        return CTMR_OK;
    }

    // level p.level with words of bits: every member's partial bits, merged on member 0 and copied back to every member
    int insert(uint64_t words) {
        for (uint32_t r = 0; r < W; ++r) {
            ctmr_ctx* c = m[r];
            CUG(g, c, cudaSetDevice(c->device));
            int rc = cascade_ensure(c, 0, words, r == 0 && W > 1);
            if (rc) return gfail(c, rc);
            CascadeState* s = c->cascade.get();
            const CascadeParams q = params(c);
            CUG(g, c, cudaMemsetAsync(s->bits, 0, words * 4, c->stream));
            if (ml[r].n_inc) {
                cascade_insert_kernel<<<grid(ml[r].n_inc, kCascadeThreads), kCascadeThreads, 0, c->stream>>>(q, s->list[ml[r].inc], ml[r].n_inc,
                                                                                                            s->bits);
                CUG(g, c, cudaGetLastError());
            }
        }
        if (W == 1) return CTMR_OK;
        ctmr_ctx* c0 = m[0];
        CascadeState* s0 = c0->cascade.get();
        for (uint32_t r = 1; r < W; ++r) {
            ctmr_ctx* c = m[r];
            CUG(g, c, cudaSetDevice(c->device));
            CUG(g, c, cudaStreamSynchronize(c->stream));
            CUG(g, c0, cudaSetDevice(c0->device));
            CUG(g, c0, cudaMemcpyPeerAsync(s0->recv, c0->device, c->cascade->bits, c->device, words * 4, c0->stream));
            cascade_or_kernel<<<grid(words, 256), 256, 0, c0->stream>>>(s0->bits, s0->recv, words);
            CUG(g, c0, cudaGetLastError());
        }
        CUG(g, c0, cudaStreamSynchronize(c0->stream));
        for (uint32_t r = 1; r < W; ++r) {
            ctmr_ctx* c = m[r];
            CUG(g, c, cudaSetDevice(c->device));
            CUG(g, c, cudaMemcpyPeerAsync(c->cascade->bits, c->device, s0->bits, c0->device, words * 4, c->stream));
        }
        return CTMR_OK;
    }
};

// the call on member 0 of `W` members (W == 1: one ctx)
int revoked_cascade(ctmr_ctx* const* m, uint32_t W, ctmr_group* g, const ctmr_crl_batch* b, int64_t now, const uint8_t* salt,
                    uint32_t salt_len, ctmr_cascade_out* out) {
    ctmr_ctx* c0 = m[0];
    const auto gf = [&](ctmr_ctx* c, int rc) { return group_fail(g, c, rc); };
    CUG(g, c0, cudaSetDevice(c0->device));
    if (salt_len > kMaxSalt) return gf(c0, fail(c0, CTMR_E_INVALID, "ctmr_revoked_cascade: salt_len > 32"));
    if (salt_len && !salt) return gf(c0, fail(c0, CTMR_E_INVALID, "ctmr_revoked_cascade: NULL salt"));
    std::vector<uint32_t> issuer;
    int rc = crl_prepare(c0, b, out, "ctmr_revoked_cascade: ", issuer);
    if (rc) return gf(c0, rc);
    if ((rc = refresh_digests(c0))) return gf(c0, rc);
    const uint32_t n_issuers = (uint32_t)c0->digests.size();

    Cascade cs{m, W, g};
    cs.p.n_issuers = n_issuers;
    cs.p.salt_len = salt_len;
    cs.p.now = now;
    for (uint32_t j = 0; j < salt_len; ++j) cs.p.salt[j >> 2] |= (uint32_t)salt[j] << (8 * (j & 3));
    cs.p.one = 1;
    cs.ml.assign(W, MemberLevel{});

    // every member's scratch, its slot bits cleared, the registry's digests
    for (uint32_t r = 0; r < W; ++r) {
        ctmr_ctx* c = m[r];
        CUG(g, c, cudaSetDevice(c->device));
        if ((rc = cascade_ensure(c, 0, 0, false))) return gf(c, rc);
        CascadeState* s = c->cascade.get();
        CUG(g, c, cudaMemsetAsync(s->revoked, 0, s->slot_words * 4, c->stream));
        if (n_issuers) CUG(g, c, cudaMemcpyAsync(s->dig, c0->digests.data(), (size_t)n_issuers * 32, cudaMemcpyHostToDevice, c->stream));
        CUG(g, c, cudaStreamSynchronize(c->stream));
    }

    // the chunks: member 0 builds each chunk's set, every member marks its own shard against it
    std::vector<uint8_t> crl_status(b->n_crls, CTMR_CRL_OK);
    CUG(g, c0, cudaSetDevice(c0->device));
    uint32_t at = 0;  // the member the chunk path is working on: a failure's text is on it
    rc = crl_each_set(c0, b, issuer, [&](uint64_t lo, const std::vector<uint8_t>& st, const CrlSetSlot* set, uint64_t mask) -> int {
        std::copy(st.begin(), st.end(), crl_status.begin() + lo);
        if (!set) return CTMR_OK;
        for (uint32_t r = 0; r < W; ++r) {
            ctmr_ctx* c = m[at = r];
            CUG(g, c, cudaSetDevice(c->device));
            const CrlSetSlot* probe = set;
            if (r) {
                int rc2 = crl_set_ensure(c, mask + 1, false);
                if (rc2) return gf(c, rc2);
                CUG(g, c, cudaMemcpyPeerAsync(c->crl->set, c->device, set, c0->device, (mask + 1) * sizeof(CrlSetSlot), c->stream));
                probe = c->crl->set;
            }
            cascade_mark_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->st.table, c->st.table_mask + 1, now, probe, mask, c->cascade->revoked);
            CUG(g, c, cudaGetLastError());
        }
        for (uint32_t r = W; r-- > 1;) {  // the next chunk rewrites member 0's set
            at = r;
            CUG(g, m[r], cudaSetDevice(m[r]->device));
            CUG(g, m[r], cudaStreamSynchronize(m[r]->stream));
        }
        at = 0;
        CUG(g, c0, cudaSetDevice(c0->device));
        return CTMR_OK;
    });
    if (rc) return gf(m[at], rc);

    // coverage: every CRL of an issuer in the batch is CTMR_CRL_OK
    std::vector<uint8_t> seen(n_issuers, 0), bad(n_issuers, 0);
    for (uint64_t k = 0; k < b->n_crls; ++k) {
        if (issuer[k] >= n_issuers) continue;
        seen[issuer[k]] = 1;
        if (crl_status[k] != CTMR_CRL_OK) bad[issuer[k]] = 1;
    }
    std::vector<uint32_t> covered(n_issuers / 32 + 1, 0);
    uint32_t n_covered = 0;
    for (uint32_t i = 0; i < n_issuers; ++i)
        if (seen[i] && !bad[i]) {
            covered[i >> 5] |= 1u << (i & 31);
            ++n_covered;
        }

    // R and S: each member's R list and counts
    for (uint32_t r = 0; r < W; ++r) {
        ctmr_ctx* c = m[r];
        CUG(g, c, cudaSetDevice(c->device));
        CUG(g, c, cudaMemcpyAsync(c->cascade->covered, covered.data(), covered.size() * 4, cudaMemcpyHostToDevice, c->stream));
        uint64_t nr = 0, ns = 0;
        if ((rc = cs.split(r, c->cascade->list_cap, &nr, &ns))) return gf(c, rc);
        if (nr > c->cascade->list_cap && (rc = cs.split(r, nr, &nr, &ns))) return gf(c, rc);
        cs.ml[r].n_inc = nr;
        cs.ml[r].n_exc = ns;
        cs.R += nr;
        cs.S += ns;
    }

    // the levels, each read back into the image behind the header
    std::vector<uint8_t> img = {2, 0, 0, (uint8_t)salt_len};
    img.insert(img.end(), salt, salt + salt_len);
    uint64_t n_inc = cs.R;
    uint32_t level = 0;
    std::vector<uint64_t> fr(W, 0);  // each member's F_l
    for (;;) {
        if (++level > kMaxLevels)
            return gf(c0, fail(c0, CTMR_E_INVALID, "ctmr_revoked_cascade: more than 255 levels; build with another salt"));
        const double p = level == 1 ? (cs.R == 0 || cs.S == 0 ? 0.5 : std::min(0.5, (double)cs.R / (std::sqrt(2.0) * (double)cs.S))) : 0.5;
        const LevelSize ls = level_size(n_inc, p);
        if (ls.m >= 4294967296.0) {
            out->bytes = 0;
            return gf(c0, fail(c0, CTMR_E_BATCH_TOO_LARGE, "ctmr_revoked_cascade: level " + std::to_string(level) + " needs 2^32 bits or more"));
        }
        const uint32_t mbits = (uint32_t)ls.m;
        const uint64_t words = ((uint64_t)mbits + 31) / 32;
        cs.p.level = level;
        cs.p.k = ls.k;
        cs.p.m = mbits;
        if ((rc = cs.insert(words))) return rc;
        uint64_t F = 0;
        for (uint32_t r = 0; r < W; ++r) {
            uint64_t& f = fr[r];
            if ((rc = cs.test(r, &f))) return gf(m[r], rc);
            if (f > m[r]->cascade->list_cap) {  // level 1 only: F_1 outgrew the lists, which hold R; make room and run again
                uint64_t nr = 0, ns = 0;
                if ((rc = cs.split(r, f, &nr, &ns)) || (rc = cs.test(r, &f))) return gf(m[r], rc);
            }
            F += f;
        }
        const uint64_t nbytes = ((uint64_t)mbits + 7) / 8;
        const size_t at = img.size();
        img.resize(at + 10 + nbytes);
        img[at] = 2;
        std::memcpy(&img[at + 1], &mbits, 4);
        std::memcpy(&img[at + 5], &ls.k, 4);
        img[at + 9] = (uint8_t)level;
        CUG(g, c0, cudaSetDevice(c0->device));
        CUG(g, c0, cudaMemcpyAsync(&img[at + 10], c0->cascade->bits, nbytes, cudaMemcpyDeviceToHost, c0->stream));
        CUG(g, c0, cudaStreamSynchronize(c0->stream));
        if (F == 0) break;
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
    CUG(g, c0, cudaSetDevice(c0->device));
    out->bytes = img.size();
    if (img.size() > out->cap || !out->buf)
        return gf(c0, fail(c0, CTMR_E_BATCH_TOO_LARGE, "ctmr_revoked_cascade: cap " + std::to_string(out->cap) + " < " +
                                                           std::to_string(img.size()) + " bytes"));
    std::memcpy(out->buf, img.data(), img.size());
    if (out->crl_status) std::memcpy(out->crl_status, crl_status.data(), crl_status.size());
    out->issuers = n_covered;
    out->levels = level;
    out->revoked = cs.R;
    out->valid = cs.S;
    return CTMR_OK;
}

// ---- one process per GPU: the collective call on a ctx attached to peers (include/ctmr.h states the rules) -----------
// Every rank checks its arguments and builds its buffers; agreement 1 posts its chunk count (or that it failed), and one
// more mailbox word a hash of (now, salt), which must equal rank 0's.  Then:
//   mark      the steps and rounds of the collective ctmr_revoked_known (crl_peer_each_set): in each round every rank
//             marks its own shard against the union set of every rank's valid records of the round
//   coverage  each rank's seen and bad bitmaps over dense indices from its own CRLs, OR-reduced; covered = seen & ~bad;
//             each rank splits its own shard, and |R| and |S| are mailbox sums
//   levels    each rank inserts its own include list into partial bits, the OR all-reduce merges them on every rank, each
//             rank tests its own exclude list (level 1: S straight from its table); |F_l| is a mailbox sum, and every rank
//             reads the merged level into its own image
// The OR all-reduce goes through the parity-0 region of source `rank` on every rank, 16 X words a slice: the rank's words
// of the slice into that region on every rank, a barrier, the OR of the world regions into the rank's bits, a barrier.
// Every decision after agreement 1 is made from agreed sizes or from a mailbox row that every rank reads alike, so a rank
// that failed still issues every barrier and exchange the others do.  A final agreement makes its failure every rank's,
// and then a cap too small on any rank every rank's CTMR_E_BATCH_TOO_LARGE.

int launched(ctmr_ctx* c) {
    CU(c, cudaGetLastError());
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
// row and goes to the final agreement); else *sum = the sum of the payloads.
bool peer_sum(ctmr_ctx* c, PeerLocal& local, uint64_t mine, uint64_t* sum) {
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
    return true;
}

// 63 bits of FNV-1a over (now, salt_len, salt): equal on every rank that passes the same arguments
uint64_t args_hash(int64_t now, const uint8_t* salt, uint32_t salt_len) {
    uint64_t h = 14695981039346656037ull;
    const auto put = [&](uint8_t v) { h = (h ^ v) * 1099511628211ull; };
    for (int i = 0; i < 8; ++i) put((uint8_t)((uint64_t)now >> (8 * i)));
    put((uint8_t)salt_len);
    for (uint32_t j = 0; j < salt_len; ++j) put(salt[j]);
    return h >> 1;
}

// this rank's part of the collective call
int revoked_cascade_peer(ctmr_ctx* c, const ctmr_crl_batch* b, int64_t now, const uint8_t* salt, uint32_t salt_len, ctmr_cascade_out* out) {
    const char* call = "ctmr_revoked_cascade: ";
    CU(c, cudaSetDevice(c->device));
    if (out) out->bytes = 0;
    const uint32_t W = c->st.peer.world;
    const uint64_t IW = c->st.max_issuers / 32 + 1;  // words of the seen bitmap, and of the bad one after it
    std::vector<uint32_t> issuer;
    uint64_t n_chunks = 0;
    // everything that can fail before any work, allocations included, so that it travels in agreement 1
    int rc = salt_len > kMaxSalt ? fail(c, CTMR_E_INVALID, "ctmr_revoked_cascade: salt_len > 32")
             : salt_len && !salt ? fail(c, CTMR_E_INVALID, "ctmr_revoked_cascade: NULL salt")
                                 : CTMR_OK;
    if (rc == CTMR_OK) rc = crl_peer_prepare(c, b, out, call, issuer, &n_chunks);
    if (rc == CTMR_OK) rc = cascade_ensure(c, 0, 2 * IW, false);
    if (rc == CTMR_OK) rc = refresh_digests(c);
    uint64_t row[kMaxWorld] = {};
    rc = peer_agree(c, rc, n_chunks, row, call, "collective call failed");  // agreement 1
    if (rc) return rc;
    {  // now and salt define R, S and every bit: they must be rank 0's
        uint64_t hrow[kMaxWorld] = {};
        const uint64_t h = args_hash(now, salt, salt_len);
        rc = peer_mailbox(c, h, hrow);
        if (rc == CTMR_OK) rc = ctmr_check_device(c, nullptr);  // a barrier that timed out
        if (rc) return rc;
        if (h != hrow[0]) return fail(c, CTMR_E_INVALID, "ctmr_revoked_cascade: now_unix_sec or salt differs from rank 0's");
        for (uint32_t r = 1; r < W; ++r)
            if (hrow[r] != hrow[0])
                return fail(c, CTMR_E_PEER_FAILED, "ctmr_revoked_cascade: rank " + std::to_string(r) + "'s now_unix_sec or salt differs from rank 0's");
    }
    const uint32_t n_issuers = (uint32_t)c->digests.size();
    ctmr_ctx* m[1] = {c};
    Cascade cs{m, 1, nullptr};
    cs.p.n_issuers = n_issuers;
    cs.p.salt_len = salt_len;
    cs.p.now = now;
    for (uint32_t j = 0; j < salt_len; ++j) cs.p.salt[j >> 2] |= (uint32_t)salt[j] << (8 * (j & 3));
    cs.p.one = 1;
    cs.ml.assign(1, MemberLevel{});
    CascadeState* s = c->cascade.get();
    PeerLocal local;  // this rank's error after agreement 1: it does no more work, and the ranks stop at the next exchange
    // the slot bits cleared, the registry's digests
    local.fail(c, [&]() -> int {
        CU(c, cudaMemsetAsync(s->revoked, 0, s->slot_words * 4, c->stream));
        if (n_issuers) CU(c, cudaMemcpyAsync(s->dig, c->digests.data(), (size_t)n_issuers * 32, cudaMemcpyHostToDevice, c->stream));
        return CTMR_OK;
    }());
    // mark: every round's union set against the own shard
    std::vector<uint8_t> crl_status(b->n_crls, CTMR_CRL_OK);
    const bool going = crl_peer_each_set(c, b, issuer, row, [&](const CrlSetSlot* set, uint64_t mask) -> int {
        cascade_mark_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->st.table, c->st.table_mask + 1, now, set, mask, s->revoked);
        return launched(c);
    }, crl_status, local);

    std::vector<uint8_t> img;
    uint32_t n_covered = 0, level = 0;
    const auto build = [&]() {  // every return is one that all ranks take together, to the final agreement
        if (!going) return;
        // coverage: seen and bad bitmaps of the rank's own CRLs, OR-reduced over the ranks
        std::vector<uint32_t> sb(2 * IW, 0);
        for (uint64_t k = 0; k < b->n_crls; ++k) {
            const uint32_t i = issuer[k];
            if (i >= n_issuers) continue;
            sb[i >> 5] |= 1u << (i & 31);
            if (crl_status[k] != CTMR_CRL_OK) sb[IW + (i >> 5)] |= 1u << (i & 31);
        }
        if (!local.code) local.fail(c, [&]() -> int {
            CU(c, cudaMemcpyAsync(s->bits, sb.data(), sb.size() * 4, cudaMemcpyHostToDevice, c->stream));
            return CTMR_OK;
        }());
        local.fail(c, cascade_peer_or(c, s->bits, 2 * IW, !local.code));
        std::vector<uint32_t> covered(n_issuers / 32 + 1, 0);
        uint64_t nr = 0, ns = 0;
        if (!local.code) local.fail(c, [&]() -> int {
            CU(c, cudaMemcpyAsync(sb.data(), s->bits, sb.size() * 4, cudaMemcpyDeviceToHost, c->stream));
            CU(c, cudaStreamSynchronize(c->stream));
            for (uint32_t i = 0; i < n_issuers; ++i)
                if ((sb[i >> 5] & ~sb[IW + (i >> 5)]) >> (i & 31) & 1u) {
                    covered[i >> 5] |= 1u << (i & 31);
                    ++n_covered;
                }
            CU(c, cudaMemcpyAsync(s->covered, covered.data(), covered.size() * 4, cudaMemcpyHostToDevice, c->stream));
            int rc2 = cs.split(0, s->list_cap, &nr, &ns);  // R and S of the own shard
            if (rc2 == CTMR_OK && nr > s->list_cap) rc2 = cs.split(0, nr, &nr, &ns);
            return rc2;
        }());
        if (!peer_sum(c, local, nr, &cs.R) || !peer_sum(c, local, ns, &cs.S)) return;
        cs.ml[0].n_inc = nr;
        cs.ml[0].n_exc = ns;

        // the levels, each merged on every rank and read back into the image behind the header
        img = {2, 0, 0, (uint8_t)salt_len};
        img.insert(img.end(), salt, salt + salt_len);
        uint64_t n_inc = cs.R;
        for (;;) {
            if (++level > kMaxLevels) {
                local.fail(c, fail(c, CTMR_E_INVALID, "ctmr_revoked_cascade: more than 255 levels; build with another salt"));
                return;
            }
            const double p = level == 1 ? (cs.R == 0 || cs.S == 0 ? 0.5 : std::min(0.5, (double)cs.R / (std::sqrt(2.0) * (double)cs.S))) : 0.5;
            const LevelSize ls = level_size(n_inc, p);
            if (ls.m >= 4294967296.0) {
                local.fail(c, fail(c, CTMR_E_BATCH_TOO_LARGE, "ctmr_revoked_cascade: level " + std::to_string(level) + " needs 2^32 bits or more"));
                return;
            }
            const uint32_t mbits = (uint32_t)ls.m;
            const uint64_t words = ((uint64_t)mbits + 31) / 32;
            cs.p.level = level;
            cs.p.k = ls.k;
            cs.p.m = mbits;
            if (!local.code) local.fail(c, cs.insert(words));  // the own include list into partial bits
            local.fail(c, cascade_peer_or(c, s->bits, words, !local.code));
            uint64_t f = 0;
            if (!local.code) {
                int rc2 = cs.test(0, &f);
                if (rc2 == CTMR_OK && f > s->list_cap) {  // level 1 only: F_1 outgrew the lists, which hold R; make room and run again
                    rc2 = cs.split(0, f, &nr, &ns);
                    if (rc2 == CTMR_OK) rc2 = cs.test(0, &f);
                }
                local.fail(c, rc2);
            }
            uint64_t F = 0;
            if (!peer_sum(c, local, f, &F)) return;
            const uint64_t nbytes = ((uint64_t)mbits + 7) / 8;
            const size_t at = img.size();
            img.resize(at + 10 + nbytes);
            img[at] = 2;
            std::memcpy(&img[at + 1], &mbits, 4);
            std::memcpy(&img[at + 5], &ls.k, 4);
            img[at + 9] = (uint8_t)level;
            if (!local.code) local.fail(c, [&]() -> int {
                CU(c, cudaMemcpyAsync(&img[at + 10], s->bits, nbytes, cudaMemcpyDeviceToHost, c->stream));
                CU(c, cudaStreamSynchronize(c->stream));
                return CTMR_OK;
            }());
            if (F == 0) return;
            MemberLevel& l = cs.ml[0];  // I_{l+1} = F_l, E_{l+1} = I_l
            const uint32_t free_list = l.exc == kNoList ? 3 - l.inc - l.out : l.exc;
            l.exc = l.inc;
            l.n_exc = l.n_inc;
            l.inc = l.out;
            l.n_inc = f;
            l.out = free_list;
            n_inc = F;
        }
    };
    build();

    const cudaStream_t drain[] = {c->crl->copy_stream, c->stream};
    drain_streams(c, drain, 2);  // no upload may read the caller's data after the call
    if (!local.code && (rc = ctmr_check_device(c, nullptr))) local.fail(c, rc);  // a barrier that timed out
    if (local.code) c->err = local.err;
    const bool short_cap = img.size() > out->cap || !out->buf;
    rc = peer_agree(c, local.code, short_cap ? 1 : 0, row, call, "collective call failed");  // the final agreement
    if (rc) return rc;
    out->bytes = img.size();
    for (uint32_t r = 0; r < W; ++r)
        if (row[r])
            return fail(c, CTMR_E_BATCH_TOO_LARGE, r == c->px.rank ? "ctmr_revoked_cascade: cap " + std::to_string(out->cap) + " < " + std::to_string(img.size()) + " bytes"
                                                                  : "ctmr_revoked_cascade: rank " + std::to_string(r) + "'s cap < " + std::to_string(img.size()) + " bytes");
    std::memcpy(out->buf, img.data(), img.size());
    if (out->crl_status) std::memcpy(out->crl_status, crl_status.data(), crl_status.size());
    out->issuers = n_covered;
    out->levels = level;
    out->revoked = cs.R;
    out->valid = cs.S;
    return CTMR_OK;
}

}  // namespace

extern "C" {

int ctmr_revoked_cascade(ctmr_ctx* c, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* salt, uint32_t salt_len,
                         ctmr_cascade_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group) return fail(c, CTMR_E_INVALID, "ctmr_revoked_cascade: a member of a group; use ctmr_group_revoked_cascade");
    if (peer_call(c)) return revoked_cascade_peer(c, batch, now_unix_sec, salt, salt_len, out);
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

}  // extern "C"
