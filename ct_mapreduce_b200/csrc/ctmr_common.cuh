// ctmr_common.cuh -- device helpers shared by the map and reduce translation units: PTX wrappers
// (cp.async), the known-certificate table probe, streaming geometry.
#pragma once
#include "ctmr_device.cuh"
#include "ctmr_kernels.cuh"

namespace ctmr {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint32_t warp_max_u32(uint32_t v) { return __reduce_max_sync(0xffffffffu, v); }

// ------------------------------------------------------------------------------------------------
// known-certificate table
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* p) {
    return *reinterpret_cast<const volatile unsigned long long*>(p);
}

__device__ __forceinline__ uint64_t key_hash(const uint32_t (&b)[12]) {
    uint64_t h = 0x9E3779B97F4A7C15ull;
#pragma unroll
    for (int i = 0; i < 12; i += 2) h = mix64(h ^ (((uint64_t)b[i + 1] << 32) | b[i])) + 0x632BE59BD9B4E019ull * (i + 1);
    return h;
}

// Scope of the table atomics: device scope on a single GPU, system scope once peers' tables are addressed
// over NVLink (the atomic is performed at the owner's L2 either way; the scope decides what it is ordered with).
template <bool SYS>
__device__ __forceinline__ unsigned long long tab_cas(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
    return SYS ? atomicCAS_system(p, cmp, v) : atomicCAS(p, cmp, v);
}
template <bool SYS>
__device__ __forceinline__ void tab_max(unsigned long long* p, unsigned long long v) {
    if (SYS) asm volatile("red.relaxed.sys.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
    else asm volatile("red.relaxed.gpu.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
template <bool SYS>
__device__ __forceinline__ void tab_add(unsigned long long* p, unsigned long long v) {
    if (SYS) asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
    else asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
template <bool SYS>
__device__ __forceinline__ void tab_store_release(unsigned long long* p, unsigned long long v) {
    if (SYS) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
    else asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
template <bool SYS>
__device__ __forceinline__ unsigned long long tab_load_acquire(const unsigned long long* p) {
    unsigned long long v;
    if (SYS) asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    else asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// 16 bytes of a slot another SM (or, SYS, another GPU) has written: from L2 / the owner's memory, never a stale L1 line
template <bool SYS>
__device__ __forceinline__ uint4 ld_slot_u4(const uint4* p) { return SYS ? __ldcv(p) : __ldcg(p); }
__device__ __forceinline__ uint4 ld_cv_u4(const uint4* p) { return __ldcv(p); }

// Find-or-insert of a 48-byte key body; lowest global index wins through an atomic max on ~index.  An empty slot is
// claimed by an optimistic CAS (the tag read is the CAS's return value), the key bytes are published by a release
// store of the ready tag.  Returns the slot, or 0xFFFFFFFF when the table is full (error flag set).  Shared by
// K_insert and by K_map's fused insert; SYS = system scope (only the string-identity table is touched across GPUs).
template <bool SYS>
__device__ __forceinline__ uint32_t known_insert(KnownSlot* __restrict__ table, uint64_t table_mask, int* error_flag,
                                                 const uint32_t (&body)[12], unsigned long long inv_idx) {
    const uint64_t h = key_hash(body);
    const unsigned long long tag_ready = (h & ~3ull) | 2ull, tag_pending = (h & ~3ull) | 1ull;
    uint64_t pos = (h >> 7) & table_mask;
    uint32_t probes = 0;
    for (;;) {
        KnownSlot* sl = table + pos;
        unsigned long long t = tab_cas<SYS>(&sl->tag, 0ull, tag_pending);
        if (t == 0ull) {  // claimed: publish the key bytes, then flip to ready
            uint4* bp = reinterpret_cast<uint4*>(sl->body);
            bp[0] = make_uint4(body[0], body[1], body[2], body[3]);
            bp[1] = make_uint4(body[4], body[5], body[6], body[7]);
            bp[2] = make_uint4(body[8], body[9], body[10], body[11]);
            tab_store_release<SYS>(&sl->tag, tag_ready);
            tab_max<SYS>(&sl->inv_first, inv_idx);
            return (uint32_t)pos;
        }
        if ((t & ~3ull) == (h & ~3ull)) {
            while ((t & 3ull) == 1ull) t = tab_load_acquire<SYS>(&sl->tag);  // another thread is publishing this slot
            const uint4* bp = reinterpret_cast<const uint4*>(sl->body);
            const uint4 b0 = ld_slot_u4<SYS>(bp), b1 = ld_slot_u4<SYS>(bp + 1), b2 = ld_slot_u4<SYS>(bp + 2);
            const bool same = b0.x == body[0] && b0.y == body[1] && b0.z == body[2] && b0.w == body[3] && b1.x == body[4] &&
                              b1.y == body[5] && b1.z == body[6] && b1.w == body[7] && b2.x == body[8] && b2.y == body[9] &&
                              b2.z == body[10] && b2.w == body[11];
            if (same) {
                tab_max<SYS>(&sl->inv_first, inv_idx);
                return (uint32_t)pos;
            }
        }
        pos = (pos + 1) & table_mask;
        if (++probes > 4096u) {  // table effectively full
            atomicExch(error_flag, CTMR_E_TABLE_FULL);
            return 0xFFFFFFFFu;
        }
    }
}

// a CRL join's (issuer, serial) pair exactly as words 1..11 of a KnownSlot body: issuer, then {serial_len, serial[39]}
// little-endian (ctmr_crl.cu's set, probed by ctmr_cascade.cu too)
__device__ __host__ __forceinline__ uint32_t pair_hash(const uint32_t (&w)[11]) {
    uint64_t h = 0x9E3779B97F4A7C15ull;
#pragma unroll
    for (int i = 0; i < 11; ++i) h = mix64(h ^ ((uint64_t)w[i] << (i & 1 ? 32 : 0))) + (uint64_t)i;
    return (uint32_t)(h >> 32);
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Shape of the streaming map (K_map, DESIGN.md §3).  Each lane stages its record in a private ring of kRing bytes
// (two chunks) plus a 16-byte mirror of the ring's first granule, so that the hash's 17-word reads never wrap.
struct StreamCfg {
    static constexpr int kWarps = 8;       // warps per CTA, one certificate per lane
    static constexpr int kChunk = 128;     // record bytes staged per lane and step
    static constexpr int kCtasPerSm = 3;   // resident CTAs per SM of the persistent grid (24 warps)
    static constexpr int kRing = 2 * kChunk;
    // Lane rings are kLaneBytes apart and every lane reads the same word of its own ring, so the stride
    // decides the bank pattern: 16-byte granules (cp.async) allow at best 8 distinct bank groups; an odd
    // number of granules per lane reaches that (4-way worst case), an even one collapses to 2 groups (16-way).
    static constexpr int kLaneBytes = kRing + 16;
    static constexpr int kWarpBytes = 32 * kLaneBytes;
    static constexpr int kBlocksPerChunk = kChunk / 64;
    static constexpr int kGranulesPerChunk = kChunk / 16;
    static constexpr size_t kSmem = (size_t)kWarps * kWarpBytes;
};
static_assert((StreamCfg::kLaneBytes / 16) % 2 == 1, "odd number of 16-byte granules per lane");
static_assert(StreamCfg::kCtasPerSm * (StreamCfg::kSmem + 1024) <= 228 * 1024, "kCtasPerSm CTAs fit one SM's shared memory");

// K_map's copy schedule.  Source granule y is the 16 bytes at 16*y from the record's 16-byte aligned base, i.e. record
// bytes [16y - m, 16y + 16 - m) for a record m bytes past that base; it lives at ring offset 16*y mod kRing.  Chunk k
// (record bytes [k*kChunk, (k+1)*kChunk)) spans source granules [8k, 8k + 8], the ninth only when m != 0.  When
// m != 0 and k > 0 chunk k-1 has already brought granule 8k, so every chunk but the first copies at most 8 granules.
// `yend` is one past the record's last source granule.  [y0, ymid) and [ymid, y1) are the two parts of the copy
// (ring_step says why there are two); neither crosses the ring's end.
struct RingCopy {
    uint32_t y0, ymid, y1;
};
__host__ __device__ __forceinline__ RingCopy ring_chunk_copy(uint32_t k, uint32_t m, uint32_t yend) {
    constexpr uint32_t G = StreamCfg::kGranulesPerChunk;
    const uint32_t lo = G * k + (k != 0u && m != 0u ? 1u : 0u), next = G * (k + 1u);
    const uint32_t y1 = yend < next + (m != 0u ? 1u : 0u) ? yend : next + (m != 0u ? 1u : 0u);
    const uint32_t ymid = y1 < next ? y1 : next;
    return RingCopy{lo < ymid ? lo : ymid, ymid, y1};
}

// One step of K_map's loop, entered when chunk c has landed (chunk c-1 is still in the other half of the ring): walk
// chunk c (the walker may look back up to kWalkNeed bytes into chunk c-1), copy chunk c+1 into chunk c-1's half, hash
// chunk c.  The copy overlaps the hash.  Its ninth granule (m != 0) lies kRing bytes past chunk c's first granule and
// shares that granule's ring slot, which the hash is still reading: that one granule is copied after the hash.
template <class Walk, class Copy, class Hash>
__host__ __device__ __forceinline__ void ring_step(uint32_t c, uint32_t m, uint32_t yend, Walk&& walk, Copy&& copy, Hash&& hash) {
    walk();
    const RingCopy r = ring_chunk_copy(c + 1u, m, yend);
    copy(r.y0, r.ymid);
    hash();
    copy(r.ymid, r.y1);
}

struct GlobalBytes {
    const uint8_t* d;
    __device__ __forceinline__ uint32_t operator()(uint32_t x) const { return __ldg(d + x); }
};


}  // namespace ctmr
