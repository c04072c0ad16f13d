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

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Shape of the streaming map (K_map): the best measured before the port (DESIGN.md §3, K_map).
struct StreamCfg {
    static constexpr int kWarps = 8;       // warps per CTA, one certificate per lane
    static constexpr int kChunk = 128;     // record bytes staged per lane and step
    static constexpr int kCtasPerSm = 2;   // resident CTAs per SM of the persistent grid
    static constexpr int kOverlap = 48;  // >= kWalkNeed, multiple of 16
    // Lane slots are kSlot bytes apart and every lane reads the same word of its own slot, so the stride
    // decides the bank pattern: 16-byte granules (cp.async) allow at best 8 distinct bank groups; an odd
    // number of granules per slot reaches that (4-way worst case), an even one collapses to 2 groups (16-way).
    static constexpr int kSlotRaw = kOverlap + kChunk + 16;
    static constexpr int kSlot = kSlotRaw + (((kSlotRaw / 16) % 2 == 0) ? 16 : 0);
    static constexpr int kWarpBytes = 2 * 32 * kSlot;
    static constexpr int kBlocksPerChunk = kChunk / 64;
    // +16: the walker's word-wise header read may touch the word after the last staged byte
    static constexpr size_t kSmem = (size_t)kWarps * kWarpBytes + 16;
};

struct GlobalBytes {
    const uint8_t* d;
    __device__ __forceinline__ uint32_t operator()(uint32_t x) const { return __ldg(d + x); }
};


}  // namespace ctmr
