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

__device__ __host__ __forceinline__ uint64_t key_hash(const uint32_t (&b)[12]) {
    uint64_t h = 0x9E3779B97F4A7C15ull;
#pragma unroll
    for (int i = 0; i < 12; i += 2) h = mix64(h ^ (((uint64_t)b[i + 1] << 32) | b[i])) + 0x632BE59BD9B4E019ull * (i + 1);
    return h;
}

// ------------------------------------------------------------------------------------------------
// table epochs.  ctmr_reset_device empties the known-certificate, pair and string-identity tables by advancing the ctx's
// epoch (DeviceState::epoch, 1..kEpochMax) instead of clearing gigabytes: a slot is live only if its state is non-zero AND
// it carries the current epoch; every other slot is empty, and an insert may claim it.  Zeroed memory is empty at any epoch.
//   KnownSlot.tag:                  epoch in bits 48..63 | key_hash bits 2..47 | state in bits 0..1
//   PairSlot.pad / MetaSlot.pad:    epoch in bits 48..63 | state in bits 0..1
// The state is pending (claimed, being written) or ready (published by a release store).  Snapshots and checkpoints hold
// slots in their canonical form, which carries no epoch: a KnownSlot tag of the full key_hash with the ready state, a zero
// pad, and all-zero bytes for an empty slot.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kEpochMax = 0xFFFFu;
constexpr uint32_t kSlotPending = 1u, kSlotReady = 2u;
constexpr uint64_t kTagHashBits = 0x0000FFFFFFFFFFFCull;

// the state word of a slot: `h` = the key's key_hash for a KnownSlot tag, 0 for a pad word
__device__ __host__ __forceinline__ uint64_t slot_word(uint32_t epoch, uint32_t state, uint64_t h = 0) {
    return ((uint64_t)epoch << 48) | (h & kTagHashBits) | state;
}
// the state of a slot at `epoch`: 0 (empty) unless the word carries that epoch
__device__ __host__ __forceinline__ uint32_t slot_state(uint64_t w, uint32_t epoch) {
    return (uint32_t)(w >> 48) == epoch ? (uint32_t)w & 3u : 0u;
}
__device__ __host__ __forceinline__ bool tag_hash_eq(uint64_t tag, uint64_t h) { return ((tag ^ h) & kTagHashBits) == 0ull; }
// the canonical tag of a ready key (what the tables held before epochs, and what snapshots and checkpoints store)
__device__ __host__ __forceinline__ uint64_t canonical_tag(const uint32_t (&body)[12]) { return (key_hash(body) & ~3ull) | kSlotReady; }
// the epoch after a reset; 0: the epoch wraps, the tables must be zeroed and the next epoch is 1
__device__ __host__ __forceinline__ uint32_t next_epoch(uint32_t epoch) { return epoch < kEpochMax ? epoch + 1u : 0u; }

// a live slot in canonical form; `live` = false: all zero
__device__ __host__ __forceinline__ KnownSlot canonical_slot(const KnownSlot& s, bool live) {
    KnownSlot o{};
    if (live) {
        o = s;
        o.tag = canonical_tag(s.body);
    }
    return o;
}
__device__ __host__ __forceinline__ PairSlot canonical_slot(const PairSlot& s, bool live) {
    PairSlot o{};
    if (live) {
        o = s;
        o.pad = 0ull;
    }
    return o;
}
__device__ __host__ __forceinline__ MetaSlot canonical_slot(const MetaSlot& s, bool live) {
    MetaSlot o{};
    if (live) {
        o = s;
        o.pad = 0ull;
    }
    return o;
}
__device__ __host__ __forceinline__ uint64_t state_word(const KnownSlot& s) { return s.tag; }
__device__ __host__ __forceinline__ uint64_t state_word(const PairSlot& s) { return s.pad; }
__device__ __host__ __forceinline__ uint64_t state_word(const MetaSlot& s) { return s.pad; }
__device__ __host__ __forceinline__ unsigned long long& state_word(KnownSlot& s) { return s.tag; }
__device__ __host__ __forceinline__ unsigned long long& state_word(PairSlot& s) { return s.pad; }
__device__ __host__ __forceinline__ unsigned long long& state_word(MetaSlot& s) { return s.pad; }
// a state word moved from epoch `from` to epoch `to` (ranks agreeing on one epoch at ctmr_peer_attach): a slot live at
// `from` is live at `to`, any other word is left as it is (a ctx's slots never carry an epoch above its own)
__device__ __host__ __forceinline__ uint64_t restamp_word(uint64_t w, uint32_t from, uint32_t to) {
    return slot_state(w, from) == kSlotReady ? slot_word(to, kSlotReady, w) : w;
}
// a canonical slot as live at `epoch` (a snapshot's slots on their way in): ready if canonical form calls it live, else empty
__device__ __host__ __forceinline__ void stamp_slot(KnownSlot& s, uint32_t epoch) {
    s.tag = (s.tag & 3ull) == kSlotReady ? slot_word(epoch, kSlotReady, s.tag) : 0ull;
}
__device__ __host__ __forceinline__ void stamp_slot(PairSlot& s, uint32_t epoch) { s.pad = s.key != 0ull ? slot_word(epoch, kSlotReady) : 0ull; }
__device__ __host__ __forceinline__ void stamp_slot(MetaSlot& s, uint32_t epoch) { s.pad = s.h1 != 0ull ? slot_word(epoch, kSlotReady) : 0ull; }

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

// The probe rule of the three tables (known-certificate, (issuer, hour) pair, string identity), all open addressing with
// linear probing (DESIGN.md §3 "Probe rule"):
//   finding  a find-or-insert or a lookup walks from the home slot until it meets its key or a slot empty at the current
//            epoch.  Its only bound is the table size, so it finds every record the table holds, however far from home.
//   placing  a NEW record of the batch path or of a preload goes at most kProbeLimit slots past its home slot; the empty
//            slot the walk ended at lies further, or there is none: the table's *_TABLE_FULL.
//   again    a record the state already holds, placed again (eviction's reinsert, the resize rehash, a checkpoint load),
//            may go anywhere in the table (limit = the table's mask): the order of those inserts decides how far each
//            record lands, so no survivor is lost to a limit and a state always fits tables of its own size.
constexpr uint64_t kProbeLimit = 4096;

// Find-or-insert of a 48-byte key body; lowest global index wins through an atomic max on ~index.  A slot empty at
// `epoch` (zero, or left by an earlier epoch) is claimed by a CAS from the tag observed to pending; the claimer writes
// the key bytes and inv_first, then publishes them by a release store of the ready tag (a slot of an earlier epoch may
// hold a larger ~index, so inv_first is stored, not max'ed, and before the release).  Equal keys act only once they see
// ready.  `limit`: how far past its home a new key may be placed (kProbeLimit, or the table's mask for a key placed
// again).  Returns the slot, or 0xFFFFFFFF when the table is full (error flag set).  Shared by K_insert and by K_map's
// fused insert; SYS = system scope (only the string-identity table is touched across GPUs).
template <bool SYS>
__device__ __forceinline__ uint32_t known_insert(KnownSlot* __restrict__ table, uint64_t table_mask, uint32_t epoch, int* error_flag,
                                                 const uint32_t (&body)[12], unsigned long long inv_idx, uint64_t limit = kProbeLimit) {
    const uint64_t h = key_hash(body);
    const unsigned long long tag_ready = slot_word(epoch, kSlotReady, h), tag_pending = slot_word(epoch, kSlotPending, h);
    uint64_t pos = (h >> 7) & table_mask;
    uint64_t probes = 0;  // distance of pos from the home slot
    for (;;) {
        KnownSlot* sl = table + pos;
        unsigned long long t = ld_volatile_u64(&sl->tag);  // relaxed: an acquire here would invalidate the SM's L1 per probe
        if (slot_state(t, epoch) == 0u) {
            if (probes > limit) break;  // the key is not in the table, and its place would lie past the limit
            const unsigned long long seen = t;
            t = tab_cas<SYS>(&sl->tag, seen, tag_pending);
            if (t != seen) continue;  // another thread claimed the slot first: look at it again
            uint4* bp = reinterpret_cast<uint4*>(sl->body);
            bp[0] = make_uint4(body[0], body[1], body[2], body[3]);
            bp[1] = make_uint4(body[4], body[5], body[6], body[7]);
            bp[2] = make_uint4(body[8], body[9], body[10], body[11]);
            sl->inv_first = inv_idx;
            tab_store_release<SYS>(&sl->tag, tag_ready);
            return (uint32_t)pos;
        }
        if (tag_hash_eq(t, h)) {
            // the key bytes are read only after an acquire of the ready tag: a relaxed read of ready does not order them,
            // and a slot of the last epoch may hold an equal key
            do t = tab_load_acquire<SYS>(&sl->tag);  // pending: another thread is publishing this slot
            while (slot_state(t, epoch) == kSlotPending);
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
        if (++probes > table_mask) break;  // every slot holds another key
    }
    atomicExch(error_flag, CTMR_E_TABLE_FULL);
    return 0xFFFFFFFFu;
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
