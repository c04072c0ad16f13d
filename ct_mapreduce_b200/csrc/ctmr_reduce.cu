// ctmr_reduce.cu -- the reduce half: known-certificate table insert / resolve, (issuer, hour) first-seen,
// IssuerMetadata string identities, issuer preparation, set cardinality, the owner / source passes of the multi-GPU key
// exchange, the issuer registry, the cross-process barrier and the histogram merge, and the rehash of ctmr_resize.
#include <algorithm>
#include <type_traits>

#include "ctmr_common.cuh"

namespace ctmr {

// ------------------------------------------------------------------------------------------------
// K_insert / K_resolve / K_pairs.  Every table operation is LOCAL: a rank only ever inserts, resolves and counts
// keys of sets it owns -- its own entries' (K_map's fused insert) and the records other ranks appended to its inbox.
// Ownership is disjoint, so one sum over the ranks' histograms (ctmr_peer_allreduce_histogram_device /
// ctmr_group_issuer_counts) is exact.  The same three bodies serve a plain key array (m on the host) and the inbox
// regions of an exchange parity (blockIdx.y = source rank, record count read from device memory).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void insert_one(const DeviceState& st, const ctmr_key* __restrict__ keys, uint64_t j, uint32_t* __restrict__ slot_of) {
    const uint4* kr = reinterpret_cast<const uint4*>(keys + j);
    const uint4 q0 = kr[0], q1 = kr[1], q2 = kr[2], q3 = kr[3];
    if (q3.z == 0u) {  // not a Store-reaching entry
        slot_of[j] = 0xFFFFFFFFu;
        return;
    }
    const unsigned long long inv_idx = ~(((unsigned long long)q0.y << 32) | q0.x);
    const uint32_t body[12] = {q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y};
    slot_of[j] = known_insert<false>(st.table, st.table_mask, st.epoch, st.error_flag, body, inv_idx);
}

__global__ void __launch_bounds__(256) insert_kernel(DeviceState st, const ctmr_key* __restrict__ keys, uint64_t m,
                                                     uint32_t* __restrict__ slot_of) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) insert_one(st, keys, j, slot_of);
}

// Find-or-insert of an (issuer, hour) key.  The pad word carries the slot's epoch and state (ctmr_common.cuh): the same key
// recurs after every reset, so a key word left by an earlier epoch cannot tell whether the slot is live.  The claimer
// writes key, inv_first and count = 0 while the slot is pending; equal keys act (max, add) only once they see it ready.
// `limit` and the probe rule as for known_insert (ctmr_common.cuh).
template <bool SYS>
__device__ __forceinline__ uint32_t pair_insert(PairSlot* __restrict__ pairs, uint64_t pair_mask, uint32_t epoch, int* error_flag,
                                                unsigned long long pk, unsigned long long inv_idx, uint64_t limit = kProbeLimit) {
    uint64_t pos = mix64(pk) & pair_mask;
    for (uint64_t probes = 0; probes <= pair_mask; ++probes) {
        PairSlot* sl = pairs + pos;
        unsigned long long w = ld_volatile_u64(&sl->pad);
        while (slot_state(w, epoch) == 0u && probes <= limit) {
            const unsigned long long seen = w;
            w = tab_cas<SYS>(&sl->pad, seen, slot_word(epoch, kSlotPending));
            if (w != seen) continue;  // another thread claimed the slot first
            sl->key = pk;
            sl->inv_first = inv_idx;
            sl->count = 0ull;
            tab_store_release<SYS>(&sl->pad, slot_word(epoch, kSlotReady));
            return (uint32_t)pos;
        }
        if (slot_state(w, epoch) == 0u) break;  // the key is not in the table, and its place would lie past the limit
        // the key is read only after an acquire of the ready word (a relaxed read of ready does not order it, and the slot
        // may hold the same key from the last epoch); pending: another thread is publishing the slot
        do w = tab_load_acquire<SYS>(&sl->pad);
        while (slot_state(w, epoch) == kSlotPending);
        if (ld_volatile_u64(&sl->key) == pk) {
            tab_max<SYS>(&sl->inv_first, inv_idx);
            return (uint32_t)pos;
        }
        pos = (pos + 1) & pair_mask;
    }
    atomicExch(error_flag, CTMR_E_PAIR_TABLE_FULL);
    return 0xFFFFFFFFu;
}

// `in` lanes hold record j; every lane of the warp takes part in the aggregation
__device__ __forceinline__ void resolve_one(const DeviceState& st, const ctmr_key* __restrict__ keys, uint64_t j, bool in,
                                            const uint32_t* __restrict__ slot_of, uint32_t* __restrict__ pair_slot,
                                            uint8_t* __restrict__ was_unknown) {
    bool unknown = false;
    uint32_t issuer = 0;
    int32_t hour = 0;
    unsigned long long inv_idx = 0;
    if (in) {
        const uint32_t s = slot_of[j];
        if (s != 0xFFFFFFFFu) {
            const uint4 q0 = reinterpret_cast<const uint4*>(keys + j)[0];
            inv_idx = ~(((unsigned long long)q0.y << 32) | q0.x);
            hour = (int32_t)q0.z;
            issuer = q0.w;
            // I am the first sighting of this key: every insert of a lower index happened before this pass
            unknown = ld_volatile_u64(&st.table[s].inv_first) == inv_idx;
        }
        was_unknown[j] = unknown ? 1 : 0;
    }
    const uint32_t umask = __ballot_sync(0xffffffffu, unknown);
    uint32_t ps = 0xFFFFFFFFu;
    if (unknown) {
        // per-issuer unique count: one atomic per distinct issuer per warp
        const uint32_t peers = __match_any_sync(umask, issuer);
        if ((threadIdx.x & 31u) == (uint32_t)__ffs(peers) - 1u && issuer < st.max_issuers)
            atomicAdd(st.issuer_counts + issuer, (unsigned long long)__popc(peers));
        // the set's (issuer, exp_hour) slot: first-seen index + cardinality
        const unsigned long long pk = ((((unsigned long long)issuer) << 32) | (uint32_t)hour) + 1ull;
        const uint32_t same_set = __match_any_sync(umask, pk);
        ps = pair_insert<false>(st.pairs, st.pair_mask, st.epoch, st.error_flag, pk, inv_idx);
        if (ps != 0xFFFFFFFFu && (threadIdx.x & 31u) == (uint32_t)__ffs(same_set) - 1u)
            tab_add<false>(&st.pairs[ps].count, (unsigned long long)__popc(same_set));
    }
    if (in) pair_slot[j] = ps;
}

__global__ void __launch_bounds__(256) resolve_kernel(DeviceState st, const ctmr_key* __restrict__ keys, uint64_t m,
                                                      const uint32_t* __restrict__ slot_of, uint32_t* __restrict__ pair_slot,
                                                      uint8_t* __restrict__ was_unknown) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    resolve_one(st, keys, j, j < m, slot_of, pair_slot, was_unknown);
}

__device__ __forceinline__ void pairs_one(const DeviceState& st, const ctmr_key* __restrict__ keys, uint64_t j,
                                          const uint32_t* __restrict__ pair_slot, const uint8_t* __restrict__ was_unknown,
                                          uint8_t* __restrict__ first_issuer_hour) {
    uint8_t first = 0;
    const uint32_t ps = pair_slot[j];
    if (was_unknown[j] && ps != 0xFFFFFFFFu) {
        const uint4 q0 = reinterpret_cast<const uint4*>(keys + j)[0];
        const unsigned long long inv_idx = ~(((unsigned long long)q0.y << 32) | q0.x);
        first = ld_volatile_u64(&st.pairs[ps].inv_first) == inv_idx ? 1 : 0;
    }
    first_issuer_hour[j] = first;
}

__global__ void __launch_bounds__(256) pairs_kernel(DeviceState st, const ctmr_key* __restrict__ keys, uint64_t m,
                                                    const uint32_t* __restrict__ pair_slot,
                                                    const uint8_t* __restrict__ was_unknown,
                                                    uint8_t* __restrict__ first_issuer_hour) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) pairs_one(st, keys, j, pair_slot, was_unknown, first_issuer_hour);
}

// ---- the owner's side of the exchange: the same passes over the inbox regions of one parity ------------------
__global__ void __launch_bounds__(256) inbox_insert_kernel(DeviceState st, PeerExchange px, uint32_t parity, uint32_t* __restrict__ in_slot) {
    const uint32_t src = blockIdx.y;
    if (src == px.rank) return;
    const uint64_t region = ((uint64_t)parity * px.world + src) * px.X;
    const uint64_t m = min((unsigned long long)px.X, ld_volatile_u64(px.counts[px.rank] + parity * px.world + src));
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) insert_one(st, px.inbox[px.rank] + region, j, in_slot + region);
}
__global__ void __launch_bounds__(256) inbox_resolve_kernel(DeviceState st, PeerExchange px, uint32_t parity,
                                                            const uint32_t* __restrict__ in_slot, uint32_t* __restrict__ in_pair) {
    const uint32_t src = blockIdx.y;
    if (src == px.rank) return;
    const uint64_t region = ((uint64_t)parity * px.world + src) * px.X;
    const uint64_t m = min((unsigned long long)px.X, ld_volatile_u64(px.counts[px.rank] + parity * px.world + src));
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if ((uint64_t)blockIdx.x * blockDim.x >= m) return;  // whole block past the end (uniform: the warp collectives below stay convergent)
    resolve_one(st, px.inbox[px.rank] + region, j, j < m, in_slot + region, in_pair + region, px.out_wu[px.rank] + region);
}
__global__ void __launch_bounds__(256) inbox_pairs_kernel(DeviceState st, PeerExchange px, uint32_t parity, const uint32_t* __restrict__ in_pair) {
    const uint32_t src = blockIdx.y;
    if (src == px.rank) return;
    const uint64_t region = ((uint64_t)parity * px.world + src) * px.X;
    const uint64_t m = min((unsigned long long)px.X, ld_volatile_u64(px.counts[px.rank] + parity * px.world + src));
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) pairs_one(st, px.inbox[px.rank] + region, j, in_pair + region, px.out_wu[px.rank] + region, px.out_first[px.rank] + region);
}

// ---- the source's side: region sizes to the owners, result bits back by position -------------------------------
__global__ void publish_counts_kernel(PeerExchange px, uint32_t parity, const unsigned long long* __restrict__ cursor) {
    const uint32_t t = threadIdx.x;
    if (t < px.world && t != px.rank) px.counts[t][parity * px.world + px.rank] = cursor[t];  // one 8-byte peer store per owner
}
__global__ void __launch_bounds__(256) pull_bits_kernel(PeerExchange px, uint32_t parity, const unsigned long long* __restrict__ cursor,
                                                        const uint32_t* __restrict__ rev, uint8_t* __restrict__ was_unknown,
                                                        uint8_t* __restrict__ first_issuer_hour) {
    const uint32_t owner = blockIdx.y;
    if (owner == px.rank) return;
    const uint64_t m = min((unsigned long long)px.X, cursor[owner]);
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint64_t at = ((uint64_t)parity * px.world + px.rank) * px.X + i;  // my region in the owner's outbox: contiguous reads
    const uint32_t e = rev[(uint64_t)owner * px.X + i];
    if (was_unknown) was_unknown[e] = __ldcv(px.out_wu[owner] + at);
    if (first_issuer_hour) first_issuer_hour[e] = __ldcv(px.out_first[owner] + at);
}

// ------------------------------------------------------------------------------------------------
// K_meta: IssuerMetadata's string reducers (storage/issuermetadata.go:92-138).  For every NEW
// certificate the reference looks up the issuer DN and each CRL distribution point in per-issuer
// memo sets and only on a miss talks to Redis.  Here the (issuer, bytes) identity of the raw issuer
// Name and of the raw cRLDistributionPoints value is inserted into a device table (two independent
// 64-bit hashes; lowest index wins), so the host formats / parses those strings only for the
// first-seen candidates.  Raw-bytes identity is finer than the reference's string identity, so the
// candidate set is a superset of the reference's misses: nothing new can be hidden.
// ------------------------------------------------------------------------------------------------
__device__ inline void hash_bytes(const uint8_t* __restrict__ p, uint32_t len, uint64_t seed, uint64_t& h1, uint64_t& h2) {
    uint64_t a = seed ^ 0x9E3779B97F4A7C15ull, b = seed * 0xD6E8FEB86659FD93ull + 0x2545F4914F6CDD1Dull;
    for (uint32_t i = 0; i < len; i += 8) {
        uint64_t v = 0;
        const uint32_t n = len - i < 8u ? len - i : 8u;
        for (uint32_t k = 0; k < n; ++k) v |= (uint64_t)__ldg(p + i + k) << (8 * k);
        a = mix64(a ^ v) + 0x632BE59BD9B4E019ull;
        b = mix64(b + v * 0xFF51AFD7ED558CCDull) ^ (v >> 17);
    }
    h1 = mix64(a ^ len) | 1ull;
    h2 = mix64(b + len) | 1ull;
}

// owner of a string identity: by its first hash (any rank may meet any issuer's strings)
__device__ __forceinline__ uint32_t meta_owner(uint64_t h1, uint32_t world) { return world > 1u ? (uint32_t)((h1 >> 40) % world) : 0u; }

// The pad word carries the slot's epoch and state, as in pair_insert: the claimer writes h1, h2 and inv_first while the
// slot is pending.  A cross-GPU insert (SYS) stamps the inserting rank's epoch, which is the owner's: every reset is
// collective (ctmr_reset_device).  `limit` and the probe rule as for known_insert (ctmr_common.cuh).
template <bool SYS>
__device__ inline uint32_t meta_insert_at(MetaSlot* __restrict__ meta, uint64_t meta_mask, uint32_t epoch, int* error_flag, uint64_t h1,
                                          uint64_t h2, unsigned long long inv_idx, uint64_t limit = kProbeLimit) {
    uint64_t pos = (h1 >> 5) & meta_mask;
    for (uint64_t probes = 0; probes <= meta_mask; ++probes) {
        MetaSlot* sl = meta + pos;
        unsigned long long w = ld_volatile_u64(&sl->pad);
        while (slot_state(w, epoch) == 0u && probes <= limit) {
            const unsigned long long seen = w;
            w = tab_cas<SYS>(&sl->pad, seen, slot_word(epoch, kSlotPending));
            if (w != seen) continue;  // another thread claimed the slot first
            sl->h1 = h1;
            sl->h2 = h2;
            sl->inv_first = inv_idx;
            tab_store_release<SYS>(&sl->pad, slot_word(epoch, kSlotReady));
            return (uint32_t)pos;
        }
        if (slot_state(w, epoch) == 0u) break;  // the identity is not in the table, and its place would lie past the limit
        // the key is read only after an acquire of the ready word (a relaxed read of ready does not order it, and the slot
        // may hold the same key from the last epoch); pending: another thread is publishing the slot
        do w = tab_load_acquire<SYS>(&sl->pad);
        while (slot_state(w, epoch) == kSlotPending);
        if (ld_volatile_u64(&sl->h1) == h1 && ld_volatile_u64(&sl->h2) == h2) {
            tab_max<SYS>(&sl->inv_first, inv_idx);
            return (uint32_t)pos;
        }
        pos = (pos + 1) & meta_mask;
    }
    atomicExch(error_flag, CTMR_E_META_TABLE_FULL);
    return 0xFFFFFFFFu;
}

// returns (owner << 28) | slot (the table has at most 2^26 slots), 0xFFFFFFFF on failure
__device__ inline uint32_t meta_insert(const DeviceState& st, uint64_t h1, uint64_t h2, unsigned long long inv_idx) {
    if (st.peer.world <= 1u) return meta_insert_at<false>(st.meta, st.meta_mask, st.epoch, st.error_flag, h1, h2, inv_idx);
    const uint32_t owner = meta_owner(h1, st.peer.world);
    const uint32_t pos = meta_insert_at<true>(st.peer.meta[owner], st.meta_mask, st.epoch, st.error_flag, h1, h2, inv_idx);
    return pos == 0xFFFFFFFFu ? pos : ((owner << 28) | pos);
}
__device__ __forceinline__ unsigned long long meta_first(const DeviceState& st, uint32_t packed) {
    return ld_volatile_u64(&st.peer.meta[packed >> 28][packed & 0x0FFFFFFFu].inv_first);
}

__global__ void __launch_bounds__(256) meta_insert_kernel(DeviceState st, const uint8_t* __restrict__ blob,
                                                          const uint64_t* __restrict__ offsets, const ctmr_key* __restrict__ keys,
                                                          uint64_t m, const uint8_t* __restrict__ was_unknown,
                                                          const uint32_t* __restrict__ name_off, const uint32_t* __restrict__ name_len,
                                                          const uint32_t* __restrict__ crl_off, const uint32_t* __restrict__ crl_len,
                                                          uint32_t* __restrict__ meta_slots) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    uint32_t s_dn = 0xFFFFFFFFu, s_crl = 0xFFFFFFFFu;
    if (was_unknown[j]) {
        const uint4 q0 = reinterpret_cast<const uint4*>(keys + j)[0];
        const unsigned long long inv_idx = ~(((unsigned long long)q0.y << 32) | q0.x);
        const uint8_t* d = blob + offsets[j];
        uint64_t h1, h2;
        if (name_len[j]) {
            hash_bytes(d + name_off[j], name_len[j], ((uint64_t)q0.w << 8) | 1u, h1, h2);
            s_dn = meta_insert(st, h1, h2, inv_idx);
        }
        if (crl_len[j]) {
            hash_bytes(d + crl_off[j], crl_len[j], ((uint64_t)q0.w << 8) | 2u, h1, h2);
            s_crl = meta_insert(st, h1, h2, inv_idx);
        }
    }
    meta_slots[2 * j] = s_dn;
    meta_slots[2 * j + 1] = s_crl;
}

__global__ void __launch_bounds__(256) meta_resolve_kernel(DeviceState st, const ctmr_key* __restrict__ keys, uint64_t m,
                                                           const uint32_t* __restrict__ meta_slots, uint8_t* __restrict__ first_dn,
                                                           uint8_t* __restrict__ first_crl) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint4 q0 = reinterpret_cast<const uint4*>(keys + j)[0];
    const unsigned long long inv_idx = ~(((unsigned long long)q0.y << 32) | q0.x);
    const uint32_t a = meta_slots[2 * j], b = meta_slots[2 * j + 1];
    if (first_dn) first_dn[j] = (a != 0xFFFFFFFFu && meta_first(st, a) == inv_idx) ? 1 : 0;
    if (first_crl) first_crl[j] = (b != 0xFFFFFFFFu && meta_first(st, b) == inv_idx) ? 1 : 0;
}

static inline unsigned blocks_for(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

// string identities in two halves: in a group a sync separates every rank's inserts from the read-back
cudaError_t launch_meta_insert(const DeviceState& st, const uint8_t* blob, const uint64_t* offsets, const ctmr_key* keys, uint64_t m,
                               const uint8_t* was_unknown, const uint32_t* name_off, const uint32_t* name_len, const uint32_t* crl_off,
                               const uint32_t* crl_len, uint32_t* meta_slots, cudaStream_t s) {
    if (!m) return cudaSuccess;
    meta_insert_kernel<<<blocks_for(m, 256), 256, 0, s>>>(st, blob, offsets, keys, m, was_unknown, name_off, name_len, crl_off,
                                                          crl_len, meta_slots);
    return cudaGetLastError();
}
cudaError_t launch_meta_resolve(const DeviceState& st, const ctmr_key* keys, uint64_t m, const uint32_t* meta_slots, uint8_t* first_dn,
                                uint8_t* first_crl, cudaStream_t s) {
    if (!m) return cudaSuccess;
    meta_resolve_kernel<<<blocks_for(m, 256), 256, 0, s>>>(st, keys, m, meta_slots, first_dn, first_crl);
    return cudaGetLastError();
}

cudaError_t launch_insert(const DeviceState& st, const ctmr_key* keys, uint64_t m, uint32_t* slot_of, cudaStream_t s) {
    if (!m) return cudaSuccess;
    insert_kernel<<<blocks_for(m, 256), 256, 0, s>>>(st, keys, m, slot_of);
    return cudaGetLastError();
}
cudaError_t launch_resolve(const DeviceState& st, const ctmr_key* keys, uint64_t m, const uint32_t* slot_of,
                           uint32_t* pair_slot, uint8_t* was_unknown, cudaStream_t s) {
    if (!m) return cudaSuccess;
    // 128 threads: the block fits beside K_map's three resident CTAs (ctmr_map.cu, kLenThreads), so the pass runs under
    // the next round's K_map instead of waiting for its CTAs to retire
    resolve_kernel<<<blocks_for(m, 128), 128, 0, s>>>(st, keys, m, slot_of, pair_slot, was_unknown);
    return cudaGetLastError();
}
cudaError_t launch_resolve_pairs(const DeviceState& st, const ctmr_key* keys, uint64_t m, const uint32_t* pair_slot,
                                 const uint8_t* was_unknown, uint8_t* first_issuer_hour, cudaStream_t s) {
    if (!m) return cudaSuccess;
    pairs_kernel<<<blocks_for(m, 256), 256, 0, s>>>(st, keys, m, pair_slot, was_unknown, first_issuer_hour);
    return cudaGetLastError();
}

cudaError_t launch_inbox_insert(const DeviceState& st, const PeerExchange& px, uint32_t parity, uint64_t max_per_region, uint32_t* in_slot,
                                cudaStream_t s) {
    if (px.world <= 1 || !max_per_region) return cudaSuccess;
    inbox_insert_kernel<<<dim3(blocks_for(max_per_region, 256), px.world), 256, 0, s>>>(st, px, parity, in_slot);
    return cudaGetLastError();
}
cudaError_t launch_inbox_resolve(const DeviceState& st, const PeerExchange& px, uint32_t parity, uint64_t max_per_region,
                                 const uint32_t* in_slot, uint32_t* in_pair, cudaStream_t s) {
    if (px.world <= 1 || !max_per_region) return cudaSuccess;
    inbox_resolve_kernel<<<dim3(blocks_for(max_per_region, 256), px.world), 256, 0, s>>>(st, px, parity, in_slot, in_pair);
    return cudaGetLastError();
}
cudaError_t launch_inbox_pairs(const DeviceState& st, const PeerExchange& px, uint32_t parity, uint64_t max_per_region,
                               const uint32_t* in_pair, cudaStream_t s) {
    if (px.world <= 1 || !max_per_region) return cudaSuccess;
    inbox_pairs_kernel<<<dim3(blocks_for(max_per_region, 256), px.world), 256, 0, s>>>(st, px, parity, in_pair);
    return cudaGetLastError();
}
cudaError_t launch_publish_counts(const PeerExchange& px, uint32_t parity, const unsigned long long* cursor, cudaStream_t s) {
    if (px.world <= 1) return cudaSuccess;
    publish_counts_kernel<<<1, 32, 0, s>>>(px, parity, cursor);
    return cudaGetLastError();
}
cudaError_t launch_pull_bits(const PeerExchange& px, uint32_t parity, const unsigned long long* cursor, const uint32_t* rev,
                             uint64_t max_per_region, uint8_t* was_unknown, uint8_t* first_issuer_hour, cudaStream_t s) {
    if (px.world <= 1 || !max_per_region) return cudaSuccess;
    pull_bits_kernel<<<dim3(blocks_for(max_per_region, 256), px.world), 256, 0, s>>>(px, parity, cursor, rev, was_unknown, first_issuer_hour);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// issuers: x509.ParseCertificate(Chain[0]) + SHA-256(RawSubjectPublicKeyInfo)
// ------------------------------------------------------------------------------------------------
__global__ void issuer_prepare_kernel(const uint8_t* __restrict__ blob, const uint64_t* __restrict__ offsets, uint32_t n,
                                      uint8_t* __restrict__ digests, uint8_t* __restrict__ ok) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint64_t off = offsets[k], end = offsets[k + 1];
    ParsedCert pc;
    bool good = end >= off && end - off <= 0x7fffffffull && parse_cert(blob + off, (uint32_t)(end - off), pc);
    uint32_t h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (good) sha256_global(blob + off + pc.spki_off, pc.spki_len, h);
    for (int i = 0; i < 8; ++i) {
        digests[k * 32 + 4 * i + 0] = (uint8_t)(h[i] >> 24);
        digests[k * 32 + 4 * i + 1] = (uint8_t)(h[i] >> 16);
        digests[k * 32 + 4 * i + 2] = (uint8_t)(h[i] >> 8);
        digests[k * 32 + 4 * i + 3] = (uint8_t)h[i];
    }
    ok[k] = good ? 1 : 0;
}

cudaError_t launch_issuer_prepare(const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint8_t* digests, uint8_t* ok,
                                  cudaStream_t s) {
    if (!n) return cudaSuccess;
    issuer_prepare_kernel<<<blocks_for(n, 64), 64, 0, s>>>(blob, offsets, n, digests, ok);
    return cudaGetLastError();
}

// SetCardinality("serials::<expDate>::<issuer>") (storage/knowncertificates.go:57-63): the set's (issuer, hour) slot at
// its owner carries the count, maintained by K_resolve and by the TTL eviction -- one probe, not a table scan
// (the reference's consumer asks once per set, cmd/storage-statistics/storage-statistics.go:44-53).
__global__ void cardinality_kernel(DeviceState st, int32_t hour, uint32_t issuer, unsigned long long* out) {
    const unsigned long long pk = ((((unsigned long long)issuer) << 32) | (uint32_t)hour) + 1ull;
    const PairSlot* pairs = st.peer.pairs[st.peer.world > 1u ? key_owner(hour, issuer, st.peer.world) : 0u];
    uint64_t pos = mix64(pk) & st.pair_mask;
    unsigned long long v = 0;
    for (uint64_t probes = 0; probes <= st.pair_mask; ++probes) {  // to the key or an empty slot (the probe rule, ctmr_common.cuh)
        if (slot_state(ld_volatile_u64(&pairs[pos].pad), st.epoch) == 0u) break;
        if (ld_volatile_u64(&pairs[pos].key) == pk) {
            v = ld_volatile_u64(&pairs[pos].count);
            break;
        }
        pos = (pos + 1) & st.pair_mask;
    }
    *out = v;
}

__global__ void __launch_bounds__(256) table_count_kernel(DeviceState st, unsigned long long* out) {
    unsigned int local = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= st.table_mask; i += (uint64_t)gridDim.x * blockDim.x)
        local += slot_state(st.table[i].tag, st.epoch) == kSlotReady;
    local = __reduce_add_sync(0xffffffffu, local);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(out, (unsigned long long)local);
}

// ---- TTL eviction (SURVEY §8(f)-4): sets whose EXPIREAT time has passed vanish ---------------------------
// pass 1: count expired / surviving ready slots, take the expired ones out of the per-issuer histogram
__global__ void __launch_bounds__(256) evict_count_kernel(DeviceState st, int64_t now_sec, unsigned long long* counters /* [2]: live, expired */) {
    unsigned int live = 0, dead = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= st.table_mask; i += (uint64_t)gridDim.x * blockDim.x) {
        const KnownSlot& sl = st.table[i];
        if (slot_state(sl.tag, st.epoch) != kSlotReady) continue;
        const int64_t hour = (int32_t)sl.body[0];
        if (hour * 3600 <= now_sec) {
            ++dead;
            if (sl.body[1] < st.max_issuers) atomicAdd(st.issuer_counts + sl.body[1], ~0ull);  // -1
        } else {
            ++live;
        }
    }
    live = __reduce_add_sync(0xffffffffu, live);
    dead = __reduce_add_sync(0xffffffffu, dead);
    if ((threadIdx.x & 31) == 0) {
        if (live) atomicAdd(counters, (unsigned long long)live);
        if (dead) atomicAdd(counters + 1, (unsigned long long)dead);
    }
}

// pass 2: the live slots of a table, compacted in slot order (ctmr_evict_expired: the surviving keys; a checkpoint: the
// ready keys, the pairs and the string identities).  Tile b (kCompactTile slots from t0 * kCompactTile on) is one CTA:
// with counts set, counts[b] = its live slots; otherwise it writes them from keep[base[t0 + b] - base[t0]] on, in slot
// order (a ballot per warp and a scan over the CTA's eight warps per row of 256 slots).  Two runs over the same state
// write the same bytes.
// since > 0 (a delta checkpoint) also asks for a first-seen index at or above `since` (inv_first = ~index)
__device__ __forceinline__ bool slot_live(const KnownSlot& sl, uint32_t epoch, int64_t now_sec, uint64_t since) {
    return slot_state(sl.tag, epoch) == kSlotReady && (int64_t)(int32_t)sl.body[0] * 3600 > now_sec && ~sl.inv_first >= since;
}
__device__ __forceinline__ bool slot_live(const PairSlot& sl, uint32_t epoch, int64_t, uint64_t since) {
    return slot_state(sl.pad, epoch) == kSlotReady && ~sl.inv_first >= since;
}
__device__ __forceinline__ bool slot_live(const MetaSlot& sl, uint32_t epoch, int64_t, uint64_t since) {
    return slot_state(sl.pad, epoch) == kSlotReady && ~sl.inv_first >= since;
}

template <class Slot>
__global__ void __launch_bounds__(256) evict_compact_kernel(const Slot* __restrict__ table, uint64_t n_slots, uint32_t epoch, int64_t now_sec, uint64_t t0,
                                                            const unsigned long long* __restrict__ base, Slot* __restrict__ keep,
                                                            uint32_t* __restrict__ counts, uint64_t since) {
    __shared__ uint32_t warp_n[8];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint64_t tile = t0 + blockIdx.x;
    uint64_t out = counts ? 0ull : base[tile] - base[t0];
    uint32_t total = 0;
    for (uint32_t row = 0; row < kCompactTile / 256u; ++row) {
        const uint64_t i = tile * kCompactTile + row * 256u + threadIdx.x;
        const bool live = i < n_slots && slot_live(table[i], epoch, now_sec, since);
        const uint32_t ball = __ballot_sync(0xffffffffu, live);
        if (lane == 0) warp_n[warp] = __popc(ball);
        __syncthreads();
        uint32_t before = 0, row_n = 0;
#pragma unroll
        for (uint32_t w = 0; w < 8u; ++w) {
            before += w < warp ? warp_n[w] : 0u;
            row_n += warp_n[w];
        }
        if (live && !counts) keep[out + before + __popc(ball & ((1u << lane) - 1u))] = canonical_slot(table[i], true);
        out += row_n;
        total += row_n;
        __syncthreads();  // warp_n is rewritten by the next row
    }
    if (counts && threadIdx.x == 0) counts[blockIdx.x] = total;
}

// pass 3 (after the table has been cleared), and a checkpoint's records on their way in: linear probing leaves no holes
// only if every record is inserted again.  Records placed again, bounded by the table size alone (the probe rule,
// ctmr_common.cuh): this order may place a survivor further from home than the batch path did.  The records are
// canonical (no epoch): a ready one has state 2 in its tag.  A record whose owner under this rank's world is another rank
// is skipped (eviction: a rank only ever holds keys it owns).  Every index a record carries is checked before it is used: an
// issuer >= n_issuers, a serial longer than CTMR_MAX_SERIAL or a slot that is not ready raises CTMR_E_INVALID.  count:
// the inserted keys go into the per-issuer histogram (a checkpoint carries no histogram).
__global__ void __launch_bounds__(256) evict_reinsert_kernel(DeviceState st, const KnownSlot* __restrict__ keep, uint64_t n,
                                                             uint32_t n_issuers, bool count) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const KnownSlot sl = keep[i];
    if ((sl.tag & 3ull) != 2ull || sl.body[1] >= n_issuers || (sl.body[2] & 0xFFu) > CTMR_MAX_SERIAL) {
        atomicExch(st.error_flag, CTMR_E_INVALID);
        return;
    }
    if (st.peer.world > 1u && key_owner((int32_t)sl.body[0], sl.body[1], st.peer.world) != st.peer.rank) return;
    uint32_t body[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) body[k] = sl.body[k];
    if (known_insert<false>(st.table, st.table_mask, st.epoch, st.error_flag, body, sl.inv_first, st.table_mask) != 0xFFFFFFFFu && count)
        atomicAdd(st.issuer_counts + sl.body[1], 1ull);
}

// a checkpoint's (issuer, hour) records: the owner's pair slot again, with its first-seen index and its cardinality
__global__ void __launch_bounds__(256) ckpt_pairs_kernel(DeviceState st, const PairSlot* __restrict__ rec, uint64_t n, uint32_t n_issuers) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const PairSlot p = rec[i];
    if (p.key == 0ull || ((p.key - 1ull) >> 32) >= n_issuers) {
        atomicExch(st.error_flag, CTMR_E_INVALID);
        return;
    }
    const uint32_t issuer = (uint32_t)((p.key - 1ull) >> 32);
    const int32_t hour = (int32_t)(uint32_t)(p.key - 1ull);
    if (st.peer.world > 1u && key_owner(hour, issuer, st.peer.world) != st.peer.rank) return;
    const uint32_t ps = pair_insert<false>(st.pairs, st.pair_mask, st.epoch, st.error_flag, p.key, p.inv_first, st.pair_mask);
    if (ps != 0xFFFFFFFFu && p.count) tab_add<false>(&st.pairs[ps].count, p.count);
}

// a checkpoint's string identities: the owner's slot again, with its first-seen index
__global__ void __launch_bounds__(256) ckpt_meta_kernel(DeviceState st, const MetaSlot* __restrict__ rec, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const MetaSlot m = rec[i];
    if (m.h1 == 0ull || m.h2 == 0ull) {
        atomicExch(st.error_flag, CTMR_E_INVALID);
        return;
    }
    if (meta_owner(m.h1, st.peer.world) != (st.peer.world > 1u ? st.peer.rank : 0u)) return;
    meta_insert_at<false>(st.meta, st.meta_mask, st.epoch, st.error_flag, m.h1, m.h2, m.inv_first, st.meta_mask);
}

// A delta checkpoint's apply: every (issuer, hour) count and the per-issuer histogram again, from the ready keys alone (the
// delta carries no old pair, whose count changed).  Pass 1 zeroes the pair counts; pass 2 adds each key to its issuer and
// to its set's slot, found with the cardinality lookup's probe (a key and its set have one owner, so the slot is local).
// A key whose set is missing raises CTMR_E_INVALID.  One atomic per distinct issuer / set per warp.
__global__ void __launch_bounds__(256) recount_zero_kernel(PairSlot* __restrict__ pairs, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) pairs[i].count = 0ull;
}
__global__ void __launch_bounds__(256) recount_kernel(DeviceState st) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t end = (st.table_mask + 1 + stride - 1) / stride * stride;  // every lane runs the same trips: the warp votes stay whole
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
        bool live = false;
        uint32_t issuer = 0;
        unsigned long long pk = 0;
        if (i <= st.table_mask) {
            const KnownSlot& sl = st.table[i];
            live = slot_state(sl.tag, st.epoch) == kSlotReady && sl.body[1] < st.max_issuers;
            issuer = sl.body[1];
            pk = ((((unsigned long long)issuer) << 32) | sl.body[0]) + 1ull;
        }
        const uint32_t lmask = __ballot_sync(0xffffffffu, live);
        if (!live) continue;
        const uint32_t lane = threadIdx.x & 31u;
        const uint32_t same_issuer = __match_any_sync(lmask, issuer);
        if (lane == (uint32_t)__ffs(same_issuer) - 1u) atomicAdd(st.issuer_counts + issuer, (unsigned long long)__popc(same_issuer));
        const uint32_t same_set = __match_any_sync(lmask, pk);
        if (lane != (uint32_t)__ffs(same_set) - 1u) continue;
        uint64_t pos = mix64(pk) & st.pair_mask;
        bool found = false;
        for (uint64_t probes = 0; probes <= st.pair_mask; ++probes) {  // to the key or an empty slot (the probe rule, ctmr_common.cuh)
            const PairSlot& p = st.pairs[pos];
            if (slot_state(p.pad, st.epoch) == 0u) break;
            if (p.key == pk) {
                atomicAdd(&st.pairs[pos].count, (unsigned long long)__popc(same_set));
                found = true;
                break;
            }
            pos = (pos + 1) & st.pair_mask;
        }
        if (!found) atomicExch(st.error_flag, CTMR_E_INVALID);
    }
}

cudaError_t launch_recount(const DeviceState& st, int sm_count, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(st.issuer_counts, 0, st.max_issuers * sizeof(unsigned long long), s);
    if (e != cudaSuccess) return e;
    recount_zero_kernel<<<sm_count * 4, 256, 0, s>>>(st.pairs, st.pair_mask + 1);
    recount_kernel<<<sm_count * 8, 256, 0, s>>>(st);
    return cudaGetLastError();
}

cudaError_t launch_evict_count(const DeviceState& st, int64_t now_sec, unsigned long long* counters, int sm_count, cudaStream_t s) {
    evict_count_kernel<<<sm_count * 8, 256, 0, s>>>(st, now_sec, counters);
    return cudaGetLastError();
}
template <class Slot>
cudaError_t launch_evict_compact(const Slot* table, uint64_t n_slots, uint32_t epoch, int64_t now_sec, uint64_t t0, uint64_t t1,
                                 const unsigned long long* base, Slot* keep, uint32_t* counts, cudaStream_t s, uint64_t since) {
    if (t1 <= t0) return cudaSuccess;
    evict_compact_kernel<Slot><<<(unsigned)(t1 - t0), 256, 0, s>>>(table, n_slots, epoch, now_sec, t0, base, keep, counts, since);
    return cudaGetLastError();
}
template cudaError_t launch_evict_compact<KnownSlot>(const KnownSlot*, uint64_t, uint32_t, int64_t, uint64_t, uint64_t,
                                                     const unsigned long long*, KnownSlot*, uint32_t*, cudaStream_t, uint64_t);
template cudaError_t launch_evict_compact<PairSlot>(const PairSlot*, uint64_t, uint32_t, int64_t, uint64_t, uint64_t,
                                                    const unsigned long long*, PairSlot*, uint32_t*, cudaStream_t, uint64_t);
template cudaError_t launch_evict_compact<MetaSlot>(const MetaSlot*, uint64_t, uint32_t, int64_t, uint64_t, uint64_t,
                                                    const unsigned long long*, MetaSlot*, uint32_t*, cudaStream_t, uint64_t);

template <class Slot>
__global__ void __launch_bounds__(256) stamp_kernel(Slot* __restrict__ table, uint64_t n_slots, uint32_t epoch) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slots; i += (uint64_t)gridDim.x * blockDim.x)
        stamp_slot(table[i], epoch);
}
template <class Slot>
__global__ void __launch_bounds__(256) restamp_kernel(Slot* __restrict__ table, uint64_t n_slots, uint32_t from, uint32_t to) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slots; i += (uint64_t)gridDim.x * blockDim.x)
        state_word(table[i]) = restamp_word(state_word(table[i]), from, to);
}
cudaError_t launch_restamp_tables(const DeviceState& st, uint32_t from, uint32_t to, int sm_count, cudaStream_t s) {
    restamp_kernel<<<sm_count * 8, 256, 0, s>>>(st.table, st.table_mask + 1, from, to);
    restamp_kernel<<<sm_count * 4, 256, 0, s>>>(st.pairs, st.pair_mask + 1, from, to);
    restamp_kernel<<<sm_count * 4, 256, 0, s>>>(st.meta, st.meta_mask + 1, from, to);
    return cudaGetLastError();
}
cudaError_t launch_stamp_tables(const DeviceState& st, int sm_count, cudaStream_t s) {
    stamp_kernel<<<sm_count * 8, 256, 0, s>>>(st.table, st.table_mask + 1, st.epoch);
    stamp_kernel<<<sm_count * 4, 256, 0, s>>>(st.pairs, st.pair_mask + 1, st.epoch);
    stamp_kernel<<<sm_count * 4, 256, 0, s>>>(st.meta, st.meta_mask + 1, st.epoch);
    return cudaGetLastError();
}
cudaError_t launch_evict_reinsert(const DeviceState& st, const KnownSlot* keep, uint64_t n, uint32_t n_issuers, bool count, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    evict_reinsert_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(st, keep, n, n_issuers, count);
    return cudaGetLastError();
}
cudaError_t launch_ckpt_pairs(const DeviceState& st, const PairSlot* rec, uint64_t n, uint32_t n_issuers, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    ckpt_pairs_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(st, rec, n, n_issuers);
    return cudaGetLastError();
}
cudaError_t launch_ckpt_meta(const DeviceState& st, const MetaSlot* rec, uint64_t n, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    ckpt_meta_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(st, rec, n);
    return cudaGetLastError();
}

cudaError_t launch_table_count(const DeviceState& st, unsigned long long* out, int sm_count, cudaStream_t s) {
    table_count_kernel<<<sm_count * 8, 256, 0, s>>>(st, out);
    return cudaGetLastError();
}

// ---- resize (ctmr_resize): the slots ready at the current epoch into tables of another size ----------------------------
// One slot in 16-byte streaming loads: the old table is read once and never again.
template <class Slot>
__device__ __forceinline__ Slot ld_slot_once(const Slot* p) {
    static_assert(sizeof(Slot) % 16 == 0, "slots are whole 16-byte vectors");
    union {
        uint4 v[sizeof(Slot) / 16];
        Slot s;
    } u;
#pragma unroll
    for (int k = 0; k < (int)(sizeof(Slot) / 16); ++k) u.v[k] = __ldcs(reinterpret_cast<const uint4*>(p) + k);
    return u.s;
}

// A record into the new tables with the insert of the batch path, bounded by the new table's size alone (a record placed
// again, ctmr_common.cuh); returns the issuer whose histogram entry the record
// adds to (a known key that went in), else 0xFFFFFFFF.  A pair keeps its first-seen index and its count (an evicted set's
// 0 included); a string identity its first-seen index.  Every record is unique in its table, so the claimer of a slot is
// the only writer of its count.
__device__ __forceinline__ uint32_t rehash_one(const DeviceState& to, const KnownSlot& sl) {
    uint32_t body[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) body[k] = sl.body[k];
    return known_insert<false>(to.table, to.table_mask, to.epoch, to.error_flag, body, sl.inv_first, to.table_mask) != 0xFFFFFFFFu ? sl.body[1]
                                                                                                                      : 0xFFFFFFFFu;
}
__device__ __forceinline__ uint32_t rehash_one(const DeviceState& to, const PairSlot& p) {
    const uint32_t ps = pair_insert<false>(to.pairs, to.pair_mask, to.epoch, to.error_flag, p.key, p.inv_first, to.pair_mask);
    if (ps != 0xFFFFFFFFu) to.pairs[ps].count = p.count;
    return 0xFFFFFFFFu;
}
__device__ __forceinline__ uint32_t rehash_one(const DeviceState& to, const MetaSlot& m) {
    meta_insert_at<false>(to.meta, to.meta_mask, to.epoch, to.error_flag, m.h1, m.h2, m.inv_first, to.meta_mask);
    return 0xFFFFFFFFu;
}

// Grid-stride over the old table in warp-wide steps (every lane of a warp takes part in each step's histogram vote).  The
// known keys rebuild to.issuer_counts, one atomic per distinct issuer of a warp's step, as a checkpoint load rebuilds it.
template <class Slot>
__global__ void __launch_bounds__(256) rehash_kernel(const Slot* __restrict__ old, uint64_t n_old, uint32_t epoch, DeviceState to) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n_old; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint32_t issuer = 0xFFFFFFFFu;
        if (i < n_old) {
            const Slot sl = ld_slot_once(old + i);
            if (slot_state(state_word(sl), epoch) == kSlotReady) issuer = rehash_one(to, sl);
        }
        if constexpr (std::is_same<Slot, KnownSlot>::value) {
            const bool counted = issuer < to.max_issuers;
            const uint32_t mask = __ballot_sync(0xffffffffu, counted);
            if (counted) {
                const uint32_t peers = __match_any_sync(mask, issuer);
                if (lane == (uint32_t)__ffs(peers) - 1u) atomicAdd(to.issuer_counts + issuer, (unsigned long long)__popc(peers));
            }
        }
    }
}

template <class Slot>
__global__ void __launch_bounds__(256) live_count_kernel(const Slot* __restrict__ table, uint64_t n, uint32_t epoch, unsigned long long* out) {
    unsigned int local = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        local += slot_state(state_word(table[i]), epoch) == kSlotReady;
    local = __reduce_add_sync(0xffffffffu, local);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(out, (unsigned long long)local);
}

template <class Slot>
cudaError_t launch_rehash(const Slot* old, uint64_t n_old, uint32_t epoch, const DeviceState& to, int sm_count, cudaStream_t s) {
    const uint64_t blocks = std::min<uint64_t>((n_old + 255) / 256, (uint64_t)sm_count * 8);
    if (blocks) rehash_kernel<Slot><<<(unsigned)blocks, 256, 0, s>>>(old, n_old, epoch, to);
    return cudaGetLastError();
}
template <class Slot>
cudaError_t launch_live_count(const Slot* table, uint64_t n, uint32_t epoch, unsigned long long* out, int sm_count, cudaStream_t s) {
    const uint64_t blocks = std::min<uint64_t>((n + 255) / 256, (uint64_t)sm_count * 8);
    if (blocks) live_count_kernel<Slot><<<(unsigned)blocks, 256, 0, s>>>(table, n, epoch, out);
    return cudaGetLastError();
}
template cudaError_t launch_rehash<KnownSlot>(const KnownSlot*, uint64_t, uint32_t, const DeviceState&, int, cudaStream_t);
template cudaError_t launch_rehash<PairSlot>(const PairSlot*, uint64_t, uint32_t, const DeviceState&, int, cudaStream_t);
template cudaError_t launch_rehash<MetaSlot>(const MetaSlot*, uint64_t, uint32_t, const DeviceState&, int, cudaStream_t);
template cudaError_t launch_live_count<KnownSlot>(const KnownSlot*, uint64_t, uint32_t, unsigned long long*, int, cudaStream_t);
template cudaError_t launch_live_count<PairSlot>(const PairSlot*, uint64_t, uint32_t, unsigned long long*, int, cudaStream_t);
template cudaError_t launch_live_count<MetaSlot>(const MetaSlot*, uint64_t, uint32_t, unsigned long long*, int, cudaStream_t);

cudaError_t launch_cardinality(const DeviceState& st, int32_t hour, uint32_t issuer, unsigned long long* out,
                               cudaStream_t s) {
    cardinality_kernel<<<1, 1, 0, s>>>(st, hour, issuer, out);
    return cudaGetLastError();
}

// TTL eviction, pair side: an expired set's cardinality is 0 again; the first-seen memo (process memory in the
// reference, storage/issuermetadata.go:95-108) stays.
__global__ void __launch_bounds__(256) evict_pairs_kernel(DeviceState st, int64_t now_sec) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= st.pair_mask; i += (uint64_t)gridDim.x * blockDim.x) {
        if (slot_state(st.pairs[i].pad, st.epoch) != kSlotReady) continue;
        const unsigned long long k = st.pairs[i].key;
        const int64_t hour = (int32_t)(uint32_t)(k - 1ull);
        if (hour * 3600 <= now_sec) st.pairs[i].count = 0ull;
    }
}
cudaError_t launch_evict_pairs(const DeviceState& st, int64_t now_sec, int sm_count, cudaStream_t s) {
    evict_pairs_kernel<<<sm_count * 4, 256, 0, s>>>(st, now_sec);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Issuer registry: Issuer.ID digest -> dense index, find-or-insert in rank 0's memory (system scope).
// ------------------------------------------------------------------------------------------------
__global__ void issuer_registry_kernel(IssuerRegistry reg, const uint8_t* __restrict__ digests, const uint8_t* __restrict__ ok,
                                       uint32_t n, uint32_t* __restrict__ idx_out, int* error_flag) {
  // one thread, the call's digests in order: within a process indices follow the order of first appearance
  for (uint32_t k = 0; k < n; ++k) {
    if (ok && !ok[k]) {
        idx_out[k] = CTMR_ISSUER_BAD;
        continue;
    }
    uint32_t w[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
        w[i] = (uint32_t)digests[32 * k + 4 * i] | ((uint32_t)digests[32 * k + 4 * i + 1] << 8) |
               ((uint32_t)digests[32 * k + 4 * i + 2] << 16) | ((uint32_t)digests[32 * k + 4 * i + 3] << 24);
    uint64_t pos = ((((uint64_t)w[1]) << 32) | w[0]) & reg.mask;
    bool done = false;
    for (uint32_t probes = 0; probes <= reg.mask && !done; ++probes) {
        IssuerRegSlot* sl = reg.slots + pos;
        unsigned long long t = atomicCAS_system(&sl->state, 0ull, 1ull);
        if (t == 0ull) {
            const unsigned long long idx = atomicAdd_system(reg.counter, 1ull);
            if (idx >= reg.max_issuers) {
                atomicExch(error_flag, CTMR_E_TOO_MANY_ISSUERS);
                idx_out[k] = CTMR_ISSUER_BAD;
                sl->idx = CTMR_ISSUER_BAD;
            } else {
                sl->idx = (uint32_t)idx;
                uint32_t* by = reinterpret_cast<uint32_t*>(reg.by_index + 32ull * idx);
#pragma unroll
                for (int i = 0; i < 8; ++i) by[i] = w[i];
                idx_out[k] = (uint32_t)idx;
            }
            uint32_t* dg = reinterpret_cast<uint32_t*>(sl->digest);
#pragma unroll
            for (int i = 0; i < 8; ++i) dg[i] = w[i];
            tab_store_release<true>(&sl->state, 2ull);
            done = true;
            break;
        }
        while (t == 1ull) t = tab_load_acquire<true>(&sl->state);  // another RANK is publishing this slot
        const uint4* dg = reinterpret_cast<const uint4*>(sl->digest);
        const uint4 d0 = ld_cv_u4(dg), d1 = ld_cv_u4(dg + 1);
        if (d0.x == w[0] && d0.y == w[1] && d0.z == w[2] && d0.w == w[3] && d1.x == w[4] && d1.y == w[5] && d1.z == w[6] && d1.w == w[7]) {
            idx_out[k] = *reinterpret_cast<const volatile uint32_t*>(&sl->idx);
            done = true;
            break;
        }
        pos = (pos + 1) & reg.mask;
    }
    if (!done) {
        atomicExch(error_flag, CTMR_E_TOO_MANY_ISSUERS);
        idx_out[k] = CTMR_ISSUER_BAD;
    }
  }
}

cudaError_t launch_issuer_registry(const IssuerRegistry& reg, const uint8_t* digests, const uint8_t* ok, uint32_t n, uint32_t* idx_out,
                                   int* error_flag, cudaStream_t s) {
    if (!n) return cudaSuccess;
    issuer_registry_kernel<<<1, 1, 0, s>>>(reg, digests, ok, n, idx_out, error_flag);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Cross-process barrier in peer memory (multi-process groups: one process per GPU, tables attached by CUDA IPC).
// Lane t signals rank t (a release store of the epoch into t's flag word for this channel and this source) and
// waits for rank t's signal in its own flag words.  Stream ordered: everything launched before it on this stream
// -- K_map's remote inserts included -- is complete when the signal leaves.  A wait that does not end within
// the group's timeout (60 s, CTMR_PEER_TIMEOUT_MS) raises the error flag instead of hanging the GPU.
// ------------------------------------------------------------------------------------------------
__global__ void peer_barrier_kernel(PeerFlags pf, uint32_t channel, unsigned long long epoch, int* error_flag) {
    const uint32_t t = threadIdx.x;
    if (t >= pf.world) return;
    __threadfence_system();
    tab_store_release<true>(pf.flags[t] + (size_t)channel * kMaxWorld + pf.rank, epoch);
    const unsigned long long* mine = pf.flags[pf.rank] + (size_t)channel * kMaxWorld + t;
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
    while (tab_load_acquire<true>(mine) < epoch) {
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
        if (t1 - t0 > pf.timeout_ns) {
            atomicExch(error_flag, CTMR_E_PEER_TIMEOUT);
            break;
        }
        __nanosleep(200);
    }
}
// mailbox: every rank leaves one word in every rank's mailbox row (read after a barrier)
__global__ void peer_post_kernel(PeerFlags pf, unsigned long long value) {
    const uint32_t t = threadIdx.x;
    if (t < pf.world) tab_store_release<true>(pf.flags[t] + (size_t)kPeerChannels * kMaxWorld + pf.rank, value);
}
cudaError_t launch_peer_post(const PeerFlags& pf, unsigned long long value, cudaStream_t s) {
    peer_post_kernel<<<1, 32, 0, s>>>(pf, value);
    return cudaGetLastError();
}
cudaError_t launch_peer_barrier(const PeerFlags& pf, uint32_t channel, unsigned long long epoch, int* error_flag, cudaStream_t s) {
    peer_barrier_kernel<<<1, 32, 0, s>>>(pf, channel, epoch, error_flag);
    return cudaGetLastError();
}

// One-shot all-reduce(sum) of [per-issuer unique counts || status counters] over peer memory: every rank reads every
// rank's arrays (a few KB each over NVLink) and adds them up.  Callers bracket it with barriers.
__global__ void __launch_bounds__(256) hist_sum_kernel(PeerFlags pf, uint32_t n_slots, unsigned long long* __restrict__ counts_dst,
                                                       unsigned long long* __restrict__ status_dst) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_slots && counts_dst) {
        unsigned long long acc = 0;
        for (uint32_t r = 0; r < pf.world; ++r) acc += ld_volatile_u64(pf.issuer_counts[r] + i);
        counts_dst[i] = acc;
    }
    if (i < CTMR_ST__COUNT && status_dst) {
        unsigned long long acc = 0;
        for (uint32_t r = 0; r < pf.world; ++r) acc += ld_volatile_u64(pf.status_counts[r] + i);
        status_dst[i] = acc;
    }
}
cudaError_t launch_hist_sum(const PeerFlags& pf, uint32_t n_slots, unsigned long long* counts_dst, unsigned long long* status_dst,
                            cudaStream_t s) {
    const uint32_t n = n_slots > CTMR_ST__COUNT ? n_slots : CTMR_ST__COUNT;
    hist_sum_kernel<<<blocks_for(n, 256), 256, 0, s>>>(pf, n_slots, counts_dst, status_dst);
    return cudaGetLastError();
}

}  // namespace ctmr
