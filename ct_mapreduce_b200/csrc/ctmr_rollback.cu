// ctmr_rollback.cu -- the device state back to the start of an earlier entry-taking call (include/ctmr.h "rollback"):
// the rollback marks the calls take, the cluster-local deletion of the records first seen at or above the target index,
// and ctmr_rollback / ctmr_group_rollback on one ctx, a group and peer ranks.
//
// Deletion.  Every table is open addressing with linear probing, so a record cannot simply be cleared: that would cut
// the probe chains of the records behind it.  But only the CLUSTER a removed record lies in (a maximal run of slots live
// at the current epoch, wrapping at the table's end) has to be rebuilt.  One select pass per table marks the first
// removed slot of each such cluster; one owner thread per marked cluster then walks it from there, clears each slot it
// reads and places each survivor again from its home slot.  Clusters are disjoint, so the owners need no atomics.
// The pair counts and the per-issuer histogram are then rebuilt from the live keys (recount_kernel, as a delta apply
// does), and the status counters come back from the mark.
#include "ctmr_ctx.cuh"

namespace ctmr {

// The state word and the first-seen index of a slot, in 16-byte streaming loads of the words that hold them (the select
// pass reads each slot once), and the slot's home under a table of mask + 1 slots (the probe start of its insert).
struct SlotHead {
    unsigned long long w, inv_first;
};
__device__ __forceinline__ SlotHead slot_head(const KnownSlot* p, bool stream) {
    const uint4 v = stream ? __ldcs(reinterpret_cast<const uint4*>(p)) : *reinterpret_cast<const uint4*>(p);
    return {((unsigned long long)v.w << 32) | v.z, ((unsigned long long)v.y << 32) | v.x};
}
__device__ __forceinline__ SlotHead slot_head(const PairSlot* p, bool stream) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    const uint4 a = stream ? __ldcs(q) : q[0], b = stream ? __ldcs(q + 1) : q[1];
    return {((unsigned long long)b.w << 32) | b.z, ((unsigned long long)a.w << 32) | a.z};
}
__device__ __forceinline__ SlotHead slot_head(const MetaSlot* p, bool stream) {
    const uint4* q = reinterpret_cast<const uint4*>(p) + 1;
    const uint4 v = stream ? __ldcs(q) : *q;
    return {((unsigned long long)v.w << 32) | v.z, ((unsigned long long)v.y << 32) | v.x};
}
// known_insert's home: (key_hash >> 7) & mask.  The tag keeps key_hash bits 2..47 and a table has at most 2^32 slots, so
// the tag alone gives it.
__device__ __forceinline__ uint64_t slot_home(const KnownSlot& s, uint64_t mask) { return ((s.tag & kTagHashBits) >> 7) & mask; }
__device__ __forceinline__ uint64_t slot_home(const PairSlot& s, uint64_t mask) { return mix64(s.key) & mask; }      // pair_insert
__device__ __forceinline__ uint64_t slot_home(const MetaSlot& s, uint64_t mask) { return (s.h1 >> 5) & mask; }      // meta_insert_at

__device__ __forceinline__ bool head_live(const SlotHead& h, uint32_t epoch) { return slot_state(h.w, epoch) != 0u; }
__device__ __forceinline__ bool head_removed(const SlotHead& h, uint32_t epoch, uint64_t since) {
    return head_live(h, epoch) && ~h.inv_first >= since;
}

// Whether removed slot i is the first removed slot of its cluster: walk back to the cluster's start (an empty slot)
// and meet no other removed slot.  The table is not written during the select pass, so every walk of a cluster sees the
// same cluster.  A walk that wraps the table's end meets slots of higher index that still lie before i in the cluster.
// A table with no empty slot at all is one cyclic cluster: its lowest removed slot owns it (kOwnerNoEmpty).
enum : int { kNotOwner = 0, kOwner = 1, kOwnerNoEmpty = 2 };
template <class Slot>
__device__ int first_removed(const Slot* table, uint64_t mask, uint32_t epoch, uint64_t since, uint64_t i) {
    bool wrapped = false;
    for (uint64_t k = 1; k <= mask; ++k) {
        const uint64_t q = (i - k) & mask;
        const SlotHead h = slot_head(table + q, false);
        if (!head_live(h, epoch)) return wrapped ? kNotOwner : kOwner;
        if (~h.inv_first >= since) {
            if (q < i) return kNotOwner;
            wrapped = true;
        }
    }
    return kOwnerNoEmpty;
}

// Select: one pass over the table; owners[0 .. n_words) gets bit i set for the first removed slot i of every cluster,
// owners[n_words] = 1 when the table has no empty slot.
template <class Slot>
__global__ void __launch_bounds__(256) rollback_select_kernel(const Slot* __restrict__ table, uint64_t mask, uint32_t epoch, uint64_t since,
                                                              uint32_t* __restrict__ owners, uint64_t n_words) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= mask; i += (uint64_t)gridDim.x * blockDim.x) {
        if (!head_removed(slot_head(table + i, true), epoch, since)) continue;
        const int o = first_removed(table, mask, epoch, since, i);
        if (o != kNotOwner) atomicOr(owners + (i >> 5), 1u << (i & 31u));
        if (o == kOwnerNoEmpty) owners[n_words] = 1u;
    }
}

// Knuth's Algorithm R: slot i cleared, and each record behind it up to the next empty slot moved back into the hole when
// its home does not lie between the hole and the record.  Returns the slot left empty.
template <class Slot>
__device__ uint64_t shift_delete(Slot* table, uint64_t mask, uint32_t epoch, uint64_t i) {
    table[i] = Slot{};
    for (uint64_t j = (i + 1) & mask;; j = (j + 1) & mask) {
        const Slot s = table[j];
        if (!head_live(slot_head(&s, false), epoch)) return i;
        if (((slot_home(s, mask) - i - 1) & mask) < ((j - i) & mask)) continue;  // home in (i, j]: the record stays
        table[i] = s;
        table[j] = Slot{};
        i = j;
    }
}

// Rebuild the cluster whose first removed slot is f.  The slots before f keep their places: with nothing removed ahead
// of them, placing them again would put each where it is.  From f on, each slot is read, cleared (all zero: the
// canonical empty slot), and a survivor is placed again at the first empty slot from its home.  The slots from its home
// to its old position were all live, the ones read so far are cleared or hold survivors placed earlier, and its old slot
// is cleared: the survivor lands at or before its old position, never further from home than it was, so the probe rule
// (ctmr_common.cuh) holds.  The probe never passes the slot just read, so the slots not read yet stay as they were, and
// the walk ends at the first slot that was empty.  A table with no empty slot has no cluster start to keep the slots
// before f in place: f is taken out by shift_delete first, and the walk covers the one cluster that remains, from its
// first removed slot to the slot shift_delete left empty.
template <class Slot>
__device__ void rebuild_cluster(Slot* table, uint64_t mask, uint32_t epoch, uint64_t since, uint64_t f, bool no_empty) {
    if (no_empty) {
        const uint64_t e = shift_delete(table, mask, epoch, f);
        uint64_t d = 1;
        while (d <= mask && !head_removed(slot_head(table + ((e + d) & mask), false), epoch, since)) ++d;
        if (d > mask) return;
        f = (e + d) & mask;
    }
    for (uint64_t k = 0; k <= mask; ++k) {
        const uint64_t r = (f + k) & mask;
        const Slot s = table[r];
        const SlotHead h = slot_head(&s, false);
        if (k > 0 && !head_live(h, epoch)) break;
        table[r] = Slot{};
        if (~h.inv_first >= since) continue;
        uint64_t pos = slot_home(s, mask);
        while (head_live(slot_head(table + pos, false), epoch)) pos = (pos + 1) & mask;
        table[pos] = s;
    }
}

template <class Slot>
__global__ void __launch_bounds__(256) rollback_rebuild_kernel(Slot* table, uint64_t mask, uint32_t epoch, uint64_t since,
                                                               const uint32_t* __restrict__ owners, uint64_t n_words) {
    const bool no_empty = owners[n_words] != 0u;
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (uint64_t)gridDim.x * blockDim.x)
        for (uint32_t bits = owners[w]; bits; bits &= bits - 1u)
            rebuild_cluster(table, mask, epoch, since, (w << 5) + (uint64_t)(__ffs(bits) - 1), no_empty);
}

template <class Slot>
cudaError_t launch_rollback_table(Slot* table, uint64_t mask, uint32_t epoch, uint64_t since, uint32_t* owners, int sm_count, cudaStream_t s) {
    const uint64_t n_words = (mask + 1 + 31) / 32;
    cudaError_t e = cudaMemsetAsync(owners, 0, (n_words + 1) * sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    const unsigned sel = (unsigned)std::min<uint64_t>((mask + 1 + 255) / 256, (uint64_t)sm_count * 8);
    rollback_select_kernel<Slot><<<sel, 256, 0, s>>>(table, mask, epoch, since, owners, n_words);
    const unsigned reb = (unsigned)std::min<uint64_t>((n_words + 255) / 256, (uint64_t)sm_count * 8);
    rollback_rebuild_kernel<Slot><<<reb, 256, 0, s>>>(table, mask, epoch, since, owners, n_words);
    return cudaGetLastError();
}

}  // namespace ctmr

namespace ctmr_host {

int note_call_start(ctmr_ctx** m, uint32_t W, uint64_t next_index, cudaStream_t s) {
    ctmr_ctx* c0 = m[0];
    if (c0->marks > c0->marks_lo && c0->mark_index[(c0->marks - 1) % CTMR_ROLLBACK_MARKS] == next_index) return CTMR_OK;
    const uint64_t slot = c0->marks % CTMR_ROLLBACK_MARKS;
    for (uint32_t r = 0; r < W; ++r) {
        ctmr_ctx* c = m[r];
        const cudaStream_t cs = s ? s : c->stream.get();
        CU(c, cudaSetDevice(c->device));
        CU(c, cudaMemcpyAsync(c->mark_status + slot * CTMR_ST__COUNT, c->st.status_counts, CTMR_ST__COUNT * sizeof(unsigned long long),
                              cudaMemcpyDeviceToDevice, cs));
        CU(c, cudaEventRecord(c->mark_taken, cs));
    }
    c0->mark_index[slot] = next_index;
    ++c0->marks;
    c0->marks_lo = std::max<uint64_t>(c0->marks_lo, c0->marks > CTMR_ROLLBACK_MARKS ? c0->marks - CTMR_ROLLBACK_MARKS : 0);
    return CTMR_OK;
}

}  // namespace ctmr_host

namespace {

// The mark at n of c (the ctx that holds the delta state, whose next index is `cur`): *kept = the marks that stay (the
// mark at n is the last of them).  Every refusal is CTMR_E_INVALID with nothing touched.
int find_mark(ctmr_ctx* c, uint64_t cur, uint64_t n, uint64_t* kept) {
    const std::string at = "rollback to next index " + std::to_string(n);
    if (n > cur) return fail(c, CTMR_E_INVALID, at + ": past the next index " + std::to_string(cur));
    if (n < c->delta_floor)
        return fail(c, CTMR_E_INVALID, at + ": below the delta floor " + std::to_string(c->delta_floor) + " (the last reset or load)");
    for (uint64_t k = c->marks; k > c->marks_lo; --k) {  // marks marks_lo .. marks - 1, the newest first
        const uint64_t idx = c->mark_index[(k - 1) % CTMR_ROLLBACK_MARKS];
        if (idx == n) {
            *kept = k;
            return CTMR_OK;
        }
        if (idx < n) break;
    }
    if (c->marks_lo > 0 && (c->marks == c->marks_lo || n < c->mark_index[c->marks_lo % CTMR_ROLLBACK_MARKS]))
        return fail(c, CTMR_E_INVALID, at + ": the mark has dropped out of the last " + std::to_string(CTMR_ROLLBACK_MARKS) + " call starts");
    return fail(c, CTMR_E_INVALID, at + ": not the start of an entry-taking call of this handle");
}

// What c needs before any work: no earlier call still running against its tables, its error flag read (and cleared,
// as ctmr_check_device does: a raised flag is that call's failure, reported here instead of the rollback's own
// outcome), and the owner bitmap of its largest table with its no-empty-slot word.
int rollback_prepare(ctmr_ctx* c, DevBuf<uint32_t>& owners) {
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaDeviceSynchronize());
    const int rc = ctmr_check_device(c, nullptr);
    if (rc) return rc;
    const uint64_t slots = std::max({c->st.table_mask, c->st.pair_mask, c->st.meta_mask}) + 1;
    if (alloc(owners, (slots + 31) / 32 + 1) != cudaSuccess) {
        (void)cudaGetLastError();
        return fail(c, CTMR_E_NOMEM, "ctmr_rollback: no device memory for the cluster bitmap");
    }
    return CTMR_OK;
}

// c's shard without the records first seen at or above n, its counts rebuilt, its status counters those of mark `slot`.
// The deletion works in place: after a failure the tables are undefined (raise_flag).
int rollback_shard(ctmr_ctx* c, uint64_t n, uint64_t slot, uint32_t* owners) {
    CU(c, cudaSetDevice(c->device));
    const DeviceState& st = c->st;
    CU(c, launch_rollback_table(st.table, st.table_mask, st.epoch, n, owners, c->sm_count, c->stream));
    CU(c, launch_rollback_table(st.pairs, st.pair_mask, st.epoch, n, owners, c->sm_count, c->stream));
    CU(c, launch_rollback_table(st.meta, st.meta_mask, st.epoch, n, owners, c->sm_count, c->stream));
    CU(c, launch_recount(st, c->sm_count, c->stream));
    CU(c, cudaMemcpyAsync(st.status_counts, c->mark_status + slot * CTMR_ST__COUNT, CTMR_ST__COUNT * sizeof(unsigned long long),
                          cudaMemcpyDeviceToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return ctmr_check_device(c, nullptr);
}

// a rollback that failed after its work began leaves c's tables undefined: ctmr_check_device reports it from here on
void raise_flag(ctmr_ctx* c, int rc) {
    const std::string err = c->err;
    cudaSetDevice(c->device);
    cudaMemcpy(c->st.error_flag, &rc, sizeof rc, cudaMemcpyHostToDevice);
    c->err = err;
}

// the host side of c (the ctx that holds the delta state) after its shards were rolled back to n: the marks above n go,
// and the evictions made at or above n count as made at n (the first of them has the highest now).  marks_lo stays: the
// marks that go have overwritten the ring slots of the marks below it.
void rollback_host(ctmr_ctx* c, uint64_t n, uint64_t kept) {
    c->marks = kept;
    auto& ev = c->evict_marks;
    size_t k = 0;
    while (k < ev.size() && ev[k].first < n) ++k;
    if (k < ev.size()) {
        ev[k].first = n;
        ev.resize(k + 1);
    }
}

// ctx or group (not attached to peers): members m[0..W), member 0 holds the marks
int rollback_members(ctmr_ctx** m, uint32_t W, uint64_t* next_index, ctmr_ctx** failed, uint64_t n) {
    *failed = m[0];
    if (n == *next_index) return CTMR_OK;
    uint64_t kept = 0;
    int rc = find_mark(m[0], *next_index, n, &kept);
    if (rc) return rc;
    const uint64_t slot = (kept - 1) % CTMR_ROLLBACK_MARKS;
    std::vector<DevBuf<uint32_t>> owners(W);
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = rollback_prepare(m[r], owners[r]);
        if (rc) return rc;
    }
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = rollback_shard(m[r], n, slot, owners[r]);
        if (rc) {
            raise_flag(m[r], rc);
            return rc;
        }
    }
    for (uint32_t r = 0; r < W; ++r) {  // the bitmaps are freed on their own devices
        cudaSetDevice(m[r]->device);
        owners[r].reset();
    }
    rollback_host(m[0], n, kept);
    *next_index = n;
    *failed = nullptr;
    return CTMR_OK;
}

// a rank attached to peers: its part of the collective rollback
int rollback_peer(ctmr_ctx* c, uint64_t n) {
    uint64_t row[kMaxWorld] = {};
    uint64_t kept = 0;
    DevBuf<uint32_t> owners;
    const bool noop = n == c->next_index;
    int rc = noop ? CTMR_OK : find_mark(c, c->next_index, n, &kept);
    if (rc == CTMR_OK && !noop) rc = rollback_prepare(c, owners);
    // every rank has a mark at n, or every rank returns unchanged
    rc = peer_agree(c, rc, 0, row, "", "rollback failed");
    if (rc) return rc;
    if (!noop) rc = rollback_shard(c, n, (kept - 1) % CTMR_ROLLBACK_MARKS, owners);
    const int local = rc;
    if (local == CTMR_OK && !noop) {  // this rank's shard is back at n, whatever the others report
        rollback_host(c, n, kept);
        c->next_index = n;
    }
    // no rank starts its next call (whose string identities may go into this rank's table) before every rank is done;
    // a rank whose deletion failed makes the call fail everywhere
    rc = peer_agree(c, rc, 0, row, "", "rollback failed");
    if (local) raise_flag(c, local);
    return rc;
}

}  // namespace

extern "C" {

int ctmr_rollback(ctmr_ctx* c, uint64_t next_index) {
    if (c && c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_rollback");
    if (c && peer_call(c)) return rollback_peer(c, next_index);
    return on_ctx(c, rollback_members, next_index);
}
int ctmr_group_rollback(ctmr_group* g, uint64_t next_index) { return on_group(g, rollback_members, next_index); }

}  // extern "C"
