// ctmr_checkpoint.cu -- portable checkpoints (include/ctmr.h "portable checkpoint"): the live records of the tables, the
// issuer registry, the status counters and the next index, saved in one part per ctx, group or rank, and loaded into a
// ctx, a group or peer ranks of any size and capacities.
//
// Save: a count pass gives each table's live slots per tile (compact_plan); the tiles are then compacted in slot order,
// as many at a time as the key scratch holds, and copied to the caller's buffer.  No record carries a slot position or a
// capacity.  Load: every member streams every part's records through its key scratch and inserts the ones it owns
// under the target's world (evict_reinsert_kernel, ckpt_pairs_kernel, ckpt_meta_kernel); all inserts are local.
//
// Delta checkpoints (include/ctmr.h "delta checkpoint") are parts of the same layout with their own header: the count
// and compact passes keep only the records whose first-seen index is at or above `since`.  Apply checks the parts and
// the target, appends the new digests to the registry, evicts as the source did after `since`, inserts the records
// through the load's path and rebuilds every pair count and the histogram from the keys (recount_kernel).
#include <unordered_set>

#include "ctmr_ctx.cuh"

namespace {

struct CkptHeader {
    char magic[8];  // "CTMRCKP1"
    uint32_t part, n_parts;
    uint64_t n_issuers, next_index;
    uint64_t status[CTMR_ST__COUNT];  // this part's status counters
    uint64_t n_keys, n_pairs, n_meta;
    uint64_t reserved;                // 0: keeps the records 32-byte aligned in the part
};
static_assert(sizeof(CkptHeader) == 128, "checkpoint header layout");

// A delta part's header: the checkpoint's fields, packed beside since and evict_now (a part count fits 16 bits: at most
// kMaxWorld ranks save one part each).
struct DeltaHeader {
    char magic[8];  // "CTMRDLT1"
    uint16_t part, n_parts;
    uint32_t n_issuers;
    uint64_t since, next_index;
    int64_t evict_now;                // the highest now of an eviction from `since` on; INT64_MIN: none
    uint64_t status[CTMR_ST__COUNT];  // this part's status counters (totals)
    uint64_t n_keys, n_pairs, n_meta;
};
static_assert(sizeof(DeltaHeader) == sizeof(CkptHeader), "delta header layout");

// what a delta's parts add to a checkpoint's
struct Delta {
    uint64_t since;
    int64_t evict_now;
};

constexpr int64_t kEveryKey = INT64_MIN;  // compaction filter: no key is expired

// the live records of one member's three tables
struct MemberPlan {
    CompactPlan keys, pairs, meta;
};

// since > 0: the records first seen at or above it
int plan_member(ctmr_ctx* c, MemberPlan& p, uint64_t since) {
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaDeviceSynchronize());
    int rc = compact_plan(c, c->st.table, c->st.table_mask + 1, kEveryKey, p.keys, since);
    if (rc == CTMR_OK) rc = compact_plan(c, c->st.pairs, c->st.pair_mask + 1, kEveryKey, p.pairs, since);
    if (rc == CTMR_OK) rc = compact_plan(c, c->st.meta, c->st.meta_mask + 1, kEveryKey, p.meta, since);
    return rc;
}

// One table's live slots into dst, in slot order: runs of tiles whose records fit the key scratch, compacted there and
// copied out.  The scratch holds at least one tile (ensure_scratch before).
template <class Slot>
int save_records(ctmr_ctx* c, const Slot* table, uint64_t n_slots, const CompactPlan& plan, uint64_t since, uint8_t* dst) {
    const uint64_t cap = c->scratch_cap * sizeof(ctmr_key) / sizeof(Slot);
    Slot* stage = reinterpret_cast<Slot*>(c->keys_scratch.get());
    const std::vector<unsigned long long>& base = plan.host;
    for (uint64_t t0 = 0, t1 = 0; t0 < plan.tiles(); t0 = t1) {
        t1 = t0 + 1;
        while (t1 < plan.tiles() && base[t1 + 1] - base[t0] <= cap) ++t1;
        const uint64_t n = base[t1] - base[t0];
        if (!n) continue;
        CU(c, launch_evict_compact(table, n_slots, c->st.epoch, kEveryKey, t0, t1, plan.dev.get(), stage, (uint32_t*)nullptr, c->stream,
                                   since));
        CU(c, cudaMemcpyAsync(dst + base[t0] * sizeof(Slot), stage, n * sizeof(Slot), cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
    }
    return CTMR_OK;
}

// The part of members m[0..W) (a ctx, or every member of a group): header, the registry (m[0]'s view of it), then the
// keys of every member, their pairs, their string identities.  buf == NULL: *need only.  delta != NULL: a delta part,
// the records first seen at or above delta->since (m[0] holds the delta floor and the evictions).
int save_members(ctmr_ctx** m, uint32_t W, uint32_t part, uint32_t n_parts, uint64_t next_index, const uint64_t* delta, uint8_t* buf,
                 uint64_t cap, uint64_t* need, ctmr_ctx** failed) {
    *failed = m[0];
    CU(m[0], cudaSetDevice(m[0]->device));
    const uint64_t since = delta ? *delta : 0;
    if (delta && since > next_index)
        return fail(m[0], CTMR_E_INVALID, "delta since " + std::to_string(since) + " lies past the next index " + std::to_string(next_index));
    if (delta && since < m[0]->delta_floor)
        return fail(m[0], CTMR_E_INVALID, "delta since " + std::to_string(since) + " lies before the last reset or load (next index " +
                                              std::to_string(m[0]->delta_floor) + "): take a full checkpoint");
    int rc = refresh_digests(m[0]);
    if (rc) return rc;
    CkptHeader h{};
    std::memcpy(h.magic, "CTMRCKP1", 8);
    h.part = part;
    h.n_parts = n_parts;
    h.n_issuers = m[0]->digests.size();
    h.next_index = next_index;
    std::vector<MemberPlan> plans(W);
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        uint64_t keys = 0, status[CTMR_ST__COUNT];
        if (buf || delta) {
            rc = plan_member(m[r], plans[r], since);
            if (rc == CTMR_OK && buf) rc = ensure_scratch(m[r], std::max<uint64_t>(m[r]->stage_entries, kCompactTile));
            keys = plans[r].keys.live();
        } else {  // the key count of ctmr_table_stats; the pairs and string identities from their count passes
            rc = ctmr_table_stats(m[r], &keys, nullptr);
            if (rc == CTMR_OK) rc = compact_plan(m[r], m[r]->st.pairs, m[r]->st.pair_mask + 1, kEveryKey, plans[r].pairs);
            if (rc == CTMR_OK) rc = compact_plan(m[r], m[r]->st.meta, m[r]->st.meta_mask + 1, kEveryKey, plans[r].meta);
        }
        if (rc == CTMR_OK) rc = ctmr_status_counters(m[r], status);
        if (rc) return rc;
        for (int k = 0; k < CTMR_ST__COUNT; ++k) h.status[k] += status[k];
        h.n_keys += keys;
        h.n_pairs += plans[r].pairs.live();
        h.n_meta += plans[r].meta.live();
    }
    *need = sizeof h + 32 * h.n_issuers + sizeof(KnownSlot) * h.n_keys + sizeof(PairSlot) * h.n_pairs + sizeof(MetaSlot) * h.n_meta;
    if (!buf) return CTMR_OK;
    *failed = m[0];
    if (cap < *need) return fail(m[0], CTMR_E_INVALID, "checkpoint buffer too small (ctmr_checkpoint_size)");
    uint8_t* p = buf;
    if (delta) {
        DeltaHeader dh{};
        std::memcpy(dh.magic, "CTMRDLT1", 8);
        dh.part = (uint16_t)part;
        dh.n_parts = (uint16_t)n_parts;
        dh.n_issuers = (uint32_t)h.n_issuers;
        dh.since = since;
        dh.next_index = next_index;
        dh.evict_now = evicted_since(m[0], since);
        std::memcpy(dh.status, h.status, sizeof dh.status);
        dh.n_keys = h.n_keys;
        dh.n_pairs = h.n_pairs;
        dh.n_meta = h.n_meta;
        std::memcpy(p, &dh, sizeof dh);
    } else {
        std::memcpy(p, &h, sizeof h);
    }
    p += sizeof h;
    for (const auto& d : m[0]->digests) {
        std::memcpy(p, d.data(), 32);
        p += 32;
    }
    for (int kind = 0; kind < 3; ++kind)
        for (uint32_t r = 0; r < W; ++r) {
            ctmr_ctx* c = m[r];
            *failed = c;
            const MemberPlan& pl = plans[r];
            CU(c, cudaSetDevice(c->device));
            if (kind == 0) rc = save_records(c, c->st.table, c->st.table_mask + 1, pl.keys, since, p);
            if (kind == 1) rc = save_records(c, c->st.pairs, c->st.pair_mask + 1, pl.pairs, since, p);
            if (kind == 2) rc = save_records(c, c->st.meta, c->st.meta_mask + 1, pl.meta, since, p);
            if (rc) return rc;
            p += kind == 0 ? sizeof(KnownSlot) * pl.keys.live() : 32 * (kind == 1 ? pl.pairs.live() : pl.meta.live());
        }
    *failed = nullptr;
    return CTMR_OK;
}

// The parts of one checkpoint, checked before anything changes: every part readable and whole, the same part count,
// each index once, the same registry and next index; the registry fits the target.  hs[i] = part i's header.  delta !=
// NULL: the parts of one delta checkpoint (their headers read into hs as a checkpoint's), which also agree on since;
// *delta = since and the highest evict_now of the parts.
int check_parts(ctmr_ctx* c, const uint8_t* const* parts, const uint64_t* bytes, uint32_t n, std::vector<CkptHeader>& hs,
                Delta* delta = nullptr) {
    if (!parts || !bytes || n == 0) return fail(c, CTMR_E_INVALID, "no checkpoint parts");
    hs.assign(n, CkptHeader{});
    std::vector<bool> seen(n, false);
    for (uint32_t i = 0; i < n; ++i) {
        if (!parts[i]) return fail(c, CTMR_E_INVALID, "checkpoint part " + std::to_string(i) + " is NULL");
        if (bytes[i] < sizeof(CkptHeader)) return fail(c, CTMR_E_INVALID, "truncated checkpoint part");
        CkptHeader& h = hs[i];
        std::memcpy(&h, parts[i], sizeof h);
        if (delta) {
            DeltaHeader dh;
            std::memcpy(&dh, parts[i], sizeof dh);
            if (std::memcmp(dh.magic, "CTMRDLT1", 8) != 0) return fail(c, CTMR_E_INVALID, "not a ctmr delta checkpoint part");
            h.part = dh.part;
            h.n_parts = dh.n_parts;
            h.n_issuers = dh.n_issuers;
            h.next_index = dh.next_index;
            std::memcpy(h.status, dh.status, sizeof h.status);
            h.n_keys = dh.n_keys;
            h.n_pairs = dh.n_pairs;
            h.n_meta = dh.n_meta;
            if (i == 0) *delta = Delta{dh.since, dh.evict_now};
            if (dh.since != delta->since) return fail(c, CTMR_E_INVALID, "delta parts disagree (since): parts of different deltas");
            delta->evict_now = std::max(delta->evict_now, dh.evict_now);
        } else if (std::memcmp(h.magic, "CTMRCKP1", 8) != 0) {
            return fail(c, CTMR_E_INVALID, "not a ctmr checkpoint part");
        }
        const uint64_t body = bytes[i] - sizeof h;
        const unsigned __int128 want = (unsigned __int128)32 * h.n_issuers + (unsigned __int128)sizeof(KnownSlot) * h.n_keys +
                                       (unsigned __int128)sizeof(PairSlot) * h.n_pairs + (unsigned __int128)sizeof(MetaSlot) * h.n_meta;
        if (want > body) return fail(c, CTMR_E_INVALID, "truncated checkpoint part");
        if (h.n_parts != n) return fail(c, CTMR_E_INVALID, "checkpoint of " + std::to_string(h.n_parts) + " parts, " + std::to_string(n) + " given");
        if (h.part >= n || seen[h.part]) return fail(c, CTMR_E_INVALID, "checkpoint part index given twice or out of range");
        seen[h.part] = true;
        if (h.n_issuers != hs[0].n_issuers || h.next_index != hs[0].next_index ||
            std::memcmp(parts[i] + sizeof h, parts[0] + sizeof h, 32 * h.n_issuers) != 0)
            return fail(c, CTMR_E_INVALID, "checkpoint parts disagree (issuer registry or next index): parts of different checkpoints");
    }
    std::unordered_set<std::string> distinct;
    for (uint64_t k = 0; k < hs[0].n_issuers; ++k) {
        const std::string d(reinterpret_cast<const char*>(parts[0] + sizeof(CkptHeader) + 32 * k), 32);
        if (d == std::string(32, '\0') || !distinct.insert(d).second)
            return fail(c, CTMR_E_INVALID, "checkpoint registry holds a zero or repeated issuer digest");
    }
    if (hs[0].n_issuers > c->st.max_issuers) return fail(c, CTMR_E_TOO_MANY_ISSUERS, "checkpoint holds more issuers than config.max_issuers");
    return CTMR_OK;
}

// What a load allocates before it changes anything: the registry upload (on the member that rebuilds it) and the scratch
// the records stream through.
int load_prepare(ctmr_ctx* c, bool registry, uint64_t n_issuers, RegistryUpload& u) {
    CU(c, cudaSetDevice(c->device));
    int rc = registry ? snap_registry_alloc(c, n_issuers, u) : CTMR_OK;
    if (rc == CTMR_OK) rc = ensure_scratch(c, std::max<uint64_t>(c->stage_entries, kCompactTile));
    return rc;
}

// This ctx's tables, histograms and counters to zero, the host memos of the registry and the Chain[0] mirror gone.
int load_clear(ctmr_ctx* c) {
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaDeviceSynchronize());
    int rc = reset_tables(c, c->stream);
    if (rc == CTMR_OK) rc = clear_issuer_memos(c);
    CU(c, cudaStreamSynchronize(c->stream));
    return rc;
}

// Every part's records through c's key scratch, in chunks; the kernels keep the ones c owns.
int load_records(ctmr_ctx* c, const uint8_t* const* parts, const std::vector<CkptHeader>& hs) {
    CU(c, cudaSetDevice(c->device));
    const uint64_t cap_bytes = c->scratch_cap * sizeof(ctmr_key);
    uint8_t* stage = reinterpret_cast<uint8_t*>(c->keys_scratch.get());
    const uint32_t ni = (uint32_t)hs[0].n_issuers;
    for (size_t i = 0; i < hs.size(); ++i) {
        const CkptHeader& h = hs[i];
        const uint8_t* p = parts[i] + sizeof h + 32 * h.n_issuers;
        const uint64_t counts[3] = {h.n_keys, h.n_pairs, h.n_meta}, size[3] = {sizeof(KnownSlot), sizeof(PairSlot), sizeof(MetaSlot)};
        for (int kind = 0; kind < 3; ++kind) {
            const uint64_t per = cap_bytes / size[kind];
            for (uint64_t at = 0; at < counts[kind]; at += per) {
                const uint64_t n = std::min(per, counts[kind] - at);
                // stream ordered: the copy waits for the previous chunk's kernel
                CU(c, cudaMemcpyAsync(stage, p + at * size[kind], n * size[kind], cudaMemcpyHostToDevice, c->stream));
                if (kind == 0) CU(c, launch_evict_reinsert(c->st, reinterpret_cast<const KnownSlot*>(stage), n, ni, true, c->stream));
                if (kind == 1) CU(c, launch_ckpt_pairs(c->st, reinterpret_cast<const PairSlot*>(stage), n, ni, c->stream));
                if (kind == 2) CU(c, launch_ckpt_meta(c->st, reinterpret_cast<const MetaSlot*>(stage), n, c->stream));
            }
            p += counts[kind] * size[kind];
        }
    }
    CU(c, cudaStreamSynchronize(c->stream));
    return ctmr_check_device(c, nullptr);
}

// status counters of the checkpoint (the sum over its parts) into c
int load_status(ctmr_ctx* c, const std::vector<CkptHeader>& hs) {
    uint64_t sum[CTMR_ST__COUNT] = {};
    for (const CkptHeader& h : hs)
        for (int k = 0; k < CTMR_ST__COUNT; ++k) sum[k] += h.status[k];
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaMemcpy(c->st.status_counts, sum, sizeof sum, cudaMemcpyHostToDevice));
    return CTMR_OK;
}

// After a failed insert: the members as after a reset, the checkpoint's registry kept.
void load_undo(ctmr_ctx** m, uint32_t W) {
    for (uint32_t r = 0; r < W; ++r) {
        const std::string err = m[r]->err;
        cudaSetDevice(m[r]->device);
        cudaDeviceSynchronize();
        reset_tables(m[r], m[r]->stream);
        cudaStreamSynchronize(m[r]->stream);
        m[r]->err = err;
    }
}

// ctx or group (not attached to peers): members m[0..W), member 0 rebuilds the registry
int load_members(ctmr_ctx** m, uint32_t W, const uint8_t* const* parts, const uint64_t* bytes, uint32_t n_parts, uint64_t* next_index,
                 ctmr_ctx** failed) {
    *failed = m[0];
    std::vector<CkptHeader> hs;
    int rc = check_parts(m[0], parts, bytes, n_parts, hs);
    if (rc) return rc;
    RegistryUpload u;
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = load_prepare(m[r], r == 0, hs[0].n_issuers, u);
        if (rc) return rc;
    }
    delta_floor_at(m[0], *next_index);  // from here on the old state is gone
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = load_clear(m[r]);
        if (rc) return rc;
    }
    *failed = m[0];
    rc = snap_registry_restore(m[0], parts[0] + sizeof(CkptHeader), hs[0].n_issuers, u);
    if (rc) return rc;
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = load_records(m[r], parts, hs);
        if (rc) {
            load_undo(m, W);
            return rc;
        }
    }
    *failed = m[0];
    rc = load_status(m[0], hs);
    if (rc) return rc;
    *next_index = hs[0].next_index;
    delta_floor_at(m[0], *next_index);
    *failed = nullptr;
    return CTMR_OK;
}

// a rank attached to peers: its part of the collective load
int load_peer(ctmr_ctx* c, const uint8_t* const* parts, const uint64_t* bytes, uint32_t n_parts) {
    std::vector<CkptHeader> hs;
    RegistryUpload u;
    const bool reg = c->st.peer.rank == 0;
    uint64_t row[kMaxWorld] = {};
    int rc = check_parts(c, parts, bytes, n_parts, hs);
    if (rc == CTMR_OK) rc = load_prepare(c, reg, hs[0].n_issuers, u);
    // every rank's checks passed, or every rank returns unchanged
    rc = peer_agree(c, rc, 0, row, "", "checkpoint load failed");
    if (rc) return rc;
    delta_floor_at(c, c->next_index);
    rc = load_clear(c);
    if (rc == CTMR_OK && reg) rc = snap_registry_restore(c, parts[0] + sizeof(CkptHeader), hs[0].n_issuers, u);
    const int brc = peer_barrier(c, CH_CKPT, c->stream);  // the registry is whole before any rank goes on
    if (rc == CTMR_OK) rc = brc;
    if (rc == CTMR_OK) rc = load_records(c, parts, hs);  // checks the device: a barrier that timed out too
    rc = peer_agree(c, rc, 0, row, "", "checkpoint load failed", true);  // the failed rank's own code on every rank
    if (rc) {
        load_undo(&c, 1);
        return rc;
    }
    if (reg) rc = load_status(c, hs);
    if (rc == CTMR_OK) c->next_index = hs[0].next_index;
    delta_floor_at(c, c->next_index);
    return rc;
}

// ---- delta checkpoints: apply ---------------------------------------------------------------------------------------
// The target's side of a delta's checks (parts checked by check_parts): it stands at the delta's since, so that deltas
// go on in order with no gap, and its registry is a prefix of the delta's.  c refreshes its view of the registry.
int check_target(ctmr_ctx* c, uint64_t next_index, const uint8_t* const* parts, const std::vector<CkptHeader>& hs, const Delta& d) {
    if (next_index != d.since)
        return fail(c, CTMR_E_INVALID, "delta since " + std::to_string(d.since) + " onto a state at next index " + std::to_string(next_index) +
                                           ": apply the deltas in order, onto the checkpoint they follow");
    CU(c, cudaSetDevice(c->device));
    const int rc = refresh_digests(c);
    if (rc) return rc;
    bool prefix = c->digests.size() <= hs[0].n_issuers;
    for (size_t i = 0; prefix && i < c->digests.size(); ++i)
        prefix = std::memcmp(c->digests[i].data(), parts[0] + sizeof(CkptHeader) + 32 * i, 32) == 0;
    if (!prefix) return fail(c, CTMR_E_INVALID, "the target's issuer registry is not a prefix of the delta's");
    return CTMR_OK;
}

// the delta's digests from index `have` on into the registry (c holds it), in one launch of the find-or-insert kernel,
// which takes a call's digests in order: digest i keeps index i
int registry_append(ctmr_ctx* c, const uint8_t* digests, uint64_t have, uint64_t n, const RegistryUpload& u) {
    CU(c, cudaSetDevice(c->device));
    if (n > have) {
        CU(c, cudaMemcpyAsync(u.digests, digests + 32 * have, (n - have) * 32, cudaMemcpyHostToDevice, c->stream));
        CU(c, launch_issuer_registry(c->reg, u.digests, nullptr, (uint32_t)(n - have), u.idx, c->st.error_flag, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
    }
    const int rc = refresh_digests(c);
    if (rc) return rc;
    if (c->digests.size() != n) return fail(c, CTMR_E_INVALID, "the delta's issuer digests did not take their indices");
    return ctmr_check_device(c, nullptr);
}

// members m[0..W) evict as the source did from since on, unless m[0] already evicted at that now or later from there
int apply_evict(ctmr_ctx** m, uint32_t W, const Delta& d, ctmr_ctx** failed) {
    if (d.evict_now == INT64_MIN || d.evict_now <= evicted_since(m[0], d.since)) return CTMR_OK;
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        uint64_t evicted = 0;
        const int rc = evict_shard(m[r], d.evict_now, &evicted);
        if (rc) return rc;
    }
    note_eviction(m[0], d.since, d.evict_now);
    return CTMR_OK;
}

// every part's records into c (the load's path), then c's pair counts and histogram rebuilt from its keys
int apply_records(ctmr_ctx* c, const uint8_t* const* parts, const std::vector<CkptHeader>& hs) {
    int rc = load_records(c, parts, hs);
    if (rc) return rc;
    CU(c, launch_recount(c->st, c->sm_count, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return ctmr_check_device(c, nullptr);
}

// the delta's status counters (totals) into c; holds = false: c's to zero (the sum lives on member 0 / rank 0)
int apply_status(ctmr_ctx* c, bool holds, const std::vector<CkptHeader>& hs) {
    if (holds) return load_status(c, hs);
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaMemset(c->st.status_counts, 0, CTMR_ST__COUNT * sizeof(uint64_t)));
    return CTMR_OK;
}

// ctx or group (not attached to peers): members m[0..W), member 0 holds the registry and the delta state
int apply_members(ctmr_ctx** m, uint32_t W, const uint8_t* const* parts, const uint64_t* bytes, uint32_t n_parts, uint64_t* next_index,
                  ctmr_ctx** failed) {
    *failed = m[0];
    std::vector<CkptHeader> hs;
    Delta d{};
    int rc = check_parts(m[0], parts, bytes, n_parts, hs, &d);
    if (rc == CTMR_OK) rc = check_target(m[0], *next_index, parts, hs, d);
    if (rc) return rc;
    const uint64_t have = m[0]->digests.size();
    RegistryUpload u;
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = load_prepare(m[r], r == 0, hs[0].n_issuers - have, u);
        if (rc) return rc;
    }
    *failed = m[0];
    rc = registry_append(m[0], parts[0] + sizeof(CkptHeader), have, hs[0].n_issuers, u);
    if (rc == CTMR_OK) rc = apply_evict(m, W, d, failed);
    if (rc) return rc;
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = apply_records(m[r], parts, hs);
        if (rc) {
            load_undo(m, W);
            delta_floor_at(m[0], *next_index);
            return rc;
        }
    }
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = apply_status(m[r], r == 0, hs);
        if (rc) return rc;
    }
    *next_index = hs[0].next_index;
    *failed = nullptr;
    return CTMR_OK;
}

// a rank attached to peers: its part of the collective apply, with the load's two agreements
int apply_peer(ctmr_ctx* c, const uint8_t* const* parts, const uint64_t* bytes, uint32_t n_parts) {
    std::vector<CkptHeader> hs;
    Delta d{};
    RegistryUpload u;
    const bool reg = c->st.peer.rank == 0;
    uint64_t row[kMaxWorld] = {};
    int rc = check_parts(c, parts, bytes, n_parts, hs, &d);
    if (rc == CTMR_OK) rc = check_target(c, c->next_index, parts, hs, d);
    const uint64_t have = c->digests.size();
    if (rc == CTMR_OK) rc = load_prepare(c, reg, hs[0].n_issuers - have, u);
    // every rank's checks passed, or every rank returns unchanged
    rc = peer_agree(c, rc, 0, row, "", "delta checkpoint apply failed");
    if (rc) return rc;
    if (reg) rc = registry_append(c, parts[0] + sizeof(CkptHeader), have, hs[0].n_issuers, u);
    const int brc = peer_barrier(c, CH_CKPT, c->stream);  // the registry is whole before any rank goes on
    if (rc == CTMR_OK) rc = brc;
    ctmr_ctx* failed = nullptr;
    if (rc == CTMR_OK) rc = apply_evict(&c, 1, d, &failed);
    if (rc == CTMR_OK) rc = apply_records(c, parts, hs);  // checks the device: a barrier that timed out too
    rc = peer_agree(c, rc, 0, row, "", "delta checkpoint apply failed", true);  // the failed rank's own code on every rank
    if (rc) {
        load_undo(&c, 1);
        delta_floor_at(c, c->next_index);
        return rc;
    }
    rc = apply_status(c, reg, hs);
    if (rc == CTMR_OK) c->next_index = hs[0].next_index;
    return rc;
}

// a rank attached to peers: size or save of its own part between barriers (other ranks write this rank's string
// identities and rank 0's registry during their collective calls; the first barrier orders those writes before the read)
int save_peer(ctmr_ctx* c, const uint64_t* delta, uint8_t* buf, uint64_t cap, uint64_t* need) {
    CU(c, cudaSetDevice(c->device));
    int rc = peer_barrier(c, CH_CKPT, c->stream);
    if (rc == CTMR_OK) {
        CU(c, cudaStreamSynchronize(c->stream));
        rc = ctmr_check_device(c, nullptr);
    }
    ctmr_ctx* failed = nullptr;
    if (rc == CTMR_OK) rc = save_members(&c, 1, c->st.peer.rank, c->st.peer.world, c->next_index, delta, buf, cap, need, &failed);
    if (!buf) return rc;
    const std::string err = c->err;
    const int brc = peer_barrier(c, CH_CKPT, c->stream);  // whatever this rank's outcome: the others wait for it
    if (brc) return rc ? rc : brc;
    CU(c, cudaStreamSynchronize(c->stream));
    const int crc = ctmr_check_device(c, nullptr);
    if (rc) c->err = err;
    return rc ? rc : crc;
}

}  // namespace

extern "C" {

int ctmr_checkpoint_size(ctmr_ctx* c, uint64_t* bytes) {
    if (!c || !bytes) return fail(c, CTMR_E_INVALID, "bad argument");
    if (c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_checkpoint_*");
    if (peer_call(c)) return save_peer(c, nullptr, nullptr, 0, bytes);
    ctmr_ctx* failed = nullptr;
    return save_members(&c, 1, 0, 1, c->next_index, nullptr, nullptr, 0, bytes, &failed);
}

int ctmr_checkpoint_save(ctmr_ctx* c, uint8_t* buf, uint64_t cap, uint64_t* written) {
    if (!c || !buf) return fail(c, CTMR_E_INVALID, "bad argument");
    if (c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_checkpoint_*");
    uint64_t need = 0;
    ctmr_ctx* failed = nullptr;
    const int rc = peer_call(c) ? save_peer(c, nullptr, buf, cap, &need)
                                : save_members(&c, 1, 0, 1, c->next_index, nullptr, buf, cap, &need, &failed);
    if (rc == CTMR_OK && written) *written = need;
    return rc;
}

int ctmr_checkpoint_load(ctmr_ctx* c, const uint8_t* const* parts, const uint64_t* part_bytes, uint32_t n_parts) {
    if (!c) return CTMR_E_INVALID;
    if (c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_checkpoint_*");
    if (peer_call(c)) return load_peer(c, parts, part_bytes, n_parts);
    ctmr_ctx* failed = nullptr;
    return load_members(&c, 1, parts, part_bytes, n_parts, &c->next_index, &failed);
}

int ctmr_checkpoint_delta_size(ctmr_ctx* c, uint64_t since, uint64_t* bytes) {
    if (!c || !bytes) return fail(c, CTMR_E_INVALID, "bad argument");
    if (c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_checkpoint_*");
    if (peer_call(c)) return save_peer(c, &since, nullptr, 0, bytes);
    ctmr_ctx* failed = nullptr;
    return save_members(&c, 1, 0, 1, c->next_index, &since, nullptr, 0, bytes, &failed);
}

int ctmr_checkpoint_delta_save(ctmr_ctx* c, uint64_t since, uint8_t* buf, uint64_t cap, uint64_t* written) {
    if (!c || !buf) return fail(c, CTMR_E_INVALID, "bad argument");
    if (c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_checkpoint_*");
    uint64_t need = 0;
    ctmr_ctx* failed = nullptr;
    const int rc = peer_call(c) ? save_peer(c, &since, buf, cap, &need)
                                : save_members(&c, 1, 0, 1, c->next_index, &since, buf, cap, &need, &failed);
    if (rc == CTMR_OK && written) *written = need;
    return rc;
}

int ctmr_checkpoint_apply(ctmr_ctx* c, const uint8_t* const* parts, const uint64_t* part_bytes, uint32_t n_parts) {
    if (!c) return CTMR_E_INVALID;
    if (c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_checkpoint_*");
    if (peer_call(c)) return apply_peer(c, parts, part_bytes, n_parts);
    ctmr_ctx* failed = nullptr;
    return apply_members(&c, 1, parts, part_bytes, n_parts, &c->next_index, &failed);
}

int ctmr_group_checkpoint_size(ctmr_group* g, uint64_t* bytes) {
    return on_group(g, [=](ctmr_ctx** m, uint32_t W, uint64_t* next_index, ctmr_ctx** failed) {
        if (!bytes) return fail(m[0], CTMR_E_INVALID, "bad argument");
        return save_members(m, W, 0, 1, *next_index, nullptr, nullptr, 0, bytes, failed);
    });
}

int ctmr_group_checkpoint_save(ctmr_group* g, uint8_t* buf, uint64_t cap, uint64_t* written) {
    return on_group(g, [=](ctmr_ctx** m, uint32_t W, uint64_t* next_index, ctmr_ctx** failed) {
        if (!buf) return fail(m[0], CTMR_E_INVALID, "bad argument");
        uint64_t need = 0;
        const int rc = save_members(m, W, 0, 1, *next_index, nullptr, buf, cap, &need, failed);
        if (rc == CTMR_OK && written) *written = need;
        return rc;
    });
}

int ctmr_group_checkpoint_load(ctmr_group* g, const uint8_t* const* parts, const uint64_t* part_bytes, uint32_t n_parts) {
    return on_group(g, [=](ctmr_ctx** m, uint32_t W, uint64_t* next_index, ctmr_ctx** failed) {
        return load_members(m, W, parts, part_bytes, n_parts, next_index, failed);
    });
}

int ctmr_group_checkpoint_delta_size(ctmr_group* g, uint64_t since, uint64_t* bytes) {
    return on_group(g, [=](ctmr_ctx** m, uint32_t W, uint64_t* next_index, ctmr_ctx** failed) {
        if (!bytes) return fail(m[0], CTMR_E_INVALID, "bad argument");
        return save_members(m, W, 0, 1, *next_index, &since, nullptr, 0, bytes, failed);
    });
}

int ctmr_group_checkpoint_delta_save(ctmr_group* g, uint64_t since, uint8_t* buf, uint64_t cap, uint64_t* written) {
    return on_group(g, [=](ctmr_ctx** m, uint32_t W, uint64_t* next_index, ctmr_ctx** failed) {
        if (!buf) return fail(m[0], CTMR_E_INVALID, "bad argument");
        uint64_t need = 0;
        const int rc = save_members(m, W, 0, 1, *next_index, &since, buf, cap, &need, failed);
        if (rc == CTMR_OK && written) *written = need;
        return rc;
    });
}

int ctmr_group_checkpoint_apply(ctmr_group* g, const uint8_t* const* parts, const uint64_t* part_bytes, uint32_t n_parts) {
    return on_group(g, [=](ctmr_ctx** m, uint32_t W, uint64_t* next_index, ctmr_ctx** failed) {
        return apply_members(m, W, parts, part_bytes, n_parts, next_index, failed);
    });
}

}  // extern "C"
