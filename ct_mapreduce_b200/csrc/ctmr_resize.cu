// ctmr_resize.cu -- the tables of a ctx or a group in other sizes, on the device (include/ctmr.h "resize"), and their
// occupancy.
//
// A ctx's tables live at the end of its one shared region (make_layout), after the barrier flags, the histograms and the
// issuer registry, whose offsets depend on max_issuers alone.  A resize builds a new region for every member first: the
// prefix before the tables is copied byte for byte, the per-issuer counts are rebuilt from the keys (as a checkpoint load
// rebuilds them), and one rehash pass per table inserts the records of the current epoch into the new tables.  Only when
// every member's rehash succeeded are the regions swapped and every member's views attached again; until then the old
// regions are untouched, and a failure frees the new ones.
#include "ctmr_ctx.cuh"

namespace {

// one member's new region and its shape, built beside the old one
struct Reshape {
    int device = 0;
    SharedLayout lay{};
    DevBuf<uint8_t> region;
    uint64_t table_mask = 0, pair_mask = 0, meta_mask = 0;
    ~Reshape() {  // a region that was not swapped in is released on its own device
        if (region) {
            cudaSetDevice(device);
            region.reset();
        }
    }
};

const char* full_text(int flag) {
    switch (flag) {
    case CTMR_E_TABLE_FULL: return "ctmr_resize: the known-certificate table of the new size does not hold its records";
    case CTMR_E_PAIR_TABLE_FULL: return "ctmr_resize: the (issuer, expDate) table of the new size does not hold its records";
    case CTMR_E_META_TABLE_FULL: return "ctmr_resize: the string-identity table of the new size does not hold its records";
    default: return "ctmr_resize: the rehash failed";
    }
}

// The new region of member c: allocated, its prefix copied, its tables filled by the rehash (queued on c's stream).
int build_region(ctmr_ctx* c, Reshape& x) {
    x.device = c->device;
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaDeviceSynchronize());  // nothing of an earlier call still runs against the old tables
    x.lay = make_layout(x.table_mask + 1, x.pair_mask + 1, x.meta_mask + 1, c->st.max_issuers);
    if (alloc(x.region, x.lay.total) != cudaSuccess) {
        (void)cudaGetLastError();  // a failed allocation must not surface as the error of a later launch
        return fail(c, CTMR_E_NOMEM,
                    "ctmr_resize: no device memory for the new tables beside the old ones (" + std::to_string(x.lay.total) +
                        " bytes); move the state through ctmr_checkpoint_save / ctmr_checkpoint_load instead");
    }
    uint8_t* nb = x.region;
    CU(c, cudaMemcpyAsync(nb, c->shared, x.lay.meta, cudaMemcpyDeviceToDevice, c->stream));  // flags, counters, registry
    CU(c, cudaMemsetAsync(nb + x.lay.meta, 0, x.lay.total - x.lay.meta, c->stream));
    CU(c, cudaMemsetAsync(nb + x.lay.issuer_counts, 0, (size_t)c->st.max_issuers * sizeof(unsigned long long), c->stream));
    CU(c, cudaMemsetAsync(&c->small->resize_error, 0, sizeof(int), c->stream));
    DeviceState to = c->st;
    to.table = reinterpret_cast<KnownSlot*>(nb + x.lay.table);
    to.pairs = reinterpret_cast<PairSlot*>(nb + x.lay.pairs);
    to.meta = reinterpret_cast<MetaSlot*>(nb + x.lay.meta);
    to.table_mask = x.table_mask;
    to.pair_mask = x.pair_mask;
    to.meta_mask = x.meta_mask;
    to.issuer_counts = reinterpret_cast<unsigned long long*>(nb + x.lay.issuer_counts);
    to.error_flag = &c->small->resize_error;
    CU(c, launch_rehash(c->st.table, c->st.table_mask + 1, c->st.epoch, to, c->sm_count, c->stream));
    CU(c, launch_rehash(c->st.pairs, c->st.pair_mask + 1, c->st.epoch, to, c->sm_count, c->stream));
    CU(c, launch_rehash(c->st.meta, c->st.meta_mask + 1, c->st.epoch, to, c->sm_count, c->stream));
    return CTMR_OK;
}

// the rehash of member c finished: CTMR_OK, or the *_TABLE_FULL of the table that did not hold its records
int region_done(ctmr_ctx* c) {
    CU(c, cudaSetDevice(c->device));
    int flag = 0;
    CU(c, cudaMemcpyAsync(&flag, &c->small->resize_error, sizeof flag, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return flag ? fail(c, flag, full_text(flag)) : CTMR_OK;
}

int resize_members(ctmr_ctx** m, uint32_t W, uint64_t*, ctmr_ctx** failed, uint64_t table_capacity, uint32_t pair_log2, uint32_t meta_log2) {
    *failed = m[0];
    // ctmr_create's limits
    if (table_capacity > (1ull << 32) || (table_capacity && pow2_at_least(table_capacity) > (1ull << 32) - 16))
        return fail(m[0], CTMR_E_INVALID, "table_capacity above 2^32 slots");
    if (pair_log2 > 32 || meta_log2 > 26) return fail(m[0], CTMR_E_INVALID, "pair_capacity_log2 above 32 or meta_capacity_log2 above 26");
    for (uint32_t r = 0; r < W; ++r)
        if (m[r]->peer_mode == PEER_IPC || m[r]->ipc_exported) {
            *failed = m[r];
            return fail(m[r], CTMR_E_INVALID,
                        "ctmr_resize: the tables are exported to peer ranks (ctmr_peer_export); resize before exporting, or "
                        "move the state through ctmr_checkpoint_save / ctmr_checkpoint_load");
        }
    std::vector<Reshape> nx(W);
    for (uint32_t r = 0; r < W; ++r) {
        ctmr_ctx* c = m[r];
        nx[r].table_mask = table_capacity ? pow2_at_least(table_capacity) - 1 : c->st.table_mask;
        nx[r].pair_mask = pair_log2 ? (1ull << pair_log2) - 1 : c->st.pair_mask;
        nx[r].meta_mask = meta_log2 ? (1ull << meta_log2) - 1 : c->st.meta_mask;
    }
    // every member's new region before any old one goes: the peak is old plus new for every member of a device
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        const int rc = build_region(m[r], nx[r]);
        if (rc) {  // no rehash may outlive the region it writes
            for (uint32_t q = 0; q <= r; ++q) {
                const cudaStream_t s = m[q]->stream;
                drain_streams(m[q], &s, 1);
            }
            return rc;
        }
    }
    int rc = CTMR_OK;
    for (uint32_t r = 0; r < W; ++r) {  // every member's rehash ends before a failure frees any new region
        const int rr = region_done(m[r]);
        if (rr && rc == CTMR_OK) {
            rc = rr;
            *failed = m[r];
        }
    }
    if (rc) return rc;
    uint8_t* bases[kMaxWorld] = {};
    for (uint32_t r = 0; r < W; ++r) {
        ctmr_ctx* c = m[r];
        cudaSetDevice(c->device);
        c->shared = std::move(nx[r].region);  // the old region goes
        c->lay = nx[r].lay;
        c->st.table_mask = nx[r].table_mask;
        c->st.pair_mask = nx[r].pair_mask;
        c->st.meta_mask = nx[r].meta_mask;
        point_at_region(c);
        bases[r] = c->shared;
    }
    for (uint32_t r = 0; r < W; ++r) attach_views(m[r], bases, W, r);
    *failed = nullptr;
    return CTMR_OK;
}

// used and capacity of the known-certificate, pair and string-identity tables, summed over the members
int occupancy_members(ctmr_ctx** m, uint32_t W, uint64_t*, ctmr_ctx** failed, uint64_t* used, uint64_t* capacity) {
    uint64_t u[3] = {0, 0, 0}, cp[3] = {0, 0, 0};
    for (uint32_t r = 0; r < W; ++r) {
        ctmr_ctx* c = m[r];
        *failed = c;
        CU(c, cudaSetDevice(c->device));
        unsigned long long* dev = c->small->occupancy;
        unsigned long long v[3] = {0, 0, 0};
        CU(c, cudaMemsetAsync(dev, 0, sizeof v, c->stream));
        CU(c, launch_live_count(c->st.table, c->st.table_mask + 1, c->st.epoch, dev, c->sm_count, c->stream));
        CU(c, launch_live_count(c->st.pairs, c->st.pair_mask + 1, c->st.epoch, dev + 1, c->sm_count, c->stream));
        CU(c, launch_live_count(c->st.meta, c->st.meta_mask + 1, c->st.epoch, dev + 2, c->sm_count, c->stream));
        CU(c, cudaMemcpyAsync(v, dev, sizeof v, cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        const uint64_t slots[3] = {c->st.table_mask + 1, c->st.pair_mask + 1, c->st.meta_mask + 1};
        for (int k = 0; k < 3; ++k) {
            u[k] += v[k];
            cp[k] += slots[k];
        }
    }
    for (int k = 0; k < 3; ++k) {
        if (used) used[k] = u[k];
        if (capacity) capacity[k] = cp[k];
    }
    *failed = nullptr;
    return CTMR_OK;
}

}  // namespace

extern "C" {

int ctmr_resize(ctmr_ctx* c, uint64_t table_capacity, uint32_t pair_capacity_log2, uint32_t meta_capacity_log2) {
    if (c && c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_resize");
    return on_ctx(c, resize_members, table_capacity, pair_capacity_log2, meta_capacity_log2);
}
int ctmr_group_resize(ctmr_group* g, uint64_t table_capacity, uint32_t pair_capacity_log2, uint32_t meta_capacity_log2) {
    return on_group(g, resize_members, table_capacity, pair_capacity_log2, meta_capacity_log2);
}
int ctmr_table_occupancy(ctmr_ctx* c, uint64_t used[3], uint64_t capacity[3]) { return on_ctx(c, occupancy_members, used, capacity); }
int ctmr_group_table_occupancy(ctmr_group* g, uint64_t used[3], uint64_t capacity[3]) {
    return on_group(g, occupancy_members, used, capacity);
}

}  // extern "C"
