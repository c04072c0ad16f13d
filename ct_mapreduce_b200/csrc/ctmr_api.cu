// ctmr_api.cu -- the C ABI of include/ctmr.h: context, issuer registry, the steps of a round of the key exchange and
// run_round, which sequences them for every caller, and the device-resident entry points.
// There is deliberately no CPU implementation of the path in this file or anywhere in the library:
// without a CUDA device ctmr_create fails.
#include "ctmr_ctx.cuh"

thread_local std::string ctmr_host::g_create_error;

namespace ctmr_host {

int fail(ctmr_ctx* ctx, int code, const std::string& msg) {
    if (ctx) ctx->err = msg;
    else g_create_error = msg;
    return code;
}

uint64_t pow2_at_least(uint64_t v) {
    uint64_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

}  // namespace ctmr_host

namespace {

int fe_add_issuer(ctmr_ctx* c, FrontEnd* f, const std::string& der, uint32_t idx);
int fe_clear_issuers(ctmr_ctx* c);

// strings.Split(*ctconfig.IssuerCNFilter, ",") -- no trimming (ct-fetch.go:58)
int build_filter(const ctmr_config* cfg, FilterCfg& f) {
    std::memset(&f, 0, sizeof f);
    f.filter_nonempty = cfg->issuer_cn_filter_len != 0;
    f.log_expired = cfg->log_expired_entries != 0;
    f.flags = cfg->flags;
    if (!f.filter_nonempty) return 0;
    if (cfg->issuer_cn_filter_len > sizeof f.bytes) return -1;
    uint32_t start = 0, np = 0, used = 0;
    for (uint32_t i = 0; i <= cfg->issuer_cn_filter_len; ++i) {
        if (i == cfg->issuer_cn_filter_len || cfg->issuer_cn_filter[i] == ',') {
            if (np >= 32) return -1;
            f.off[np] = (uint16_t)used;
            std::memcpy(f.bytes + used, cfg->issuer_cn_filter + start, i - start);
            used += i - start;
            ++np;
            f.off[np] = (uint16_t)used;
            start = i + 1;
        }
    }
    f.n_prefix = np;
    return 0;
}

SharedLayout make_layout(uint64_t table_slots, uint64_t pair_slots, uint64_t meta_slots, uint32_t max_issuers) {
    SharedLayout l;
    auto take = [&](size_t bytes) {
        const size_t at = l.total;
        l.total += (bytes + 255) & ~(size_t)255;
        return at;
    };
    l.flags = take((kPeerChannels + 1) * kMaxWorld * sizeof(unsigned long long));
    l.reg_counter = take(sizeof(unsigned long long));
    l.status_counts = take(CTMR_ST__COUNT * sizeof(unsigned long long));
    l.issuer_counts = take((size_t)max_issuers * sizeof(unsigned long long));
    l.reg_digests = take((size_t)max_issuers * 32);
    l.reg_mask = pow2_at_least(2ull * max_issuers) - 1;
    l.reg_slots = take((size_t)(l.reg_mask + 1) * sizeof(IssuerRegSlot));
    l.meta = take((size_t)meta_slots * sizeof(MetaSlot));
    l.pairs = take((size_t)pair_slots * sizeof(PairSlot));
    l.table = take((size_t)table_slots * sizeof(KnownSlot));
    return l;
}

}  // namespace
namespace ctmr_host {
int ensure_scratch(ctmr_ctx* c, uint64_t n) {
    if (n <= c->scratch_cap) return CTMR_OK;
    CU(c, cudaDeviceSynchronize());
    c->scratch_cap = 0;  // the old buffers go first, so that peak memory is the new set
    c->keys_scratch.reset(); c->slot_scratch.reset(); c->pair_scratch.reset(); c->bits_scratch.reset(); c->meta_scratch.reset();
    DevBuf<ctmr_key> keys;
    DevBuf<uint32_t> slot, pair, meta;
    DevBuf<uint8_t> bits;
    CU(c, alloc(keys, n)); CU(c, alloc(slot, n)); CU(c, alloc(pair, n)); CU(c, alloc(bits, 2 * n)); CU(c, alloc(meta, 2 * n));
    c->keys_scratch = std::move(keys); c->slot_scratch = std::move(slot); c->pair_scratch = std::move(pair);
    c->bits_scratch = std::move(bits); c->meta_scratch = std::move(meta);
    c->scratch_cap = n;
    return CTMR_OK;
}

static void fill_map_params(ctmr_ctx* c, const ctmr_dev_batch* b, const ctmr_dev_out* o, MapParams& p, uint32_t* fused_slot_of,
                            int parity) {
    std::memset(&p, 0, sizeof p);
    p.blob = b->blob;
    p.blob_bytes = b->blob_bytes;
    p.offsets = b->offsets;
    p.lens = b->lens;
    p.n = b->n;
    p.issuer_idx = b->issuer_idx;
    p.issuer_map = b->issuer_map;
    p.issuer_map_len = b->issuer_map_len;
    p.first_index = b->first_index;
    // NotAfter.Before(now): split now into whole seconds and "has a fractional part"
    int64_t ns = b->now_unix_ns;
    int64_t sec = ns >= 0 ? ns / 1000000000LL : -((-ns + 999999999LL) / 1000000000LL);
    p.now_sec = sec;
    p.now_frac_nonzero = (ns - sec * 1000000000LL) != 0;
    p.one = 1;
    p.status = o->status;
    p.sha256 = (c->flags & CTMR_F_NO_FINGERPRINT) ? nullptr : o->sha256;
    p.exp_hour = o->exp_hour;
    p.serial_off = o->serial_off;
    p.serial_len = o->serial_len;
    p.keys = o->keys;
    if (o->issuer_name_off && o->issuer_name_len && o->crldp_off && o->crldp_len) {
        p.issuer_name_off = o->issuer_name_off;
        p.issuer_name_len = o->issuer_name_len;
        p.crldp_off = o->crldp_off;
        p.crldp_len = o->crldp_len;
    }
    p.status_counts = c->st.status_counts;
    p.filter = c->filter;
    p.route.world = 1;
    if (fused_slot_of && p.keys) {  // K_insert fused into K_map: own keys into the own table, the others to their owners' inboxes
        p.table = c->st.table;
        const uint32_t W = c->px.world;
        if (W > 1) {
            for (uint32_t r = 0; r < W; ++r) p.route.inbox[r] = c->px.inbox[r] + ((uint64_t)parity * W + c->px.rank) * c->px.X;
            p.route.cursor = c->cursors + (size_t)parity * kMaxWorld;
            p.route.rev = c->rev + (uint64_t)parity * W * c->px.X;
            p.route.X = c->px.X;
            p.route.world = W;
            p.route.rank = c->px.rank;
        }
        p.table_mask = c->st.table_mask;
        p.error_flag = c->st.error_flag;
        p.slot_of = fused_slot_of;
    }
}

// K_map over one slice on stream s.  fused_slot_of != NULL: the keys go straight into the table (this rank's) or to
// their owners' inboxes of exchange `parity`, slot -> fused_slot_of.  The fingerprint path of more than 64 entries first
// orders the slice by length into order[0..n), with len_hist (256 counters) as scratch: rounds that may run concurrently
// pass separate histograms.
int map_slice(ctmr_ctx* c, const ctmr_dev_batch* b, const ctmr_dev_out* o, uint32_t* fused_slot_of, int parity, uint32_t* order,
              unsigned int* len_hist, cudaStream_t s) {
    MapParams p;
    fill_map_params(c, b, o, p, fused_slot_of, parity);
    if (b->n > 64 && p.sha256) {  // the light (no-fingerprint) kernel has no lock-step loop to balance
        CU(c, launch_len_order(b->offsets, b->lens, b->n, b->blob_bytes, len_hist, order, c->sm_count, s));
        p.order = order;
    }
    CU(c, launch_map(p, c->sm_count, s));
    return CTMR_OK;
}

int ensure_order(ctmr_ctx* c, uint64_t n) {
    if (n > c->order_cap) {
        CU(c, cudaDeviceSynchronize());  // the old buffer may still be in use
        c->order_cap = 0;
        CU(c, alloc(c->order_scratch, n));
        c->order_cap = n;
    }
    if (!c->len_hist) CU(c, alloc(c->len_hist, 256));
    return CTMR_OK;
}

// what ctmr_process_device needs for a batch of n entries: scratch, the length order, its streams, events and histograms
int ensure_device_path(ctmr_ctx* c, uint64_t n) {
    int rc = ensure_scratch(c, n);
    if (rc) return rc;
    rc = ensure_order(c, n);
    if (rc || c->dp) return rc;
    std::unique_ptr<DevicePipeline> dp(new (std::nothrow) DevicePipeline());
    if (!dp) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    CU(c, create(dp->stream_a));
    CU(c, create(dp->stream_a2));
    CU(c, create(dp->ev_join_a2));
    CU(c, create(dp->stream_b));
    CU(c, create(dp->ev_fork));
    CU(c, create(dp->ev_join_a));
    CU(c, create(dp->ev_join_b));
    for (int k = 0; k < kMaxRounds; ++k) {
        CU(c, create(dp->ev_map0[k], cudaEventDefault));
        CU(c, create(dp->ev_map1[k], cudaEventDefault));
        CU(c, create(dp->ev_red1[k], cudaEventDefault));
        CU(c, create(dp->ev_tok[k]));
        CU(c, alloc(dp->len_hist[k], 256));
    }
    for (Event& e : dp->ev_pulled) CU(c, create(e));
    c->dp = std::move(dp);
    return CTMR_OK;
}

// views of every rank's shared region: the tables K_map / K_resolve address, the flags and histograms of the
// cross-process barrier and all-reduce, the issuer registry in rank 0's region
void attach_views(ctmr_ctx* c, uint8_t* const* bases, uint32_t world, uint32_t rank) {
    const SharedLayout& l = c->lay;
    c->st.peer = PeerTables{};
    c->pf = PeerFlags{};
    for (uint32_t r = 0; r < world; ++r) {
        c->st.peer.table[r] = reinterpret_cast<KnownSlot*>(bases[r] + l.table);
        c->st.peer.pairs[r] = reinterpret_cast<PairSlot*>(bases[r] + l.pairs);
        c->st.peer.meta[r] = reinterpret_cast<MetaSlot*>(bases[r] + l.meta);
        c->pf.flags[r] = reinterpret_cast<unsigned long long*>(bases[r] + l.flags);
        c->pf.issuer_counts[r] = reinterpret_cast<unsigned long long*>(bases[r] + l.issuer_counts);
        c->pf.status_counts[r] = reinterpret_cast<unsigned long long*>(bases[r] + l.status_counts);
    }
    c->st.peer.world = c->pf.world = world;
    c->st.peer.rank = c->pf.rank = rank;
    c->pf.timeout_ns = 60000ull * 1000000ull;
    if (const char* ev = getenv("CTMR_PEER_TIMEOUT_MS")) {
        const unsigned long long ms = strtoull(ev, nullptr, 10);
        if (ms) c->pf.timeout_ns = ms * 1000000ull;
    }
    c->reg.slots = reinterpret_cast<IssuerRegSlot*>(bases[0] + l.reg_slots);
    c->reg.mask = l.reg_mask;
    c->reg.counter = reinterpret_cast<unsigned long long*>(bases[0] + l.reg_counter);
    c->reg.by_index = bases[0] + l.reg_digests;
    c->reg.max_issuers = c->st.max_issuers;
}

size_t exchange_bytes(uint32_t world, uint64_t X) {
    return 4096 + (size_t)kParities * world * X * (sizeof(ctmr_key) + 2);
}

// layout of a rank's exchange area: [counts: kParities x world u64, padded to 4 KiB][inbox][out_wu][out_first]
void attach_exchange(ctmr_ctx* c, uint8_t* const* bases, uint32_t world, uint32_t rank) {
    c->px = PeerExchange{};
    const uint64_t per = (uint64_t)kParities * world * c->X;
    for (uint32_t r = 0; r < world; ++r) {
        c->px.counts[r] = reinterpret_cast<unsigned long long*>(bases[r]);
        c->px.inbox[r] = reinterpret_cast<ctmr_key*>(bases[r] + 4096);
        c->px.out_wu[r] = bases[r] + 4096 + per * sizeof(ctmr_key);
        c->px.out_first[r] = c->px.out_wu[r] + per;
    }
    c->px.X = c->X;
    c->px.world = world;
    c->px.rank = rank;
}

int alloc_exchange(ctmr_ctx* c, uint32_t world) {
    if (c->xchg || world <= 1) return CTMR_OK;
    const uint64_t X = std::max(c->cfg_round_entries ? c->cfg_round_entries : c->stage_entries,
                                c->stage_entries);  // the host pipeline maps stage_entries per round
    const size_t per = (size_t)kParities * world * X;
    DevBuf<uint8_t> xchg;  // set last: a ctx with c->xchg has all of the exchange
    CU(c, alloc(xchg, exchange_bytes(world, X)));
    CU(c, cudaMemsetAsync(xchg, 0, 4096, c->stream));
    CU(c, alloc(c->cursors, (size_t)kParities * kMaxWorld));
    CU(c, cudaMemsetAsync(c->cursors, 0, (size_t)kParities * kMaxWorld * sizeof(unsigned long long), c->stream));
    CU(c, alloc(c->rev, per));
    CU(c, alloc(c->in_slot, per));
    CU(c, alloc(c->in_pair, per));
    CU(c, cudaStreamSynchronize(c->stream));
    c->X = X;
    c->xchg = std::move(xchg);
    return CTMR_OK;
}

// The steps of one round of the exchange on stream s (no-ops on a single GPU); run_round sequences them.
// before K_map: the cursors of this parity to 0
int round_begin(ctmr_ctx* c, int parity, cudaStream_t s) {
    if (c->px.world <= 1) return CTMR_OK;
    CU(c, cudaMemsetAsync(c->cursors + (size_t)parity * kMaxWorld, 0, kMaxWorld * sizeof(unsigned long long), s));
    return CTMR_OK;
}
// after K_map: the region sizes to the owners
int round_publish(ctmr_ctx* c, int parity, cudaStream_t s) {
    if (c->px.world <= 1) return CTMR_OK;
    CU(c, launch_publish_counts(c->px, (uint32_t)parity, c->cursors + (size_t)parity * kMaxWorld, s));
    return CTMR_OK;
}
// owner: the inbox records into the table, then their was_unknown, counts and pair slots, then their first_issuer_hour
int round_owner_insert(ctmr_ctx* c, int parity, uint64_t maxr, cudaStream_t s) {
    if (c->px.world <= 1) return CTMR_OK;
    CU(c, launch_inbox_insert(c->st, c->px, (uint32_t)parity, maxr, c->in_slot, s));
    return CTMR_OK;
}
int round_owner_resolve(ctmr_ctx* c, int parity, uint64_t maxr, cudaStream_t s) {
    if (c->px.world <= 1) return CTMR_OK;
    CU(c, launch_inbox_resolve(c->st, c->px, (uint32_t)parity, maxr, c->in_slot, c->in_pair, s));
    return CTMR_OK;
}
int round_owner_pairs(ctmr_ctx* c, int parity, uint64_t maxr, cudaStream_t s) {
    if (c->px.world <= 1) return CTMR_OK;
    CU(c, launch_inbox_pairs(c->st, c->px, (uint32_t)parity, maxr, c->in_pair, s));
    return CTMR_OK;
}
// the bits of the entries routed away, from their owners
int round_pull(ctmr_ctx* c, int parity, uint64_t maxr, uint8_t* was_unknown, uint8_t* first, cudaStream_t s) {
    if (c->px.world <= 1) return CTMR_OK;
    CU(c, launch_pull_bits(c->px, (uint32_t)parity, c->cursors + (size_t)parity * kMaxWorld,
                           c->rev + (uint64_t)parity * c->px.world * c->px.X, maxr, was_unknown, first, s));
    return CTMR_OK;
}
// the owner passes of a round after every insert of it (own keys and inbox records) has landed, in the order
// lowest-index-wins needs: K_resolve, inbox resolve, K_pairs, inbox pairs
int round_resolve(ctmr_ctx* c, int parity, uint64_t maxr, const ctmr_key* keys, uint64_t cnt, const uint32_t* slot_of,
                  uint32_t* pair_slot, uint8_t* was_unknown, uint8_t* first, cudaStream_t s) {
    CU(c, launch_resolve(c->st, keys, cnt, slot_of, pair_slot, was_unknown, s));
    int rc = round_owner_resolve(c, parity, maxr, s);
    if (rc) return rc;
    CU(c, launch_resolve_pairs(c->st, keys, cnt, pair_slot, was_unknown, first, s));
    return round_owner_pairs(c, parity, maxr, s);
}

// A sync: member r's reduce stream waits for event `ev` of every other member, then meets the other processes at
// `channel` (peer_barrier does nothing unless the ctx is in PEER_IPC mode).
static int sync_members(const RoundMember* m, uint32_t W, uint32_t r, cudaEvent_t RoundMember::*ev, uint32_t channel) {
    ctmr_ctx* c = m[r].c;
    for (uint32_t q = 0; q < W; ++q)
        if (q != r) CU(c, cudaStreamWaitEvent(m[r].reduce_stream, m[q].*ev, 0));
    return peer_barrier(c, channel, m[r].reduce_stream);
}

// One round of the key exchange, the one sequence the host pipeline, the group front end and ctmr_process_device share:
//
//     map + route: round_begin, K_map (a key of a set this GPU owns goes straight into its table, any other key is
//                  appended as a 64-byte record to the OWNER's inbox over NVLink), round_publish
//     -- sync 1: every member's appends of this round have landed --
//     owner passes: inbox insert; K_resolve and K_pairs over the own entries AND the inbox records (round_resolve)
//     -- sync 2: every owner's bits of this round are ready --
//     pull of the bits of the entries routed away [-> string identities: insert, sync 3, read-back]
//
// sync = CUDA events between the members one process drives, a barrier kernel on flags in peer memory between
// processes.  Sync 1, and the chain (or one reduce stream) that orders the owner passes of consecutive rounds, give the
// invariant lowest-index-wins needs: when an entry is resolved, every entry with a lower global index has been inserted.
int run_round(const RoundMember* m, uint32_t W, int parity, uint64_t max_per_region, bool want_meta, ctmr_ctx** failed) {
    // The host issues phase p for every member before phase p + 1 for any member: cudaStreamWaitEvent on an event that
    // has not been recorded yet returns at once and waits for nothing.
    auto each = [&](auto phase) -> int {
        for (uint32_t r = 0; r < W; ++r) {
            *failed = m[r].c;
            CU(m[r].c, cudaSetDevice(m[r].c->device));
            const int rc = phase(m[r], r);
            if (rc) return rc;
        }
        return CTMR_OK;
    };
    int rc = each([&](const RoundMember& x, uint32_t) -> int {  // map + route: own keys into the own table, the others to their owners
        ctmr_ctx* c = x.c;
        if (x.map_start) CU(c, cudaEventRecord(x.map_start, x.map_stream));
        int rc = round_begin(c, parity, x.map_stream);
        if (rc == CTMR_OK && x.db.n) rc = map_slice(c, &x.db, &x.dout, x.slot_of, parity, x.order, x.len_hist, x.map_stream);
        if (rc) return rc;
        if (x.map_end) CU(c, cudaEventRecord(x.map_end, x.map_stream));
        rc = round_publish(c, parity, x.map_stream);
        if (rc) return rc;
        CU(c, cudaEventRecord(x.mapped, x.map_stream));
        return CTMR_OK;
    });
    if (rc) return rc;
    rc = each([&](const RoundMember& x, uint32_t r) -> int {  // sync 1: every member's appends have landed; the owner passes
        ctmr_ctx* c = x.c;
        const cudaStream_t s = x.reduce_stream;
        if (x.map_stream != s) CU(c, cudaStreamWaitEvent(s, x.mapped, 0));
        int rc = sync_members(m, W, r, &RoundMember::mapped, x.ch_map);
        if (rc == CTMR_OK) rc = round_owner_insert(c, parity, max_per_region, s);
        if (rc) return rc;
        if (x.prev_reduced) CU(c, cudaStreamWaitEvent(s, x.prev_reduced, 0));
        rc = round_resolve(c, parity, max_per_region, x.dout.keys, x.db.n, x.slot_of, x.pair_slot, x.dout.was_unknown,
                           x.dout.first_issuer_hour, s);
        if (rc) return rc;
        if (x.reduced) CU(c, cudaEventRecord(x.reduced, s));
        return CTMR_OK;
    });
    if (rc) return rc;
    rc = each([&](const RoundMember& x, uint32_t r) -> int {  // sync 2: every owner has the bits ready; pull, string identities' insert
        ctmr_ctx* c = x.c;
        const cudaStream_t s = x.reduce_stream;
        int rc = sync_members(m, W, r, &RoundMember::reduced, x.ch_resolve);
        if (rc == CTMR_OK) rc = round_pull(c, parity, max_per_region, x.dout.was_unknown, x.dout.first_issuer_hour, s);
        if (rc || !want_meta) return rc;
        if (x.prev_meta_done) CU(c, cudaStreamWaitEvent(s, x.prev_meta_done, 0));
        const ctmr_dev_out& o = x.dout;
        if (x.db.n)  // needs this member's was_unknown bits, i.e. the pull
            CU(c, launch_meta_insert(c->st, x.db.blob, x.db.offsets, o.keys, x.db.n, o.was_unknown, o.issuer_name_off, o.issuer_name_len,
                                     o.crldp_off, o.crldp_len, x.meta_slots, s));
        if (x.meta_done) CU(c, cudaEventRecord(x.meta_done, s));
        return CTMR_OK;
    });
    if (rc == CTMR_OK && want_meta)
        rc = each([&](const RoundMember& x, uint32_t r) -> int {  // sync 3: every member's string identities are in; read-back
            ctmr_ctx* c = x.c;
            int rc = sync_members(m, W, r, &RoundMember::meta_done, x.ch_meta);
            if (rc == CTMR_OK && x.db.n)
                CU(c, launch_meta_resolve(c->st, x.dout.keys, x.db.n, x.meta_slots, x.dout.first_issuer_dn, x.dout.first_crldp,
                                          x.reduce_stream));
            return rc;
        });
    if (rc == CTMR_OK) *failed = nullptr;
    return rc;
}

// Rounds of E entries with a SHORT last round (a quarter of E): what a call exposes at its end is the reduce chain of its
// last round, so that round is kept small; E stays uniform, which is all the global-index formula needs.
uint64_t device_round_entries(uint64_t n, uint32_t rounds) {
    if (rounds >= 4) return (4 * n + 4 * (uint64_t)rounds - 4) / (4 * (uint64_t)rounds - 3);
    return rounds ? (n + rounds - 1) / rounds : n;
}

uint32_t peer_rounds() {
    static const int r = env_int("CTMR_PEER_ROUNDS", (int)CTMR_PEER_ROUNDS);
    return (uint32_t)(r < 1 ? 1 : (r > kMaxRounds ? kMaxRounds : r));
}

int peer_barrier(ctmr_ctx* c, uint32_t channel, cudaStream_t s) {
    if (c->peer_mode != PEER_IPC) return CTMR_OK;
    CU(c, launch_peer_barrier(c->pf, channel, ++c->epoch[channel], c->st.error_flag, s));
    return CTMR_OK;
}
}  // namespace ctmr_host

namespace {
int reduce_on(ctmr_ctx* c, const ctmr_key* keys, uint64_t m, uint32_t* slot_of, uint32_t* pair_slot, uint8_t* was_unknown,
              uint8_t* first, cudaStream_t s, bool already_inserted = false) {
    if (!already_inserted) CU(c, launch_insert(c->st, keys, m, slot_of, s));
    CU(c, launch_resolve(c->st, keys, m, slot_of, pair_slot, was_unknown, s));
    CU(c, launch_resolve_pairs(c->st, keys, m, pair_slot, was_unknown, first, s));
    return CTMR_OK;
}

// the outputs of entries [lo, ..): every array of o offset by lo entries
ctmr_dev_out dev_out_at(const ctmr_dev_out& o, uint64_t lo) {
    auto at = [lo](auto* p, uint64_t per = 1) { return p ? p + lo * per : p; };
    ctmr_dev_out w;
    w.status = at(o.status); w.sha256 = at(o.sha256, 32); w.exp_hour = at(o.exp_hour);
    w.serial_off = at(o.serial_off); w.serial_len = at(o.serial_len); w.keys = at(o.keys);
    w.was_unknown = at(o.was_unknown); w.first_issuer_hour = at(o.first_issuer_hour);
    w.issuer_name_off = at(o.issuer_name_off); w.issuer_name_len = at(o.issuer_name_len);
    w.crldp_off = at(o.crldp_off); w.crldp_len = at(o.crldp_len);
    w.first_issuer_dn = at(o.first_issuer_dn); w.first_crldp = at(o.first_crldp);
    return w;
}


// ------------------------------------------------------------------------------------------------ front end plumbing
uint64_t host_issuer_cert_hash(const std::string& der) {
    const uint32_t len = (uint32_t)der.size();
    uint64_t acc = 0;
    for (uint32_t i = 0; 8u * i < len; ++i) {
        uint64_t w = 0;
        const uint32_t rem = len - 8u * i;
        std::memcpy(&w, der.data() + 8u * i, rem < 8u ? rem : 8u);  // little-endian host (x86-64 / aarch64)
        acc += issuer_cert_word(w, i);
    }
    return issuer_cert_finish(acc, len);
}

// one more certificate in f, c's front end (installed or being built): bytes into the arena, slot into the probe table
int fe_add_issuer(ctmr_ctx* c, FrontEnd* f, const std::string& der, uint32_t idx) {
    if (der.empty()) return CTMR_OK;  // the framing never yields an empty Chain[0]
    if (2 * (f->slots_used + 1) > f->slot_mask + 1)
        return fail(c, CTMR_E_TOO_MANY_ISSUERS, "more distinct Chain[0] certificates than the front end's table holds (raise config.max_issuers)");
    const uint64_t padded = (der.size() + 15) & ~15ull;
    if (f->arena_used + padded > f->arena_cap) {
        uint64_t cap = f->arena_cap ? f->arena_cap * 2 : (64ull << 20);
        while (f->arena_used + padded > cap) cap *= 2;
        DevBuf<uint8_t> bigger;
        CU(c, cudaDeviceSynchronize());
        CU(c, alloc(bigger, cap));
        if (f->arena_used) CU(c, cudaMemcpyAsync(bigger, f->arena, f->arena_used, cudaMemcpyDeviceToDevice, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        f->arena = std::move(bigger);
        f->arena_cap = cap;
    }
    std::string buf = der;
    buf.resize(padded, '\0');
    CU(c, cudaMemcpyAsync(f->arena + f->arena_used, buf.data(), padded, cudaMemcpyHostToDevice, c->stream));
    IssuerCertSlot sl{};
    sl.h = host_issuer_cert_hash(der);
    sl.len = (uint32_t)der.size();
    sl.idx = idx;
    sl.arena_off = f->arena_used;
    f->arena_used += padded;
    uint64_t slot = sl.h & f->slot_mask;
    while (f->slots_host[slot].h != 0) slot = (slot + 1) & f->slot_mask;
    f->slots_host[slot] = sl;
    ++f->slots_used;
    CU(c, cudaMemcpyAsync(f->slots_dev + slot, &sl, sizeof sl, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));  // both sources are locals
    return CTMR_OK;
}

int fe_clear_issuers(ctmr_ctx* c) {
    FrontEnd* f = c->fe.get();
    CU(c, cudaDeviceSynchronize());
    std::fill(f->slots_host.begin(), f->slots_host.end(), IssuerCertSlot{});
    f->slots_used = 0;
    f->arena_used = 0;
    CU(c, cudaMemsetAsync(f->slots_dev, 0, (f->slot_mask + 1) * sizeof(IssuerCertSlot), c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return tiles_clear_fingerprints(c);  // the tiles' fingerprint table follows the mirror
}

int ensure_frontend(ctmr_ctx* c) {
    if (c->fe) return CTMR_OK;
    std::unique_ptr<FrontEnd> f(new (std::nothrow) FrontEnd());
    if (!f) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    const uint64_t E = c->stage_entries;
    uint64_t T = E * 6144ull < (64ull << 20) ? (64ull << 20) : E * 6144ull;  // leaf_input + extra_data characters per chunk
    if (const char* ev = getenv("CTMR_FE_TEXT_CAP")) {  // tests shrink it to reach the multi-chunk and packing paths
        const uint64_t v = strtoull(ev, nullptr, 10);
        if (v >= (1ull << 16)) T = v;
    }
    f->cap_entries = E;
    f->cap_text = T;
    f->cap_decoded = T / 4 * 3 + 32 * E + 256;
    for (FeStage& st : f->stage) {
        CU(c, alloc(st.text, 16 + T + 64));
        CU(c, alloc(st.leaf_off, E)); CU(c, alloc(st.extra_off, E)); CU(c, alloc(st.leaf_len, E)); CU(c, alloc(st.extra_len, E));
        CU(c, alloc(st.h_leaf_off, E)); CU(c, alloc(st.h_extra_off, E)); CU(c, alloc(st.h_leaf_len, E)); CU(c, alloc(st.h_extra_len, E));
        CU(c, create(st.uploaded));
        CU(c, create(st.consumed));
        CU(c, cudaMemsetAsync(st.text, 0, 16 + T + 64, c->stream));
    }
    CU(c, create(f->copy_stream));
    CU(c, alloc(f->pad_size, 2 * E + 1)); CU(c, alloc(f->dec_off, 2 * E + 1)); CU(c, alloc(f->dec_len, 2 * E)); CU(c, alloc(f->str_bad, 2 * E));
    CU(c, alloc(f->decoded, f->cap_decoded));
    // the 16-byte padding between decoded strings is read (never consumed) by K_map's staging
    CU(c, cudaMemsetAsync(f->decoded, 0, f->cap_decoded, c->stream));
    f->scan_temp_bytes = fe_scan_temp_bytes(2 * E + 1);
    CU(c, alloc(f->scan_temp, f->scan_temp_bytes ? f->scan_temp_bytes : 16));
    CU(c, alloc(f->entry_status, E)); CU(c, alloc(f->entry_type, E)); CU(c, alloc(f->leaf_src, E)); CU(c, alloc(f->timestamp, E));
    CU(c, alloc(f->leaf_abs, E)); CU(c, alloc(f->chain_abs, E)); CU(c, alloc(f->tbs_abs, E));
    CU(c, alloc(f->leaf_rel, E)); CU(c, alloc(f->leaf_len_out, E)); CU(c, alloc(f->chain_len, E)); CU(c, alloc(f->tbs_len, E));
    CU(c, alloc(f->issuer_idx, E));
    CU(c, alloc(f->status, E)); CU(c, alloc(f->sha, E * 32)); CU(c, alloc(f->was_unknown, E)); CU(c, alloc(f->first, E));
    CU(c, alloc(f->first_meta, 2 * E));
    CU(c, alloc(f->exp_hour, E)); CU(c, alloc(f->serial_off, E)); CU(c, alloc(f->serial_len, E)); CU(c, alloc(f->spans, 4 * E));
    f->slot_mask = pow2_at_least(4ull * c->st.max_issuers) - 1;
    CU(c, alloc(f->slots_dev, f->slot_mask + 1));
    f->slots_host.assign(f->slot_mask + 1, IssuerCertSlot{});
    f->pending_mask = (1ull << 16) - 1;
    CU(c, alloc(f->pending, f->pending_mask + 1));
    f->unknown_cap = 1u << 14;
    CU(c, alloc(f->unknown_list, f->unknown_cap));
    CU(c, alloc(f->unknown_count, 4));
    CU(c, cudaMemsetAsync(f->slots_dev, 0, (f->slot_mask + 1) * sizeof(IssuerCertSlot), c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    CU(c, create(f->ev0, cudaEventDefault)); CU(c, create(f->ev1, cudaEventDefault)); CU(c, create(f->ev2, cudaEventDefault));
    CU(c, create(f->mapped)); CU(c, create(f->reduced)); CU(c, create(f->meta_done));
    for (const auto& kv : c->issuer_by_der) {  // certificates registered before the front end existed
        int rc = fe_add_issuer(c, f.get(), kv.first, kv.second);
        if (rc) return rc;
    }
    c->fe = std::move(f);
    return CTMR_OK;
}

}  // namespace

namespace ctmr_host {
int frontend_ensure(ctmr_ctx* c) { return ensure_frontend(c); }
}  // namespace ctmr_host

// =================================================================================================
extern "C" {

uint32_t ctmr_abi_version(void) { return CTMR_ABI_VERSION; }

const char* ctmr_last_error(ctmr_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

void* ctmr_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    return p;
}
void ctmr_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

int ctmr_create(const ctmr_config* cfg, ctmr_ctx** out) {
    if (!cfg || !out || cfg->struct_size < sizeof(ctmr_config)) return fail(nullptr, CTMR_E_INVALID, "bad config");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || cfg->device < 0 || cfg->device >= ndev) {
        (void)cudaGetLastError();
        return fail(nullptr, CTMR_E_NO_DEVICE, "no usable CUDA device (libctmr has no CPU fallback)");
    }
    std::unique_ptr<ctmr_ctx> c(new (std::nothrow) ctmr_ctx());  // failures below report through ctmr_last_error(NULL)
    if (!c) return fail(nullptr, CTMR_E_NOMEM, "host allocation failed");
    c->device = cfg->device;
    c->flags = cfg->flags;
    if (build_filter(cfg, c->filter)) return fail(nullptr, CTMR_E_INVALID, "issuerCNFilter too long (max 446 bytes, 32 prefixes)");
    CU(nullptr, cudaSetDevice(c->device));
    cudaDeviceProp prop;
    CU(nullptr, cudaGetDeviceProperties(&prop, c->device));
    if (prop.major != 9 || prop.minor != 0) return fail(nullptr, CTMR_E_NO_DEVICE, "libctmr is built for sm_90a (H100) only");
    c->sm_count = prop.multiProcessorCount;
    CU(nullptr, create(c->stream));
    const uint64_t cap = pow2_at_least(cfg->table_capacity ? cfg->table_capacity : (1ull << 20));
    if (cap > (1ull << 32) - 16) return fail(nullptr, CTMR_E_INVALID, "table_capacity above 2^32 slots");
    c->st.table_mask = cap - 1;
    const uint32_t plog = cfg->pair_capacity_log2 ? cfg->pair_capacity_log2 : 24;
    const uint32_t mlog = cfg->meta_capacity_log2 ? cfg->meta_capacity_log2 : 20;
    if (plog > 32 || mlog > 26) return fail(nullptr, CTMR_E_INVALID, "pair_capacity_log2 above 32 or meta_capacity_log2 above 26");
    c->st.pair_mask = (1ull << plog) - 1;
    c->st.meta_mask = (1ull << mlog) - 1;  // IssuerMetadata string identities: O(issuers x few)
    c->st.max_issuers = cfg->max_issuers ? cfg->max_issuers : 65536;
    // ONE allocation for everything another rank of a group may address (tables, histograms, barrier flags, issuer
    // registry): one CUDA IPC handle exports it; on a single GPU it is simply this ctx's state
    c->lay = make_layout(cap, c->st.pair_mask + 1, c->st.meta_mask + 1, c->st.max_issuers);
    CU(nullptr, alloc(c->shared, c->lay.total));
    CU(nullptr, cudaMemsetAsync(c->shared, 0, c->lay.total, c->stream));
    c->st.table = reinterpret_cast<KnownSlot*>(c->shared + c->lay.table);
    c->st.pairs = reinterpret_cast<PairSlot*>(c->shared + c->lay.pairs);
    c->st.meta = reinterpret_cast<MetaSlot*>(c->shared + c->lay.meta);
    c->st.issuer_counts = reinterpret_cast<unsigned long long*>(c->shared + c->lay.issuer_counts);
    c->st.status_counts = reinterpret_cast<unsigned long long*>(c->shared + c->lay.status_counts);
    CU(nullptr, alloc(c->small, 1));
    CU(nullptr, cudaMemsetAsync(c->small, 0, sizeof(SmallDev), c->stream));
    c->st.slots_used = &c->small->slots_used;
    c->st.error_flag = &c->small->error_flag;
    {
        uint8_t* self[1] = {c->shared};
        attach_views(c.get(), self, 1, 0);  // a single GPU is a group of one
    }
    c->stage_entries = cfg->max_batch_entries ? (cfg->max_batch_entries < kStageEntries ? cfg->max_batch_entries : kStageEntries)
                                              : kStageEntries;
    const uint64_t want_bytes = cfg->max_batch_bytes ? cfg->max_batch_bytes : c->stage_entries * 2048ull;
    c->stage_bytes = want_bytes < kStageBytes ? want_bytes : kStageBytes;
    c->cfg_round_entries = cfg->max_round_entries;
    c->px.world = 1;
    CU(nullptr, cudaStreamSynchronize(c->stream));
    *out = c.release();
    return CTMR_OK;
}

void ctmr_destroy(ctmr_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    delete c;
}

// ------------------------------------------------------------------------------------------------ issuers
// The registry (Issuer.ID digest -> dense index) is a find-or-insert table in the device memory of the group's rank 0,
// reached with system-scope atomics: whichever rank meets an issuer first, every rank gets the same index for it.
// The host keeps memos only (DER -> index, digest -> index, index -> digest), filled from the device.
}  // extern "C"

namespace ctmr_host {

int refresh_digests(ctmr_ctx* c) {
    unsigned long long cnt = 0;
    CU(c, cudaMemcpyAsync(&cnt, c->reg.counter, sizeof cnt, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (cnt > c->reg.max_issuers) cnt = c->reg.max_issuers;
    const size_t have = c->digests.size();
    if (cnt <= have) return CTMR_OK;
    std::vector<uint8_t> rows((cnt - have) * 32);
    CU(c, cudaMemcpyAsync(rows.data(), c->reg.by_index + 32 * have, rows.size(), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    for (size_t i = have; i < cnt; ++i) {
        const uint8_t* row = rows.data() + 32 * (i - have);
        bool zero = true;
        for (int k = 0; k < 32; ++k) zero &= row[k] == 0;
        if (zero) break;  // index handed out by another rank's kernel, digest not written yet: next time
        std::array<uint8_t, 32> a;
        std::memcpy(a.data(), row, 32);
        c->digests.push_back(a);
        c->issuer_by_digest.emplace(std::string(reinterpret_cast<const char*>(row), 32), (uint32_t)i);
    }
    return CTMR_OK;
}

// digest -> dense index; `insert` registers an unknown digest (state written by an earlier process, preloads)
int lookup_digest(ctmr_ctx* c, const uint8_t digest[32], bool insert, uint32_t* idx_out, bool* found) {
    const std::string dk(reinterpret_cast<const char*>(digest), 32);
    *found = false;
    auto it = c->issuer_by_digest.find(dk);
    if (it == c->issuer_by_digest.end()) {
        int rc = refresh_digests(c);
        if (rc) return rc;
        it = c->issuer_by_digest.find(dk);
    }
    if (it != c->issuer_by_digest.end()) {
        *idx_out = it->second;
        *found = true;
        return CTMR_OK;
    }
    if (!insert) return CTMR_OK;
    uint8_t* d_dig = c->small->digest;
    uint32_t* d_idx = &c->small->idx;
    uint32_t idx = CTMR_ISSUER_BAD;
    CU(c, cudaMemcpyAsync(d_dig, digest, 32, cudaMemcpyHostToDevice, c->stream));
    CU(c, launch_issuer_registry(c->reg, d_dig, nullptr, 1, d_idx, c->st.error_flag, c->stream));
    CU(c, cudaMemcpyAsync(&idx, d_idx, 4, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (idx == CTMR_ISSUER_BAD) {
        ctmr_check_device(c, nullptr);  // clears the flag
        return fail(c, CTMR_E_TOO_MANY_ISSUERS, "more distinct issuers than config.max_issuers");
    }
    c->issuer_by_digest.emplace(dk, idx);
    *idx_out = idx;
    *found = true;
    return refresh_digests(c);
}

int upload_issuer_map(ctmr_ctx* c, const uint32_t* dense, uint32_t n) {
    if (n > c->issuer_map_cap) {
        c->issuer_map_cap = 0;
        CU(c, alloc(c->issuer_map_dev, n));
        c->issuer_map_cap = n;
    }
    CU(c, cudaMemcpyAsync(c->issuer_map_dev, dense, n * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return CTMR_OK;
}

}  // namespace ctmr_host

extern "C" {

int ctmr_register_issuers(ctmr_ctx* c, const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint32_t* dense_out) {
    if (!c || (n && (!blob || !offsets || !dense_out))) return fail(c, CTMR_E_INVALID, "bad argument");
    CU(c, cudaSetDevice(c->device));
    std::vector<uint32_t> fresh;  // positions whose DER has not been seen before
    std::vector<std::string> ders(n);
    for (uint32_t k = 0; k < n; ++k) {
        if (offsets[k + 1] < offsets[k]) return fail(c, CTMR_E_INVALID, "issuer offsets not monotonic");
        ders[k].assign(reinterpret_cast<const char*>(blob + offsets[k]), (size_t)(offsets[k + 1] - offsets[k]));
        auto it = c->issuer_by_der.find(ders[k]);
        if (it != c->issuer_by_der.end()) {
            dense_out[k] = it->second;
        } else {
            bool dup = false;
            for (uint32_t f : fresh)
                if (ders[f] == ders[k]) { dup = true; break; }
            if (!dup) fresh.push_back(k);
            dense_out[k] = CTMR_ISSUER_NONE;  // patched below
        }
    }
    if (!fresh.empty()) {
        // only never-seen certificates go to the GPU: parse + SHA-256(SPKI) there, then find-or-insert of the digest
        // in the registry (rank 0's memory); indices and digests come back
        std::vector<uint8_t> packed;
        std::vector<uint64_t> poff(1, 0);
        for (uint32_t f : fresh) {
            packed.insert(packed.end(), ders[f].begin(), ders[f].end());
            poff.push_back(packed.size());
        }
        const uint32_t nf = (uint32_t)fresh.size();
        DevBuf<uint8_t> d_blob, d_dig, d_ok;
        DevBuf<uint64_t> d_off;
        DevBuf<uint32_t> d_idx;
        CU(c, alloc(d_blob, packed.size() + 64));
        CU(c, alloc(d_off, poff.size()));
        CU(c, alloc(d_dig, nf * 32));
        CU(c, alloc(d_ok, nf));
        CU(c, alloc(d_idx, nf));
        CU(c, cudaMemcpyAsync(d_blob, packed.data(), packed.size(), cudaMemcpyHostToDevice, c->stream));
        CU(c, cudaMemcpyAsync(d_off, poff.data(), poff.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
        CU(c, launch_issuer_prepare(d_blob, d_off, nf, d_dig, d_ok, c->stream));
        CU(c, launch_issuer_registry(c->reg, d_dig, d_ok, nf, d_idx, c->st.error_flag, c->stream));
        std::vector<uint8_t> dig(nf * 32), ok(nf);
        std::vector<uint32_t> idx(nf);
        CU(c, cudaMemcpyAsync(dig.data(), d_dig, nf * 32, cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaMemcpyAsync(ok.data(), d_ok, nf, cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaMemcpyAsync(idx.data(), d_idx, nf * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        for (uint32_t i = 0; i < nf; ++i) {
            if (ok[i] && idx[i] == CTMR_ISSUER_BAD) {
                ctmr_check_device(c, nullptr);  // clears the flag
                return fail(c, CTMR_E_TOO_MANY_ISSUERS, "more distinct issuers than config.max_issuers");
            }
            if (ok[i]) c->issuer_by_digest.emplace(std::string(reinterpret_cast<const char*>(dig.data() + 32 * i), 32), idx[i]);
            if (c->fe) {  // first the mirror: a DER it has no room for must not count as registered (a retry fails the same way)
                int rc2 = fe_add_issuer(c, c->fe.get(), ders[fresh[i]], idx[i]);
                if (rc2) return rc2;
            }
            c->issuer_by_der.emplace(ders[fresh[i]], idx[i]);
        }
        for (uint32_t k = 0; k < n; ++k)
            if (dense_out[k] == CTMR_ISSUER_NONE) dense_out[k] = c->issuer_by_der[ders[k]];
        int rc = refresh_digests(c);
        if (rc) return rc;
    }
    return CTMR_OK;
}

int ctmr_issuer_digest(ctmr_ctx* c, uint32_t idx, uint8_t out[32]) {
    if (!c || !out) return fail(c, CTMR_E_INVALID, "bad argument");
    if (idx >= c->digests.size()) {
        CU(c, cudaSetDevice(c->device));
        int rc = refresh_digests(c);  // another rank of the group may have registered it
        if (rc) return rc;
    }
    if (idx >= c->digests.size()) return fail(c, CTMR_E_INVALID, "no such issuer");
    std::memcpy(out, c->digests[idx].data(), 32);
    return CTMR_OK;
}

uint32_t ctmr_issuer_count(ctmr_ctx* c) {
    if (!c) return 0;
    if (cudaSetDevice(c->device) == cudaSuccess) refresh_digests(c);
    return (uint32_t)c->digests.size();
}

// ------------------------------------------------------------------------------------------------ device entry points
int ctmr_map_device(ctmr_ctx* c, const ctmr_dev_batch* b, const ctmr_dev_out* o, void* stream) {
    if (!c || !b || !o) return fail(c, CTMR_E_INVALID, "bad argument");
    if (b->n && (!b->blob || !b->offsets)) return fail(c, CTMR_E_INVALID, "null batch buffers");
    CU(c, cudaSetDevice(c->device));
    int rc = ensure_order(c, b->n);
    if (rc) return rc;
    return map_slice(c, b, o, nullptr, 0, c->order_scratch, c->len_hist, stream ? (cudaStream_t)stream : c->stream);
}

int ctmr_reduce_device(ctmr_ctx* c, const ctmr_key* keys, uint64_t m, uint8_t* was_unknown, uint8_t* first, void* stream) {
    if (!c || (m && !keys)) return fail(c, CTMR_E_INVALID, "bad argument");
    CU(c, cudaSetDevice(c->device));
    int rc = ensure_scratch(c, m);
    if (rc) return rc;
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    return reduce_on(c, keys, m, c->slot_scratch, c->pair_scratch, was_unknown ? was_unknown : c->bits_scratch,
                     first ? first : c->bits_scratch + m, s);
}

int ctmr_process_device(ctmr_ctx* c, const ctmr_dev_batch* b, const ctmr_dev_out* o, void* stream) {
    if (!c || !b || !o) return fail(c, CTMR_E_INVALID, "bad argument");
    if (b->n && (!b->blob || !b->offsets)) return fail(c, CTMR_E_INVALID, "null batch buffers");
    CU(c, cudaSetDevice(c->device));
    int rc = ensure_device_path(c, b->n);
    if (rc) return rc;
    DevicePipeline& dp = *c->dp;
    const bool want_meta = o->first_issuer_dn || o->first_crldp;
    if (want_meta && !(o->issuer_name_off && o->issuer_name_len && o->crldp_off && o->crldp_len))
        return fail(c, CTMR_E_INVALID, "first_issuer_dn / first_crldp need the four span outputs as well");
    cudaStream_t user = stream ? (cudaStream_t)stream : c->stream;
    // The map half is INT-pipe bound and the reduce half is latency/atomic bound: run sub-batch
    // k+1's K_map (stream A) while sub-batch k's insert/resolve/pairs run (stream B).
    // In a multi-process group the call is collective: every rank runs CTMR_PEER_ROUNDS rounds (empty ones included)
    // and meets the others at two barriers per round; round k of rank r carries the global indices
    // first_index + (k * world + r) * E .. , i.e. the rounds are ordered, and inside a round the ranks.
    const uint32_t world = c->st.peer.world, rank = c->st.peer.rank;
    const bool coll = c->peer_mode == PEER_IPC && world > 1;
    if (c->peer_mode == PEER_GROUP && world > 1)
        return fail(c, CTMR_E_INVALID, "members of an in-process group are driven through ctmr_group_process_batch");
    if (want_meta && world > 1) return fail(c, CTMR_E_INVALID, "first_issuer_dn / first_crldp of a group come from the host-buffer call");
    const int nsub = coll ? (int)peer_rounds() : (b->n >= (1u << 21) ? 8 : (b->n >= (1u << 18) ? 2 : 1));
    const uint64_t per_round = device_round_entries(b->n, (uint32_t)nsub);
    if (coll && per_round > c->px.X)
        return fail(c, CTMR_E_BATCH_TOO_LARGE, "entries per round exceed the key-exchange regions: raise config.max_round_entries to ceil(n / ctmr_peer_rounds())");
    ctmr_dev_out all = *o;  // the outputs the rounds write, scratch where the caller asks for none
    if (!all.keys) all.keys = c->keys_scratch;
    if (!all.was_unknown) all.was_unknown = c->bits_scratch;
    if (!all.first_issuer_hour) all.first_issuer_hour = c->bits_scratch + b->n;
    CU(c, cudaEventRecord(dp.ev_fork, user));
    CU(c, cudaStreamWaitEvent(dp.stream_a, dp.ev_fork, 0));
    CU(c, cudaStreamWaitEvent(dp.stream_a2, dp.ev_fork, 0));
    CU(c, cudaStreamWaitEvent(dp.stream_b, dp.ev_fork, 0));
    for (int k = 0; k < nsub; ++k) {
        const uint64_t lo = std::min<uint64_t>(b->n, per_round * k), hi = std::min<uint64_t>(b->n, per_round * (k + 1));
        RoundMember x;
        x.c = c;
        x.db = *b;
        x.db.offsets = b->offsets + lo;
        x.db.lens = b->lens ? b->lens + lo : nullptr;
        x.db.n = hi - lo;
        x.db.issuer_idx = b->issuer_idx ? b->issuer_idx + lo : nullptr;
        x.db.first_index = coll ? b->first_index + ((uint64_t)k * world + rank) * per_round : b->first_index + lo;
        x.dout = dev_out_at(all, lo);
        x.slot_of = c->slot_scratch + lo; x.pair_slot = c->pair_scratch + lo; x.order = c->order_scratch + lo;
        x.len_hist = dp.len_hist[k];
        x.meta_slots = c->meta_scratch + 2 * lo;
        // consecutive K_map launches on alternating streams: the next launch's CTAs fill the SMs the previous one's
        // draining tail leaves idle (a persistent grid ends with its slowest warps)
        x.map_stream = (k & 1) ? dp.stream_a2 : dp.stream_a;
        x.reduce_stream = dp.stream_b;
        x.mapped = dp.ev_tok[k];  // K_map + the published sizes; one reduce stream orders the rounds, so no chain
        x.map_start = dp.ev_map0[k];
        x.map_end = dp.ev_map1[k];  // before the publish: map_ms times K_map alone
        x.ch_map = CH_DEV_MAP;
        x.ch_resolve = x.ch_meta = CH_DEV_RESOLVE;  // sync 3 meets no barrier: a collective call has no string identities
        const int parity = k % (int)kParities;
        if (world > 1 && k >= (int)kParities) CU(c, cudaStreamWaitEvent(x.map_stream, dp.ev_pulled[parity], 0));  // the parity's regions are free again
        ctmr_ctx* failed = nullptr;
        rc = run_round(&x, 1, parity, per_round, want_meta, &failed);
        if (rc) return rc;
        if (world > 1) CU(c, cudaEventRecord(dp.ev_pulled[parity], dp.stream_b));
        CU(c, cudaEventRecord(dp.ev_red1[k], dp.stream_b));
    }
    c->last_sub = nsub;
    CU(c, cudaEventRecord(dp.ev_join_a2, dp.stream_a2));
    CU(c, cudaStreamWaitEvent(user, dp.ev_join_a2, 0));
    CU(c, cudaEventRecord(dp.ev_join_a, dp.stream_a));
    CU(c, cudaEventRecord(dp.ev_join_b, dp.stream_b));
    CU(c, cudaStreamWaitEvent(user, dp.ev_join_a, 0));
    CU(c, cudaStreamWaitEvent(user, dp.ev_join_b, 0));
    return CTMR_OK;
}

uint32_t ctmr_peer_rounds(void) { return peer_rounds(); }
uint64_t ctmr_peer_round_entries(uint64_t n) { return device_round_entries(n, peer_rounds()); }

/* CUDA-event timings of the last ctmr_process_device call (after the caller synchronised):
 * map_ms = first K_map start -> last K_map end, total_ms = first map start -> last reduce end */
int ctmr_profile_last(ctmr_ctx* c, float* map_ms, float* total_ms) {
    if (!c || c->last_sub <= 0) return fail(c, CTMR_E_INVALID, "no ctmr_process_device call to report");
    CU(c, cudaSetDevice(c->device));
    // launches overlap (alternating streams): K_map's time is the span from the first launch's start to the last one's end,
    // during which some K_map CTA is always resident
    float m = 0.f, t = 0.f;
    for (int k = 0; k < c->last_sub; ++k) {
        float d = 0.f;
        CU(c, cudaEventElapsedTime(&d, c->dp->ev_map0[0], c->dp->ev_map1[k]));
        m = d > m ? d : m;
    }
    CU(c, cudaEventElapsedTime(&t, c->dp->ev_map0[0], c->dp->ev_red1[c->last_sub - 1]));
    if (map_ms) *map_ms = m;
    if (total_ms) *total_ms = t;
    return CTMR_OK;
}

int ctmr_read_histogram_device(ctmr_ctx* c, uint64_t* counts_dst, uint32_t n_slots, uint64_t* status_dst, void* stream) {
    if (!c || n_slots > c->st.max_issuers) return fail(c, CTMR_E_INVALID, "bad argument");
    CU(c, cudaSetDevice(c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    if (counts_dst && n_slots)
        CU(c, cudaMemcpyAsync(counts_dst, c->st.issuer_counts, n_slots * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
    if (status_dst)
        CU(c, cudaMemcpyAsync(status_dst, c->st.status_counts, CTMR_ST__COUNT * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
    return CTMR_OK;
}

int ctmr_reset_device(ctmr_ctx* c, void* stream) {
    if (!c) return CTMR_E_INVALID;
    CU(c, cudaSetDevice(c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    // multi-process group: collective.  Nobody may still be inserting into this shard when it is cleared, and nobody
    // may insert into it again before it has been cleared.
    int rc = peer_barrier(c, CH_RESET_A, s);
    if (rc) return rc;
    CU(c, cudaMemsetAsync(c->st.table, 0, (c->st.table_mask + 1) * sizeof(KnownSlot), s));
    CU(c, cudaMemsetAsync(c->st.pairs, 0, (c->st.pair_mask + 1) * sizeof(PairSlot), s));
    CU(c, cudaMemsetAsync(c->st.meta, 0, (c->st.meta_mask + 1) * sizeof(MetaSlot), s));
    CU(c, cudaMemsetAsync(c->st.issuer_counts, 0, c->st.max_issuers * sizeof(unsigned long long), s));
    CU(c, cudaMemsetAsync(c->st.status_counts, 0, CTMR_ST__COUNT * sizeof(unsigned long long), s));
    CU(c, cudaMemsetAsync(&c->small->slots_used, 0, offsetof(SmallDev, cardinality), s));  // slots_used and the error flag
    return peer_barrier(c, CH_RESET_B, s);
}

// Reads AND clears the sticky device-side failure flag: one failed batch does not poison the ctx.
int ctmr_check_device(ctmr_ctx* c, void* stream) {
    if (!c) return CTMR_E_INVALID;
    CU(c, cudaSetDevice(c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    int flag = 0;
    CU(c, cudaMemcpyAsync(&flag, c->st.error_flag, sizeof flag, cudaMemcpyDeviceToHost, s));
    CU(c, cudaStreamSynchronize(s));
    if (!flag) return CTMR_OK;
    CU(c, cudaMemsetAsync(c->st.error_flag, 0, sizeof(int), s));
    CU(c, cudaStreamSynchronize(s));
    switch (flag) {
    case CTMR_E_TABLE_FULL: return fail(c, flag, "known-certificate table is full; raise config.table_capacity");
    case CTMR_E_PAIR_TABLE_FULL: return fail(c, flag, "(issuer, expDate) table is full; raise config.pair_capacity_log2");
    case CTMR_E_META_TABLE_FULL: return fail(c, flag, "IssuerMetadata string-identity table is full; raise config.meta_capacity_log2");
    case CTMR_E_TOO_MANY_ISSUERS: return fail(c, flag, "more distinct issuers than config.max_issuers");
    case CTMR_E_PEER_TIMEOUT: return fail(c, flag, "a rank of the group did not reach a barrier in time (peer failed, or the collective calls diverged; CTMR_PEER_TIMEOUT_MS)");
    default: return fail(c, CTMR_E_CUDA, "device-side failure flag set");
    }
}

// ------------------------------------------------------------------------------------------------ warm start / checkpoint
}  // extern "C"

namespace ctmr_host {
// Seeds keys with the indices first_index .. first_index + n - 1 (the caller keeps them below every later batch
// index).  Inserts go to the set's owner, so in a group any member can run it; not collective: the group is quiescent.
int preload_impl(ctmr_ctx* c, int64_t exp_hour, const uint8_t digest[32], const uint8_t* serial_blob, const uint64_t* serial_offsets,
                 uint64_t n, uint64_t first_index) {
    if (exp_hour > INT32_MAX || exp_hour < INT32_MIN) return fail(c, CTMR_E_INVALID, "exp_hour out of range");
    CU(c, cudaSetDevice(c->device));
    uint32_t issuer = 0;
    bool found = false;
    int rc = lookup_digest(c, digest, true, &issuer, &found);  // the issuer may be unknown so far (state written by an earlier process)
    if (rc) return rc;
    if (!n) return CTMR_OK;
    if (c->st.peer.world > 1) {
        const uint32_t owner = key_owner((int32_t)exp_hour, issuer, c->st.peer.world);
        if (owner != c->st.peer.rank)
            return fail(c, CTMR_E_INVALID, "this set is owned by rank " + std::to_string(owner) + " of the group: preload it there");
    }
    std::vector<ctmr_key> keys(n);
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t len = serial_offsets[i + 1] - serial_offsets[i];
        if (serial_offsets[i + 1] < serial_offsets[i] || len == 0 || len > CTMR_MAX_SERIAL)
            return fail(c, CTMR_E_INVALID, "preloaded serial empty or longer than CTMR_MAX_SERIAL");
        std::memset(&keys[i], 0, sizeof(ctmr_key));
        keys[i].index = first_index + i;
        keys[i].exp_hour = (int32_t)exp_hour;
        keys[i].issuer = issuer;
        keys[i].serial_len = (uint8_t)len;
        std::memcpy(keys[i].serial, serial_blob + serial_offsets[i], len);
        keys[i].valid = 1;
    }
    rc = ensure_scratch(c, n);
    if (rc) return rc;
    CU(c, cudaMemcpyAsync(c->keys_scratch, keys.data(), n * sizeof(ctmr_key), cudaMemcpyHostToDevice, c->stream));
    rc = reduce_on(c, c->keys_scratch, n, c->slot_scratch, c->pair_scratch, c->bits_scratch, c->bits_scratch + n, c->stream);
    if (rc) return rc;
    CU(c, cudaStreamSynchronize(c->stream));
    return ctmr_check_device(c, nullptr);
}
}  // namespace ctmr_host

extern "C" {

int ctmr_preload_known(ctmr_ctx* c, int64_t exp_hour, const uint8_t digest[32], const uint8_t* serial_blob,
                       const uint64_t* serial_offsets, uint64_t n) {
    if (!c || !digest || (n && (!serial_blob || !serial_offsets))) return fail(c, CTMR_E_INVALID, "bad argument");
    if (c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_preload_known");
    // key records with the indices next_index .. BELOW every later batch index: preloaded keys always win "first seen"
    int rc = preload_impl(c, exp_hour, digest, serial_blob, serial_offsets, n, c->next_index);
    if (rc == CTMR_OK) c->next_index += n;
    return rc;
}

}  // extern "C"

namespace ctmr_host {

// one shard's tables and histograms, in a fixed order (device <-> host)
uint64_t snap_shard_bytes(ctmr_ctx* c) {
    return (c->st.table_mask + 1) * sizeof(KnownSlot) + (c->st.pair_mask + 1) * sizeof(PairSlot) + (c->st.meta_mask + 1) * sizeof(MetaSlot) +
           c->st.max_issuers * sizeof(uint64_t) + CTMR_ST__COUNT * sizeof(uint64_t);
}

int snap_shard_save(ctmr_ctx* c, uint8_t* p) {
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaDeviceSynchronize());
    const uint64_t t = (c->st.table_mask + 1) * sizeof(KnownSlot), pr = (c->st.pair_mask + 1) * sizeof(PairSlot),
                   m = (c->st.meta_mask + 1) * sizeof(MetaSlot), ic = c->st.max_issuers * sizeof(uint64_t);
    CU(c, cudaMemcpy(p, c->st.table, t, cudaMemcpyDeviceToHost)); p += t;
    CU(c, cudaMemcpy(p, c->st.pairs, pr, cudaMemcpyDeviceToHost)); p += pr;
    CU(c, cudaMemcpy(p, c->st.meta, m, cudaMemcpyDeviceToHost)); p += m;
    CU(c, cudaMemcpy(p, c->st.issuer_counts, ic, cudaMemcpyDeviceToHost)); p += ic;
    CU(c, cudaMemcpy(p, c->st.status_counts, CTMR_ST__COUNT * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    return CTMR_OK;
}

int snap_shard_load(ctmr_ctx* c, const uint8_t* p) {
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaDeviceSynchronize());
    const uint64_t t = (c->st.table_mask + 1) * sizeof(KnownSlot), pr = (c->st.pair_mask + 1) * sizeof(PairSlot),
                   m = (c->st.meta_mask + 1) * sizeof(MetaSlot), ic = c->st.max_issuers * sizeof(uint64_t);
    CU(c, cudaMemcpy(c->st.table, p, t, cudaMemcpyHostToDevice)); p += t;
    CU(c, cudaMemcpy(c->st.pairs, p, pr, cudaMemcpyHostToDevice)); p += pr;
    CU(c, cudaMemcpy(c->st.meta, p, m, cudaMemcpyHostToDevice)); p += m;
    CU(c, cudaMemcpy(c->st.issuer_counts, p, ic, cudaMemcpyHostToDevice)); p += ic;
    CU(c, cudaMemcpy(c->st.status_counts, p, CTMR_ST__COUNT * sizeof(uint64_t), cudaMemcpyHostToDevice));
    // host memos: the DER memo is rebuilt lazily, the digest memos come back from the device registry
    c->digests.clear();
    c->issuer_by_digest.clear();
    c->issuer_by_der.clear();
    if (c->fe) return fe_clear_issuers(c);
    return CTMR_OK;
}

// the device registry (rank 0's region) again, digest i at index i: cleared, then filled by ONE launch of the
// find-or-insert kernel, which takes a call's digests in order
int snap_registry_alloc(ctmr_ctx* c, uint64_t n, RegistryUpload& u) {
    CU(c, cudaSetDevice(c->device));
    if (n) {
        CU(c, alloc(u.digests, n * 32));
        CU(c, alloc(u.idx, n));
    }
    return CTMR_OK;
}

int snap_registry_restore(ctmr_ctx* c, const uint8_t* digests, uint64_t n, const RegistryUpload& u) {
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaMemsetAsync(c->reg.slots, 0, (c->reg.mask + 1) * sizeof(IssuerRegSlot), c->stream));
    CU(c, cudaMemsetAsync(c->reg.by_index, 0, (size_t)c->reg.max_issuers * 32, c->stream));
    CU(c, cudaMemsetAsync(c->reg.counter, 0, sizeof(unsigned long long), c->stream));
    if (n) {
        CU(c, cudaMemcpyAsync(u.digests, digests, n * 32, cudaMemcpyHostToDevice, c->stream));
        CU(c, launch_issuer_registry(c->reg, u.digests, nullptr, (uint32_t)n, u.idx, c->st.error_flag, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
    }
    int rc = refresh_digests(c);
    if (rc) return rc;
    if (c->digests.size() != n) return fail(c, CTMR_E_INVALID, "snapshot holds duplicate issuer digests");
    return ctmr_check_device(c, nullptr);
}

}  // namespace ctmr_host

namespace {
struct SnapHeader {
    char magic[8];  // "CTMRSNP3"
    uint64_t table_slots, pair_slots, meta_slots, max_issuers, n_issuers, next_index;
};
}  // namespace

extern "C" {

int ctmr_snapshot_size(ctmr_ctx* c, uint64_t* bytes) {
    if (!c || !bytes) return fail(c, CTMR_E_INVALID, "bad argument");
    if (c->st.peer.world > 1) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_snapshot_* (the shards share one issuer registry)");
    CU(c, cudaSetDevice(c->device));
    int rc = refresh_digests(c);
    if (rc) return rc;
    *bytes = sizeof(SnapHeader) + snap_shard_bytes(c) + c->digests.size() * 32;
    return CTMR_OK;
}

int ctmr_snapshot_save(ctmr_ctx* c, uint8_t* buf, uint64_t cap, uint64_t* written) {
    uint64_t need = 0;
    int rc = ctmr_snapshot_size(c, &need);
    if (rc) return rc;
    if (!buf || cap < need) return fail(c, CTMR_E_INVALID, "snapshot buffer too small");
    SnapHeader h{};
    std::memcpy(h.magic, "CTMRSNP3", 8);
    h.table_slots = c->st.table_mask + 1;
    h.pair_slots = c->st.pair_mask + 1;
    h.meta_slots = c->st.meta_mask + 1;
    h.max_issuers = c->st.max_issuers;
    h.n_issuers = c->digests.size();
    h.next_index = c->next_index;
    uint8_t* p = buf;
    std::memcpy(p, &h, sizeof h); p += sizeof h;
    rc = snap_shard_save(c, p);
    if (rc) return rc;
    p += snap_shard_bytes(c);
    for (const auto& d : c->digests) { std::memcpy(p, d.data(), 32); p += 32; }
    if (written) *written = (uint64_t)(p - buf);
    return CTMR_OK;
}

int ctmr_snapshot_load(ctmr_ctx* c, const uint8_t* buf, uint64_t bytes) {
    if (!c || !buf || bytes < sizeof(SnapHeader)) return fail(c, CTMR_E_INVALID, "bad snapshot");
    SnapHeader h;
    std::memcpy(&h, buf, sizeof h);
    if (std::memcmp(h.magic, "CTMRSNP3", 8) != 0) return fail(c, CTMR_E_INVALID, "not a ctmr snapshot");
    if (h.table_slots != c->st.table_mask + 1 || h.pair_slots != c->st.pair_mask + 1 || h.meta_slots != c->st.meta_mask + 1 ||
        h.max_issuers != c->st.max_issuers)
        return fail(c, CTMR_E_INVALID, "snapshot was taken with different capacities (table / pairs / max_issuers)");
    if (bytes < sizeof h + snap_shard_bytes(c) + h.n_issuers * 32 || h.n_issuers > h.max_issuers) return fail(c, CTMR_E_INVALID, "truncated snapshot");
    if (c->st.peer.world > 1) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_snapshot_*");
    RegistryUpload u;
    int rc = snap_registry_alloc(c, h.n_issuers, u);
    if (rc) return rc;
    rc = snap_shard_load(c, buf + sizeof h);
    if (rc) return rc;
    c->next_index = h.next_index;
    return snap_registry_restore(c, buf + sizeof h + snap_shard_bytes(c), h.n_issuers, u);
}

// ------------------------------------------------------------------------------------------------ tooling
int ctmr_sha256_ceiling_device(ctmr_ctx* c, uint32_t iters, uint32_t rolled, uint32_t ctas_per_sm, float* ms_out,
                               uint64_t* blocks_out) {
    if (!c || !iters || !ctas_per_sm || ctas_per_sm > 8) return fail(c, CTMR_E_INVALID, "bad argument");
    CU(c, cudaSetDevice(c->device));
    Event e0, e1;
    CU(c, create(e0, cudaEventDefault));
    CU(c, create(e1, cudaEventDefault));
    uint32_t* sink = &c->small->sha_sink;
    CU(c, launch_sha_ceiling(iters / 8 + 1, (int)rolled, (int)ctas_per_sm, c->sm_count, sink, c->stream));  // warm-up
    CU(c, cudaEventRecord(e0, c->stream));
    CU(c, launch_sha_ceiling(iters, (int)rolled, (int)ctas_per_sm, c->sm_count, sink, c->stream));
    CU(c, cudaEventRecord(e1, c->stream));
    CU(c, cudaEventSynchronize(e1));
    float ms = 0.f;
    CU(c, cudaEventElapsedTime(&ms, e0, e1));
    if (ms_out) *ms_out = ms;
    if (blocks_out) *blocks_out = (uint64_t)c->sm_count * ctas_per_sm * 256ull * iters;
    return CTMR_OK;
}

// ------------------------------------------------------------------------------------------------ read side
int ctmr_issuer_counts(ctmr_ctx* c, uint8_t* digests, uint64_t* counts, size_t* n) {
    if (!c || !n) return fail(c, CTMR_E_INVALID, "bad argument");
    CU(c, cudaSetDevice(c->device));
    {
        int rc0 = refresh_digests(c);  // issuers another rank of the group registered count too (with 0 here)
        if (rc0) return rc0;
    }
    const size_t have = c->digests.size(), cap = *n;
    const size_t take = have < cap ? have : cap;
    if (take) {
        if (counts) {
            CU(c, cudaMemcpyAsync(counts, c->st.issuer_counts, take * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
            CU(c, cudaStreamSynchronize(c->stream));
        }
        if (digests)
            for (size_t i = 0; i < take; ++i) std::memcpy(digests + 32 * i, c->digests[i].data(), 32);
    }
    *n = take;
    return CTMR_OK;
}

int ctmr_set_cardinality(ctmr_ctx* c, int64_t exp_hour, const uint8_t digest[32], uint64_t* out) {
    if (!c || !digest || !out) return fail(c, CTMR_E_INVALID, "bad argument");
    CU(c, cudaSetDevice(c->device));
    *out = 0;
    uint32_t issuer = 0;
    bool found = false;
    int rc = lookup_digest(c, digest, false, &issuer, &found);
    if (rc) return rc;
    if (!found || exp_hour > INT32_MAX || exp_hour < INT32_MIN) return CTMR_OK;
    // one probe of the set's (issuer, hour) slot at its owner -- which may be another GPU of the group
    CU(c, launch_cardinality(c->st, (int32_t)exp_hour, issuer, &c->small->cardinality, c->stream));
    unsigned long long v = 0;
    CU(c, cudaMemcpyAsync(&v, &c->small->cardinality, sizeof v, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    *out = v;
    return CTMR_OK;
}

int ctmr_status_counters(ctmr_ctx* c, uint64_t out[CTMR_ST__COUNT]) {
    if (!c || !out) return fail(c, CTMR_E_INVALID, "bad argument");
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaMemcpyAsync(out, c->st.status_counts, CTMR_ST__COUNT * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return CTMR_OK;
}

int ctmr_table_stats(ctmr_ctx* c, uint64_t* used, uint64_t* capacity) {
    if (!c) return CTMR_E_INVALID;
    CU(c, cudaSetDevice(c->device));
    unsigned long long u = 0;
    CU(c, cudaMemsetAsync(&c->small->table_count, 0, sizeof(unsigned long long), c->stream));
    CU(c, launch_table_count(c->st, &c->small->table_count, c->sm_count, c->stream));
    CU(c, cudaMemcpyAsync(&u, &c->small->table_count, sizeof u, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (used) *used = u;
    if (capacity) *capacity = c->st.table_mask + 1;
    return CTMR_OK;
}

// Redis TTLs firing (SURVEY §8(f)-4): every set "serials::<expDate>::<issuer>" carries EXPIREAT(expDate)
// (storage/knowncertificates.go:44-47,98-104), so at `now` the sets with expDate <= now no longer exist.
int ctmr_evict_expired(ctmr_ctx* c, int64_t now_unix_sec, uint64_t* evicted_out) {
    if (!c) return CTMR_E_INVALID;
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaDeviceSynchronize());
    unsigned long long counters[2] = {0, 0};
    unsigned long long* dev = c->small->evict;  // live, expired, compaction cursor
    // the count pass takes the expired keys off the per-issuer counts: a copy puts them back if the call cannot go on
    std::vector<unsigned long long> counts_before(c->st.max_issuers);
    CU(c, cudaMemcpyAsync(counts_before.data(), c->st.issuer_counts, counts_before.size() * sizeof(unsigned long long),
                          cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaMemsetAsync(dev, 0, 3 * sizeof(unsigned long long), c->stream));
    CU(c, launch_evict_count(c->st, now_unix_sec, dev, c->sm_count, c->stream));
    CU(c, cudaMemcpyAsync(counters, dev, sizeof counters, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (evicted_out) *evicted_out = counters[1];
    if (counters[1] == 0) return CTMR_OK;
    // open addressing with linear probing: taking slots out would cut probe chains, so the survivors are
    // compacted aside, the table is cleared and they are inserted again (first-seen indices preserved)
    DevBuf<KnownSlot> keep;
    if (counters[0] && alloc(keep, counters[0]) != cudaSuccess) {
        CU(c, cudaMemcpy(c->st.issuer_counts, counts_before.data(), counts_before.size() * sizeof(unsigned long long),
                         cudaMemcpyHostToDevice));
        return fail(c, CTMR_E_NOMEM, "ctmr_evict_expired: no device memory for the surviving keys");
    }
    CU(c, launch_evict_pairs(c->st, now_unix_sec, c->sm_count, c->stream));  // the expired sets' cardinalities are 0 again
    if (counters[0]) CU(c, launch_evict_compact(c->st, now_unix_sec, keep, dev + 2, c->sm_count, c->stream));
    CU(c, cudaMemsetAsync(c->st.table, 0, (c->st.table_mask + 1) * sizeof(KnownSlot), c->stream));
    CU(c, launch_evict_reinsert(c->st, keep, counters[0], c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return ctmr_check_device(c, nullptr);
}

int ctmr_frontend_profile_last(ctmr_ctx* c, float* frontend_ms, float* path_ms, uint64_t* frontend_launches) {
    if (!c || !c->fe) return fail(c, CTMR_E_INVALID, "no ctmr_process_raw / ctmr_process_tiles call to report");
    if (frontend_ms) *frontend_ms = c->fe->fe_ms;
    if (path_ms) *path_ms = c->fe->path_ms;
    if (frontend_launches) *frontend_launches = c->fe->launches;
    return CTMR_OK;
}

}  // extern "C"
