// ctmr_pipeline.cu -- the host-buffer batch of include/ctmr.h on one GPU, on a group of GPUs driven by one process
// (ctmr_group_*: what a Go host calls), and on one GPU of a multi-process group (ctmr_peer_*: one process per GPU); and
// the handles of those groups: a group's create, destroy and accessors, a rank's export and attach.  The table calls of
// a group share their bodies with a ctx's, in ctmr_api.cu.
//
// One pipeline serves all three.  A batch is cut into ROUNDS; in a round every member GPU takes one slice of at
// most `stage_entries` entries and runs, on the stream of the round's stage (three stages rotate, so H2D, kernels
// and D2H of consecutive rounds overlap):
//
//     H2D slice -> one round of the key exchange (run_round, ctmr_api.cu: K_map with key routing, sync 1, owner
//                  passes, sync 2, pull [, string identities]) -> D2H of the requested outputs [-> PEM]
//
// The stage index is the round's exchange parity and picks its barrier channels.  Rounds are ordered by a per-member
// chain (the owner passes of round k wait for those of round k-1), which with sync 1 gives the invariant the
// lowest-index-wins rule needs: when an entry is resolved, every entry with a lower global index has been inserted.
#include <sched.h>

#include <fstream>

#include "ctmr_ctx.cuh"

namespace ctmr_host {

// ------------------------------------------------------------------------------------------------ stages
int ensure_stages(ctmr_ctx* c) {
    if (c->stages) return CTMR_OK;
    std::unique_ptr<Stage[]> stages(new (std::nothrow) Stage[kStages]);
    if (!stages) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    const uint64_t E = c->stage_entries;
    for (int k = 0; k < kStages; ++k) {
        Stage& s = stages[k];
        CU(c, create(s.stream));
        const int rc = s.out.allocate(c, E);
        if (rc) return rc;
        CU(c, alloc(s.blob, c->stage_bytes + 64));
        // K_map stages records in 16-byte pieces, so its last copy may read up to 15 bytes past the slice's data (inside
        // this allocation, never consumed): written once here so that those bytes are defined (compute-sanitizer initcheck)
        CU(c, cudaMemsetAsync(s.blob, 0, c->stage_bytes + 64, s.stream));
        CU(c, alloc(s.offsets, E + 1));
        CU(c, alloc(s.issuer_idx, E));
        CU(c, alloc(s.keys, E));
        CU(c, alloc(s.slot_of, E));
        CU(c, alloc(s.pair_slot, E));
        CU(c, alloc(s.order, E));
        CU(c, alloc(s.len_hist, 256));
        CU(c, alloc(s.meta_slots, 2 * E));
    }
    c->stages = std::move(stages);
    return CTMR_OK;
}

// ------------------------------------------------------------------------------------------------ PEM output
int pem_ensure(ctmr_ctx* c, PemStage& ps, uint64_t entries, uint64_t der_bytes) {
    const uint64_t need_bytes = der_bytes / 3 * 4 + der_bytes / 48 + 64 * entries + 256;  // body + newlines + boundary lines
    if (ps.cap_entries >= entries && ps.cap_bytes >= need_bytes) return CTMR_OK;
    CU(c, cudaDeviceSynchronize());
    ps = PemStage{};  // the old buffers go first, so that peak memory is the new set
    PemStage grown;
    CU(c, alloc(grown.sizes, entries + 1));
    CU(c, alloc(grown.off, entries + 1));
    CU(c, alloc(grown.text, need_bytes));
    grown.scan_temp_bytes = pem_scan_temp_bytes(entries + 1);
    CU(c, alloc(grown.scan_temp, grown.scan_temp_bytes ? grown.scan_temp_bytes : 16));
    grown.cap_entries = entries;
    grown.cap_bytes = need_bytes;
    ps = std::move(grown);
    return CTMR_OK;
}

// Encodes the selected certificates of one chunk on `s`, waits for it, and appends the text to the caller's
// buffer at *base (host).  pem_off_out[i] (i < cnt) = absolute start of entry i's text.
int pem_chunk(ctmr_ctx* c, PemStage& ps, const uint8_t* blob, const uint64_t* offsets, const uint32_t* lens, const uint8_t* select,
              uint64_t cnt, const ctmr_out* out, uint64_t first, uint64_t* base, cudaStream_t s) {
    CU(c, launch_pem_encode(blob, offsets, lens, select, cnt, ps.sizes, ps.scan_temp, ps.scan_temp_bytes, ps.off, ps.text, ps.cap_bytes,
                            c->st.error_flag, c->sm_count, s));
    ps.host_off.resize(cnt + 1);
    CU(c, cudaMemcpyAsync(ps.host_off.data(), ps.off, (cnt + 1) * 8, cudaMemcpyDeviceToHost, s));
    CU(c, cudaStreamSynchronize(s));
    const uint64_t total = ps.host_off[cnt];
    if (total > ps.cap_bytes) return fail(c, CTMR_E_BATCH_TOO_LARGE, "PEM staging too small (internal sizing)");
    if (*base + total > out->pem_cap) return fail(c, CTMR_E_BATCH_TOO_LARGE, "ctmr_out.pem_cap too small for the new certificates' PEM");
    if (total) CU(c, cudaMemcpyAsync(out->pem + *base, ps.text, total, cudaMemcpyDeviceToHost, s));
    for (uint64_t i = 0; i < cnt; ++i) out->pem_off[first + i] = *base + ps.host_off[i];
    *base += total;
    return CTMR_OK;
}

int copy_out(ctmr_ctx* c, const ctmr_dev_out& d, uint64_t cnt, const ctmr_out* out, uint64_t lo, cudaStream_t s) {
    CU(c, d2h_rows(out->status, d.status, lo, cnt, s));
    CU(c, d2h_rows(out->sha256, d.sha256, lo, cnt, s, 32));
    CU(c, d2h_rows(out->exp_hour, d.exp_hour, lo, cnt, s));
    CU(c, d2h_rows(out->serial_off, d.serial_off, lo, cnt, s));
    CU(c, d2h_rows(out->serial_len, d.serial_len, lo, cnt, s));
    CU(c, d2h_rows(out->was_unknown, d.was_unknown, lo, cnt, s));
    CU(c, d2h_rows(out->first_issuer_hour, d.first_issuer_hour, lo, cnt, s));
    CU(c, d2h_rows(out->issuer_name_off, d.issuer_name_off, lo, cnt, s));
    CU(c, d2h_rows(out->issuer_name_len, d.issuer_name_len, lo, cnt, s));
    CU(c, d2h_rows(out->crldp_off, d.crldp_off, lo, cnt, s));
    CU(c, d2h_rows(out->crldp_len, d.crldp_len, lo, cnt, s));
    CU(c, d2h_rows(out->first_issuer_dn, d.first_issuer_dn, lo, cnt, s));
    CU(c, d2h_rows(out->first_crldp, d.first_crldp, lo, cnt, s));
    return CTMR_OK;
}

}  // namespace ctmr_host

namespace {

struct BatchArgs {
    const uint8_t* blob;
    const uint64_t* offsets;
    uint64_t n;
    const uint32_t* issuer_idx;
    uint32_t n_issuers;
    int64_t now_unix_ns;
    ctmr_out* out;
};

struct Slice {
    uint64_t lo = 0, hi = 0;      // entries of the caller's batch
    uint64_t first_index = 0;     // global index of entry lo
};

// rounds x members.  Every slice respects the entry budget and the byte budget of a stage; W == 1 halves as well.
int plan_rounds(ctmr_ctx* c0, uint32_t W, const BatchArgs& a, std::vector<std::vector<Slice>>& plan) {
    const uint64_t E = c0->stage_entries, B = c0->stage_bytes;
    const auto fits = [&](uint32_t, uint64_t lo, uint64_t hi, bool* ok) {
        *ok = a.offsets[hi] - a.offsets[lo] <= B;
        return CTMR_OK;
    };
    for (uint64_t pos = 0, q = 0; pos < a.n; pos = std::min(a.n, pos + W * q)) {
        split_window(a.n, pos, W, std::min<uint64_t>(E, (a.n - pos + W - 1) / W), fits, &q);
        if (q == 0) return fail(c0, CTMR_E_BATCH_TOO_LARGE, "a single entry exceeds the staging budget (config.max_batch_bytes)");
        std::vector<Slice> round(W);
        for (uint32_t r = 0; r < W; ++r) {
            round[r].lo = std::min(a.n, pos + r * q);
            round[r].hi = std::min(a.n, pos + (r + 1) * q);
        }
        plan.push_back(std::move(round));
    }
    return CTMR_OK;
}

// Upload of one member's slice to stage `sidx`, and the slice's description for run_round.  chain: the round follows
// another, whose owner passes (and string identities) this round's must follow.
int stage_slice(ctmr_ctx* c, int sidx, bool chain, const BatchArgs& a, const Slice& sl, const uint32_t* map_dev, bool meta,
                RoundMember& x) {
    Stage& s = c->stages[sidx];
    const uint64_t cnt = sl.hi - sl.lo;
    CU(c, cudaSetDevice(c->device));
    x = RoundMember{};
    x.c = c;
    if (cnt) {
        const uint64_t bytes = a.offsets[sl.hi] - a.offsets[sl.lo];
        if (bytes) CU(c, cudaMemcpyAsync(s.blob, a.blob + a.offsets[sl.lo], bytes, cudaMemcpyHostToDevice, s.stream));
        CU(c, cudaMemcpyAsync(s.offsets, a.offsets + sl.lo, (cnt + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s.stream));
        if (a.issuer_idx) CU(c, cudaMemcpyAsync(s.issuer_idx, a.issuer_idx + sl.lo, cnt * sizeof(uint32_t), cudaMemcpyHostToDevice, s.stream));
        ctmr_dev_batch& db = x.db;
        db.blob = s.blob - a.offsets[sl.lo];  // offsets stay absolute
        db.blob_bytes = a.offsets[sl.hi];
        db.offsets = s.offsets;
        db.n = cnt;
        db.issuer_idx = a.issuer_idx ? s.issuer_idx.get() : nullptr;
        db.issuer_map = map_dev;
        db.issuer_map_len = a.n_issuers;
        db.first_index = sl.first_index;
        db.now_unix_ns = a.now_unix_ns;
    }
    x.dout = s.out.dev_out(a.out->sha256 != nullptr, meta);
    x.dout.keys = s.keys;
    x.slot_of = s.slot_of; x.pair_slot = s.pair_slot; x.order = s.order; x.len_hist = s.len_hist; x.meta_slots = s.meta_slots;
    x.map_stream = x.reduce_stream = s.stream;
    x.mapped = s.out.mapped; x.reduced = s.out.reduced; x.meta_done = s.out.meta_done;
    if (chain) {
        const Stage& prev = c->stages[(sidx + kStages - 1) % kStages];
        x.prev_reduced = prev.out.reduced;
        x.prev_meta_done = prev.out.meta_done;
    }
    x.ch_map = CH_STAGE_MAP + sidx;
    x.ch_resolve = CH_STAGE_RESOLVE + sidx;
    x.ch_meta = CH_STAGE_META + sidx;
    return CTMR_OK;
}

// the requested outputs of one member's slice in stage `sidx` to the caller's buffers [, PEM]
int stage_out(const RoundMember& x, int sidx, const BatchArgs& a, const Slice& sl, bool want_pem, uint64_t* pem_base) {
    ctmr_ctx* c = x.c;
    Stage& s = c->stages[sidx];
    const uint64_t cnt = sl.hi - sl.lo;
    if (!cnt) return CTMR_OK;
    CU(c, cudaSetDevice(c->device));
    int rc = copy_out(c, x.dout, cnt, a.out, sl.lo, s.stream);
    if (rc || !want_pem) return rc;
    // StoreCertificatePEM's argument for this slice's new certificates (the host waits for this slice here)
    return pem_chunk(c, s.pem, x.db.blob, x.db.offsets, nullptr, x.dout.was_unknown, cnt, a.out, sl.lo, pem_base, s.stream);
}

// The pipeline.  m[0..W) = the member GPUs this process drives (W == 1: a plain ctx, or one rank of a multi-process
// group).  `plan` rows beyond a rank's own rounds are empty slices (multi-process: every rank runs the agreed number).
// Each round: every member's upload on its stage's stream, run_round (exchange parity and barrier channels = stage,
// chained to the previous stage), then the outputs in member order, so that PEM texts are appended in entry order.
int run_rounds(ctmr_ctx** m, uint32_t W, const BatchArgs& a, const std::vector<std::vector<Slice>>& plan,
               const std::vector<const uint32_t*>& map_dev, ctmr_ctx** failed) {
    const ctmr_out* out = a.out;
    const bool meta = want_meta(out);
    const bool want_pem = out->pem != nullptr || out->pem_off != nullptr;
    uint64_t pem_base = 0;
    int rc = CTMR_OK;
#define RR(r, call)                 \
    do {                            \
        rc = (call);                \
        if (rc) {                   \
            *failed = m[r];         \
            return rc;              \
        }                           \
    } while (0)
    RoundMember rm[kMaxWorld];
    for (size_t k = 0; k < plan.size(); ++k) {
        const int sidx = (int)(k % kStages);
        for (uint32_t r = 0; r < W; ++r) RR(r, stage_slice(m[r], sidx, k > 0, a, plan[k][r], map_dev[r], meta, rm[r]));
        rc = run_round(rm, W, sidx, m[0]->stage_entries, meta, failed);
        if (rc) return rc;
        for (uint32_t r = 0; r < W; ++r) RR(r, stage_out(rm[r], sidx, a, plan[k][r], want_pem, &pem_base));
    }
#undef RR
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        CU(m[r], cudaSetDevice(m[r]->device));
        for (int k = 0; k < kStages; ++k) CU(m[r], cudaStreamSynchronize(m[r]->stages[k].stream));
    }
    if (want_pem) out->pem_off[a.n] = pem_base;
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = ctmr_check_device(m[r], nullptr);
        if (rc) return rc;
    }
    *failed = nullptr;
    return CTMR_OK;
}

// drain_streams over every member's stage streams
void drain(ctmr_ctx** m, uint32_t W) {
    for (uint32_t r = 0; r < W; ++r) {
        if (!m[r]->stages) continue;
        cudaStream_t s[kStages];
        for (int k = 0; k < kStages; ++k) s[k] = m[r]->stages[k].stream;
        drain_streams(m[r], s, kStages);
    }
}

int process_batch_members(ctmr_ctx** m, uint32_t W, uint64_t* next_index, ctmr_ctx** failed, const uint8_t* blob, const uint64_t* offsets,
                          uint64_t n, const uint8_t* issuer_blob, const uint64_t* issuer_offsets, uint32_t n_issuers,
                          const uint32_t* issuer_idx, int64_t now_unix_ns, ctmr_out* out) {
    ctmr_ctx* c0 = m[0];
    *failed = c0;
    if (!out || (n && (!blob || !offsets))) return fail(c0, CTMR_E_INVALID, "bad argument");
    const bool ipc = peer_call(c0);
    if (n == 0 && !ipc) {
        *failed = nullptr;
        return CTMR_OK;
    }
    int rc = check_pem(c0, out);
    if (rc) return rc;
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        CU(m[r], cudaSetDevice(m[r]->device));
        rc = ensure_stages(m[r]);
        if (rc) return rc;
    }
    *failed = c0;
    rc = note_call_start(m, W, *next_index);
    if (rc) return rc;
    for (uint32_t r = 0; r < W; ++r)  // the mark's copy before any round's kernels
        for (int k = 0; k < kStages; ++k) CU(m[r], cudaStreamWaitEvent(m[r]->stages[k].stream, m[r]->mark_taken, 0));
    // issuers of this batch -> dense indices (GPU work only for certificates never seen before); the registry is
    // shared by the group, so member 0's answer holds for every member
    std::vector<const uint32_t*> map_dev(W, nullptr);
    if (n_issuers) {
        std::vector<uint32_t> dense(n_issuers);
        rc = ctmr_register_issuers(c0, issuer_blob, issuer_offsets, n_issuers, dense.data());
        if (rc) return rc;
        for (uint32_t r = 0; r < W; ++r) {
            *failed = m[r];
            CU(m[r], cudaSetDevice(m[r]->device));
            rc = upload_issuer_map(m[r], dense.data(), n_issuers);
            if (rc) return rc;
            map_dev[r] = m[r]->issuer_map_dev;
        }
        *failed = c0;
    }
    BatchArgs a{blob, offsets, n, issuer_idx, n_issuers, now_unix_ns, out};
    std::vector<std::vector<Slice>> plan;
    rc = plan_rounds(c0, W, a, plan);
    if (rc) return rc;
    if (out->pem) {  // the PEM staging of every stage a slice uses, before anything is inserted
        for (size_t k = 0; k < plan.size(); ++k)
            for (uint32_t r = 0; r < W; ++r) {
                if (plan[k][r].hi == plan[k][r].lo) continue;
                *failed = m[r];
                CU(m[r], cudaSetDevice(m[r]->device));
                rc = pem_ensure(m[r], m[r]->stages[k % kStages].pem, m[r]->stage_entries, m[r]->stage_bytes);
                if (rc) return rc;
            }
        *failed = c0;
    }
    uint64_t advance = n;
    if (ipc) {
        // collective call: the agreed number of rounds, the most any rank needs, each rank's round k at
        // (k * world + rank) * E above the base
        const uint32_t world = c0->st.peer.world, rank = c0->st.peer.rank;
        uint64_t row[kMaxWorld] = {};
        rc = peer_agree(c0, CTMR_OK, plan.size(), row, "", "collective call failed before any work");
        if (rc) return rc;
        uint64_t rounds = 1;  // at least one round: its barriers also fence the mailbox against the next call
        for (uint32_t r = 0; r < world; ++r) rounds = std::max(rounds, row[r]);
        plan.resize(rounds, std::vector<Slice>(1));
        for (uint64_t k = 0; k < rounds; ++k) {
            if (plan[k][0].hi == plan[k][0].lo) plan[k][0].lo = plan[k][0].hi = n;  // an empty round
            plan[k][0].first_index = *next_index + (k * world + rank) * c0->stage_entries;
        }
        advance = rounds * world * c0->stage_entries;
    } else {
        for (auto& round : plan)
            for (auto& sl : round) sl.first_index = *next_index + sl.lo;  // entry i of the batch = global index base + i
    }
    rc = run_rounds(m, W, a, plan, map_dev, failed);
    // Also after a failure: some rounds may have been inserted, and a retry must not find itself "first" again with
    // the same indices (its entries then read as known, which is what they are).
    *next_index += advance;
    if (rc) drain(m, W);
    return rc;
}

}  // namespace

// =================================================================================================
extern "C" {

int ctmr_process_batch(ctmr_ctx* c, const uint8_t* blob, const uint64_t* offsets, uint64_t n, const uint8_t* issuer_blob,
                       const uint64_t* issuer_offsets, uint32_t n_issuers, const uint32_t* issuer_idx, int64_t now_unix_ns,
                       ctmr_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_process_batch");
    ctmr_ctx* failed = nullptr;
    return process_batch_members(&c, 1, &c->next_index, &failed, blob, offsets, n, issuer_blob, issuer_offsets, n_issuers, issuer_idx,
                                 now_unix_ns, out);
}

// ------------------------------------------------------------------------------------------------ one process, several GPUs
int ctmr_group_create(const ctmr_config* cfg, const int32_t* devices, uint32_t n_devices, ctmr_group** out) {
    if (!cfg || !devices || !out || n_devices == 0 || n_devices > kMaxWorld || cfg->struct_size < sizeof(ctmr_config))
        return fail(nullptr, CTMR_E_INVALID, "bad group configuration (1..8 devices)");
    *out = nullptr;
    ctmr_group* g = new (std::nothrow) ctmr_group();
    if (!g) return fail(nullptr, CTMR_E_NOMEM, "host allocation failed");
    auto bail = [&](int code, const std::string& msg) {  // msg may be a member's error: report before destroying
        fail(nullptr, code, msg);
        ctmr_group_destroy(g);
        return code;
    };
    for (uint32_t r = 0; r < n_devices; ++r) {
        ctmr_config mc = *cfg;
        mc.device = devices[r];
        ctmr_ctx* c = nullptr;
        const int rc = ctmr_create(&mc, &c);
        if (rc) return bail(rc, ctmr_last_error(nullptr));
        c->group = g;
        g->m.push_back(c);
    }
    // peer access between the distinct devices (NVLink through NVSwitch on an H100 box)
    for (uint32_t r = 0; r < n_devices; ++r)
        for (uint32_t q = 0; q < n_devices; ++q) {
            if (devices[r] == devices[q]) continue;
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, devices[r], devices[q]) != cudaSuccess || !can)
                return bail(CTMR_E_PEER, "GPUs " + std::to_string(devices[r]) + " and " + std::to_string(devices[q]) + " cannot access each other's memory");
            cudaSetDevice(devices[r]);
            const cudaError_t e = cudaDeviceEnablePeerAccess(devices[q], 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return bail(CTMR_E_PEER, std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
            (void)cudaGetLastError();
        }
    if (n_devices > 1) {
        uint8_t *bases[kMaxWorld] = {}, *xb[kMaxWorld] = {};
        for (uint32_t r = 0; r < n_devices; ++r) {
            cudaSetDevice(devices[r]);
            const int rc = alloc_exchange(g->m[r], n_devices);
            if (rc) return bail(rc, g->m[r]->err);
            bases[r] = g->m[r]->shared;
            xb[r] = g->m[r]->xchg;
        }
        for (uint32_t r = 0; r < n_devices; ++r) {
            attach_views(g->m[r], bases, n_devices, r);
            attach_exchange(g->m[r], xb, n_devices, r);
            g->m[r]->peer_mode = PEER_GROUP;
        }
    }
    *out = g;
    return CTMR_OK;
}

void ctmr_group_destroy(ctmr_group* g) {
    if (!g) return;
    for (ctmr_ctx* c : g->m) {  // quiesce every member before any shard goes away
        cudaSetDevice(c->device);
        cudaDeviceSynchronize();
    }
    for (ctmr_ctx* c : g->m) ctmr_destroy(c);
    delete g;
}

const char* ctmr_group_last_error(ctmr_group* g) { return g ? g->err.c_str() : g_create_error.c_str(); }
uint32_t ctmr_group_size(ctmr_group* g) { return g ? (uint32_t)g->m.size() : 0; }
ctmr_ctx* ctmr_group_member(ctmr_group* g, uint32_t rank) { return g && rank < g->m.size() ? g->m[rank] : nullptr; }

int ctmr_group_process_batch(ctmr_group* g, const uint8_t* blob, const uint64_t* offsets, uint64_t n, const uint8_t* issuer_blob,
                             const uint64_t* issuer_offsets, uint32_t n_issuers, const uint32_t* issuer_idx, int64_t now_unix_ns,
                             ctmr_out* out) {
    return on_group(g, process_batch_members, blob, offsets, n, issuer_blob, issuer_offsets, n_issuers, issuer_idx, now_unix_ns, out);
}


// ------------------------------------------------------------------------------------------------ one process per GPU
namespace {
struct PeerHandle {
    char magic[8];  // "CTMRPEER"
    cudaIpcMemHandle_t mem, xchg;
    uint64_t table_slots, pair_slots, meta_slots, total, X;
    uint32_t max_issuers, world;
    uint32_t epoch, pad;  // the rank's table epoch at export (ctmr_common.cuh)
};
static_assert(sizeof(PeerHandle) <= CTMR_PEER_HANDLE_BYTES, "peer handle size");
}  // namespace

int ctmr_peer_export(ctmr_ctx* c, uint32_t world, uint8_t handle_out[CTMR_PEER_HANDLE_BYTES]) {
    if (!c || !handle_out || world == 0 || world > kMaxWorld) return fail(c, CTMR_E_INVALID, "bad argument (1..8 ranks)");
    if (c->peer_mode != PEER_NONE || c->group) return fail(c, CTMR_E_INVALID, "ctx already belongs to a group");
    CU(c, cudaSetDevice(c->device));
    PeerHandle h{};
    std::memcpy(h.magic, "CTMRPEER", 8);
    cudaError_t e = cudaIpcGetMemHandle(&h.mem, c->shared);
    if (e != cudaSuccess) return fail(c, CTMR_E_PEER, std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(e));
    if (world > 1) {
        if (c->xchg && c->exported_world != world) return fail(c, CTMR_E_INVALID, "already exported for a different group size");
        const int rc = alloc_exchange(c, world);
        if (rc) return rc;
        c->exported_world = world;  // the views of the peers' areas are set by ctmr_peer_attach
        e = cudaIpcGetMemHandle(&h.xchg, c->xchg);
        if (e != cudaSuccess) return fail(c, CTMR_E_PEER, std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(e));
    }
    h.X = c->X;
    h.world = world;
    h.table_slots = c->st.table_mask + 1;
    h.pair_slots = c->st.pair_mask + 1;
    h.meta_slots = c->st.meta_mask + 1;
    h.total = c->lay.total;
    h.max_issuers = c->st.max_issuers;
    h.epoch = c->st.epoch;
    std::memset(handle_out, 0, CTMR_PEER_HANDLE_BYTES);
    std::memcpy(handle_out, &h, sizeof h);
    c->ipc_exported = true;
    return CTMR_OK;
}

int ctmr_peer_attach(ctmr_ctx* c, uint32_t rank, uint32_t world, const uint8_t* handles) {
    if (!c || !handles || world == 0 || world > kMaxWorld || rank >= world) return fail(c, CTMR_E_INVALID, "bad argument (1..8 ranks)");
    if (c->peer_mode != PEER_NONE || c->group) return fail(c, CTMR_E_INVALID, "ctx already belongs to a group");
    CU(c, cudaSetDevice(c->device));
    if (world == 1) return CTMR_OK;
    if (!c->xchg || c->exported_world != world) return fail(c, CTMR_E_INVALID, "call ctmr_peer_export(ctx, world, ...) with this group size first");
    uint8_t *bases[kMaxWorld] = {}, *xb[kMaxWorld] = {};
    IpcMap base_maps[kMaxWorld], xchg_maps[kMaxWorld];  // into the ctx once every rank's region is open
    // The ranks' table epochs must be one: a cross-GPU string-identity insert stamps the inserting rank's epoch into the
    // owner's table, and each rank would read the other's slots as empty.  A rank that reset its tables or loaded a
    // checkpoint on its own before attaching is ahead; every rank moves to the highest epoch of the handles (the same on
    // every rank), its live slots with it.  From then on every reset is collective and the epochs stay in lockstep.
    uint32_t epoch = 0;
    for (uint32_t r = 0; r < world; ++r) {
        PeerHandle h;
        std::memcpy(&h, handles + (size_t)r * CTMR_PEER_HANDLE_BYTES, sizeof h);
        if (std::memcmp(h.magic, "CTMRPEER", 8) != 0) return fail(c, CTMR_E_INVALID, "not a ctmr peer handle");
        if (h.table_slots != c->st.table_mask + 1 || h.pair_slots != c->st.pair_mask + 1 || h.meta_slots != c->st.meta_mask + 1 ||
            h.max_issuers != c->st.max_issuers || h.total != c->lay.total || h.X != c->X || h.world != world)
            return fail(c, CTMR_E_INVALID, "rank " + std::to_string(r) + " was created with different capacities (or exported for another group size)");
        if (r == rank && h.epoch != c->st.epoch)
            return fail(c, CTMR_E_INVALID, "the tables were reset or loaded since ctmr_peer_export: export again");
        epoch = h.epoch > epoch ? h.epoch : epoch;
        if (r == rank) {
            bases[r] = c->shared;
            xb[r] = c->xchg;
            continue;
        }
        cudaError_t e = open(base_maps[r], h.mem);
        if (e == cudaSuccess) e = open(xchg_maps[r], h.xchg);
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            return fail(c, CTMR_E_PEER, "cudaIpcOpenMemHandle(rank " + std::to_string(r) + "): " + cudaGetErrorString(e));
        }
        bases[r] = base_maps[r];
        xb[r] = xchg_maps[r];
    }
    if (epoch != c->st.epoch) {  // done before this rank enters any collective call, whose barriers order the peers' inserts after it
        CU(c, launch_restamp_tables(c->st, c->st.epoch, epoch, c->sm_count, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
        c->st.epoch = epoch;
    }
    std::swap(c->ipc_base, base_maps);
    std::swap(c->ipc_xchg, xchg_maps);
    attach_views(c, bases, world, rank);
    attach_exchange(c, xb, world, rank);
    c->peer_mode = PEER_IPC;
    return CTMR_OK;
}

int ctmr_peer_barrier_device(ctmr_ctx* c, void* stream) {
    if (!c) return CTMR_E_INVALID;
    CU(c, cudaSetDevice(c->device));
    return peer_barrier(c, CH_USER, stream ? (cudaStream_t)stream : c->stream);
}

int ctmr_peer_allreduce_histogram_device(ctmr_ctx* c, uint64_t* counts_dst, uint32_t n_slots, uint64_t* status_dst, void* stream) {
    if (!c || n_slots > c->st.max_issuers) return fail(c, CTMR_E_INVALID, "bad argument");
    CU(c, cudaSetDevice(c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    int rc = peer_barrier(c, CH_HIST_A, s);  // every rank's counting kernels have finished
    if (rc) return rc;
    CU(c, launch_hist_sum(c->pf, n_slots, reinterpret_cast<unsigned long long*>(counts_dst), reinterpret_cast<unsigned long long*>(status_dst), s));
    return peer_barrier(c, CH_HIST_B, s);    // nobody resets its histogram while a peer still reads it
}

// ------------------------------------------------------------------------------------------------ host placement
int ctmr_bind_host_to_device(int32_t device) {
    char bus[32] = {};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) {
        (void)cudaGetLastError();
        return -1;
    }
    for (char* p = bus; *p; ++p) *p = (char)tolower(*p);
    int node = -1;
    {
        std::ifstream f(std::string("/sys/bus/pci/devices/") + bus + "/numa_node");
        if (!(f >> node) || node < 0) return -1;
    }
    std::ifstream f("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist");
    std::string list;
    if (!std::getline(f, list) || list.empty()) return -1;
    cpu_set_t allowed, want;
    CPU_ZERO(&want);
    if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return -1;
    size_t i = 0;
    int picked = 0;
    while (i < list.size()) {  // "0-31,64-95"
        size_t j = list.find(',', i);
        if (j == std::string::npos) j = list.size();
        const std::string tok = list.substr(i, j - i);
        const size_t dash = tok.find('-');
        const int a = atoi(tok.c_str()), b = dash == std::string::npos ? a : atoi(tok.c_str() + dash + 1);
        for (int cpu = a; cpu <= b && cpu < CPU_SETSIZE; ++cpu)
            if (CPU_ISSET(cpu, &allowed)) {
                CPU_SET(cpu, &want);
                ++picked;
            }
        i = j + 1;
    }
    if (!picked || sched_setaffinity(0, sizeof want, &want) != 0) return -1;
    return node;
}

}  // extern "C"
