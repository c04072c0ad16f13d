// ctmr_ctx.cuh -- internal: the context behind the opaque ctmr_ctx of include/ctmr.h, shared by the translation
// units that implement the C ABI (ctmr_api.cu: lifecycle, issuers, the steps of a round and run_round, which sequences
// one round of the key exchange for all three callers, device entry points, read side, front end plumbing;
// ctmr_pipeline.cu: the host-buffer batch pipeline on one GPU, on a group of GPUs, and across processes, and the copy of
// a round's outputs to the host; ctmr_frontend_api.cu: the wire-format front end on one GPU and on a group).
//
// Ownership: the ctx owns everything it allocates, through the handles below and std::unique_ptr, so deleting the ctx
// releases it all.  The parts built on first use (the pipeline stages, ctmr_process_device's streams and events, the
// front end and its tile and tree state) are built into a local and moved into the ctx only when every allocation
// succeeded: a failed call leaves the ctx as it was, and the next call tries again.
#pragma once
#include <algorithm>
#include <array>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <vector>

#include "ctmr_device.cuh"
#include "ctmr_kernels.cuh"

using namespace ctmr;

namespace ctmr_host {

// A handle owns one CUDA resource and releases it in its destructor.  A handle is released only while its ctx's device
// is current: every entry point sets that device first, and ctmr_destroy sets it before it deletes the ctx.
template <class P, class Arg, cudaError_t (*Release)(Arg)>
class Own {
  public:
    Own() = default;
    explicit Own(P p) : p_(p) {}
    Own(Own&& o) noexcept : p_(o.p_) { o.p_ = nullptr; }
    Own& operator=(Own&& o) noexcept {
        if (this != &o) {
            reset();
            p_ = o.p_;
            o.p_ = nullptr;
        }
        return *this;
    }
    ~Own() { reset(); }
    void reset() {
        if (p_) Release(p_);
        p_ = nullptr;
    }
    P get() const { return p_; }
    operator P() const { return p_; }
    P operator->() const { return p_; }

  private:
    P p_ = nullptr;
};

template <class T> using DevBuf = Own<T*, void*, cudaFree>;
template <class T> using HostBuf = Own<T*, void*, cudaFreeHost>;  // pinned
using Stream = Own<cudaStream_t, cudaStream_t, cudaStreamDestroy>;
using Event = Own<cudaEvent_t, cudaEvent_t, cudaEventDestroy>;
using IpcMap = Own<uint8_t*, void*, cudaIpcCloseMemHandle>;

// n elements; a buffer the handle held is released first
template <class T> cudaError_t alloc(DevBuf<T>& b, size_t n) {
    b.reset();
    void* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, n * sizeof(T));
    if (e == cudaSuccess) b = DevBuf<T>(static_cast<T*>(p));
    return e;
}
template <class T> cudaError_t alloc(HostBuf<T>& b, size_t n) {
    b.reset();
    void* p = nullptr;
    const cudaError_t e = cudaMallocHost(&p, n * sizeof(T));
    if (e == cudaSuccess) b = HostBuf<T>(static_cast<T*>(p));
    return e;
}
inline cudaError_t create(Stream& s) {
    s.reset();
    cudaStream_t h = nullptr;
    const cudaError_t e = cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking);
    if (e == cudaSuccess) s = Stream(h);
    return e;
}
inline cudaError_t create(Event& ev, unsigned flags = cudaEventDisableTiming) {
    ev.reset();
    cudaEvent_t h = nullptr;
    const cudaError_t e = cudaEventCreateWithFlags(&h, flags);
    if (e == cudaSuccess) ev = Event(h);
    return e;
}
inline cudaError_t open(IpcMap& m, cudaIpcMemHandle_t handle) {
    m.reset();
    void* p = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&p, handle, cudaIpcMemLazyEnablePeerAccess);
    if (e == cudaSuccess) m = IpcMap(static_cast<uint8_t*>(p));
    return e;
}

constexpr int kStages = 3;                      // host-API pipeline depth
constexpr int kMaxRounds = 16;                  // rounds of one ctmr_process_device call
constexpr uint64_t kStageEntries = 1ull << 18;  // entries per pipeline stage
constexpr uint64_t kStageBytes = 768ull << 20;  // leaf bytes per pipeline stage

extern thread_local std::string g_create_error;

inline int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return v && *v ? atoi(v) : dflt;
}

// device side of the PEM output (ctmr_out.pem): one per host-pipeline stage and one for the front end
struct PemStage {
    uint64_t cap_entries = 0, cap_bytes = 0;
    DevBuf<uint64_t> sizes, off;
    DevBuf<uint8_t> text;
    DevBuf<uint8_t> scan_temp;
    size_t scan_temp_bytes = 0;
    std::vector<uint64_t> host_off;
};

struct Stage {
    Stream stream;
    Event mapped;     // recorded after this stage's K_map (its inserts have reached the owners' tables)
    Event reduced;    // recorded after this stage's owner passes (resolve + pairs of own entries and inbox records)
    Event meta_done;  // recorded after this stage's string-identity insert
    DevBuf<uint8_t> blob;
    DevBuf<uint64_t> offsets;
    DevBuf<uint32_t> issuer_idx;
    DevBuf<uint8_t> status;
    DevBuf<uint8_t> sha;
    DevBuf<int64_t> exp_hour;
    DevBuf<uint32_t> serial_off;
    DevBuf<uint32_t> serial_len;
    DevBuf<uint8_t> was_unknown;
    DevBuf<uint8_t> first;
    DevBuf<ctmr_key> keys;
    DevBuf<uint32_t> slot_of;
    DevBuf<uint32_t> pair_slot;
    DevBuf<uint32_t> order;
    DevBuf<unsigned int> len_hist;
    DevBuf<uint32_t> spans;       // [4][E]: issuer name off/len, crldp off/len
    DevBuf<uint32_t> meta_slots;  // [2*E]
    DevBuf<uint8_t> first_meta;   // [2][E]: first_issuer_dn, first_crldp
    PemStage pem;                 // allocated when a caller first asks for PEM output
};

// ctmr_process_device pipelines map (stream A) against reduce (stream B) over its rounds
struct DevicePipeline {
    Stream stream_a, stream_a2, stream_b;  // K_map alternates between a and a2
    Event ev_fork, ev_join_a, ev_join_a2, ev_join_b;
    Event ev_map0[kMaxRounds], ev_map1[kMaxRounds], ev_red1[kMaxRounds];  // timed: ctmr_profile_last
    Event ev_tok[kMaxRounds];
    DevBuf<unsigned int> len_hist[kMaxRounds];
    Event ev_pulled[kParities];  // round k's bits pulled (its exchange parity may be reused)
};

// one upload stage of the front end: a chunk's characters and string spans, device side and pinned host staging
struct FeStage {
    DevBuf<uint8_t> text;  // [16 + cap_text + 64]
    DevBuf<uint64_t> leaf_off, extra_off;
    HostBuf<uint64_t> h_leaf_off, h_extra_off;
    DevBuf<uint32_t> leaf_len, extra_len;
    HostBuf<uint32_t> h_leaf_len, h_extra_len;
    Event uploaded, consumed;
    std::vector<uint8_t> pack;  // host staging of the slow path (strings scattered over more than one chunk of text)
};

// static-ct-api tiles (ctmr_process_tiles): per-chunk buffers beyond the front end's, and the fingerprint table.
// Allocated on the first tile call or chain-certificate registration.
struct TileState {
    DevBuf<TileDesc> tiles[2];  // per upload stage: the chunk's tiles, device and pinned host
    HostBuf<TileDesc> h_tiles[2];
    DevBuf<uint8_t> tile_bad;
    DevBuf<uint64_t> entry_off, leaf_index, leaf_data_off;
    DevBuf<uint32_t> entry_tile, te_len;
    DevBuf<unsigned int> first_stop;
    DevBuf<uint8_t> leaf_hash;
    Event ev_split0, ev_split1;  // around tile_split: the serial walk is timed on its own
    float split_ms = 0.f;
    // fingerprint -> dense issuer index: device table, host copy, host memo keyed by the 32 bytes
    DevBuf<FpSlot> fp_dev;
    std::vector<FpSlot> fp_host;
    uint64_t fp_mask = 0, fp_used = 0;
    std::unordered_map<std::string, uint32_t> fp_memo;
};

// whole get-entries bodies (ctmr_process_raw_bodies): the JSON kernels' buffers for a chunk of up to cap_text / 2 bytes
// and cap_entries bodies and requested entries.  Allocated on the first bodies call.
struct BodyState {
    DevBuf<BodyDesc> desc[2];  // per upload stage: the chunk's bodies, device and pinned host
    HostBuf<BodyDesc> h_desc[2];
    DevBuf<unsigned long long> starts;
    DevBuf<uint8_t> trans, carry;
    DevBuf<BlockMasks> masks;
    DevBuf<uint32_t> stack;
    DevBuf<uint8_t> body_status;
    DevBuf<uint32_t> body_count, body_base;
    DevBuf<uint64_t> s_off[2], abs_off[2];
    DevBuf<uint32_t> s_len[2], raw_len[2];
    DevBuf<uint8_t> s_esc, esc;
    DevBuf<uint8_t> temp;
    size_t temp_bytes = 0;
    Event ev_json0, ev_json1;  // around the JSON kernels: timed on their own
    float json_ms = 0.f;
};

// the logs' Merkle trees (ctmr_process_*_tree, ctmr_process_*_trees): the call's trees on the device and the scratch of
// the fold.  Allocated on the first tree call, for cap_trees trees; a call with more trees builds it again, larger.  On
// a group (ctmr_group_process_*_tree(s)) member 0 holds the trees; every other member folds its chunks into ranges, and
// member 0 receives and merges them.
struct TreeState {
    uint32_t cap_trees = 0;
    DevBuf<TreeDev> dev;          // [cap_trees] the trees for the whole call: uploaded at its start, read back at its end
    HostBuf<TreeDev> host;        // [cap_trees] pinned staging of those two copies
    DevBuf<FoldTree> desc;        // [cap_trees] the trees of the chunk being folded
    HostBuf<FoldTree> h_desc;
    DevBuf<uint32_t> order[2];    // [cap_entries] per upload stage: the chunk's entries grouped by tree
    HostBuf<uint32_t> h_order[2];
    DevBuf<uint8_t> leaf;         // [cap_entries][32] get-entries leaf hashes of a chunk
    DevBuf<uint8_t> lvl[2];       // [cap_entries / 2 + 2 * cap_trees][32] each: ping-pong level buffers
    // a group's members 1..: per upload stage, the ranges of that stage's chunk, and the range fold's missing-leaf words
    DevBuf<TreeRange> range[2];             // [cap_trees] each
    DevBuf<unsigned long long> range_miss;  // [cap_trees]
    // a group's member 0: the other members' ranges of a round, and events around the merge (timed)
    DevBuf<TreeRange> recv;                 // [recv_members][cap_trees]
    uint32_t recv_members = 0;
    Event merge0, merge1;
    // the call
    uint32_t n_trees = 0;
    const uint32_t* log = nullptr;  // the tree of each entry (pages) or tile (tiles); NULL: everything goes to tree 0
    std::vector<uint64_t> next;     // [n_trees] log position of each tree's next entry to be uploaded
    std::vector<uint64_t> start;    // [n_trees] each tree's size at the start of the call
    std::vector<uint32_t> count;    // [n_trees] scratch of the grouping
    bool active = false;            // a tree call is running: the chunks fold their leaves
    bool ranges = false;            // this ctx folds its chunks into ranges (a group's member 1..)
    bool merge_timed = false;       // merge0 / merge1 hold a merge whose time is not in fe_ms yet
};

// CT wire-format front end (include/ctmr_frontend.h): device buffers of one chunk + the device mirror of
// the issuer registry keyed by certificate bytes
struct FrontEnd {
    uint64_t cap_entries = 0, cap_text = 0, cap_decoded = 0;
    FeStage stage[2];          // upload double buffer
    Stream copy_stream;
    DevBuf<uint64_t> pad_size, dec_off;
    DevBuf<uint32_t> dec_len;
    DevBuf<uint8_t> str_bad, decoded;
    DevBuf<uint8_t> scan_temp;
    size_t scan_temp_bytes = 0;
    DevBuf<uint8_t> entry_status, entry_type, leaf_src;
    DevBuf<uint64_t> timestamp, leaf_abs, chain_abs, tbs_abs;
    DevBuf<uint32_t> leaf_rel, leaf_len_out, chain_len, tbs_len, issuer_idx;
    // outputs of the path for this chunk
    DevBuf<uint8_t> status, sha, was_unknown, first, first_meta;
    DevBuf<int64_t> exp_hour;
    DevBuf<uint32_t> serial_off, serial_len, spans;
    // issuer certificates by bytes
    DevBuf<IssuerCertSlot> slots_dev;
    std::vector<IssuerCertSlot> slots_host;
    uint64_t slot_mask = 0, slots_used = 0;
    DevBuf<uint8_t> arena;
    uint64_t arena_cap = 0, arena_used = 0;
    DevBuf<uint64_t> pending;
    uint64_t pending_mask = 0;
    DevBuf<uint32_t> unknown_list;
    uint32_t unknown_cap = 0;
    DevBuf<unsigned int> unknown_count;
    Event ev0, ev1, ev2;
    Event mapped, reduced, meta_done;  // round events of the group front end (fe_member)
    float fe_ms = 0.f, path_ms = 0.f;
    uint64_t launches = 0;
    PemStage pem;
    std::unique_ptr<TileState> tl;    // tiles_ensure
    std::unique_ptr<TreeState> tree;  // tree_ensure
    std::unique_ptr<BodyState> bd;    // bodies_ensure
};

// the ctx's private device words (one allocation)
struct SmallDev {
    unsigned long long slots_used;   // DeviceState::slots_used points here (no kernel reads it)
    int error_flag;                  // DeviceState::error_flag
    unsigned long long cardinality;  // ctmr_set_cardinality's probe result
    unsigned long long table_count;  // ctmr_table_stats' count
    unsigned long long evict[3];     // ctmr_evict_expired: live, expired, compaction cursor
    uint32_t sha_sink;               // ctmr_sha256_ceiling_device's sink
    alignas(16) uint8_t digest[32];  // lookup_digest: one digest to register
    uint32_t idx;                    //   and its index
};

}  // namespace ctmr_host
using namespace ctmr_host;

// offsets inside a rank's SHARED region: the part of its state the other ranks of a group address directly
// (one allocation, so that one CUDA IPC handle exports it).  Identical on every rank: same capacities.
struct SharedLayout {
    size_t flags = 0;          // [kPeerChannels + 1][kMaxWorld] u64: barrier epochs per channel, then the mailbox row
    size_t reg_counter = 0;    // u64 (rank 0's is THE registry)
    size_t status_counts = 0;  // [CTMR_ST__COUNT] u64
    size_t issuer_counts = 0;  // [max_issuers] u64
    size_t reg_digests = 0;    // [max_issuers][32]
    size_t reg_slots = 0;      // [reg_mask + 1] IssuerRegSlot
    size_t meta = 0, pairs = 0, table = 0, total = 0;
    uint64_t reg_mask = 0;
};

enum PeerMode { PEER_NONE = 0, PEER_GROUP = 1 /* one process, ctmr_group */, PEER_IPC = 2 /* one process per GPU */ };

// Barrier channels.  Every rank must pass a channel's epochs in the same order.  Inside one call each channel is used
// from one stream per rank, so its epochs are stream ordered.  CH_STAGE_* serve two calls: the host pipeline's rounds
// (on its stage streams) and the front end's collective rounds (on the ctx's stream).  Both calls are synchronous and
// every rank makes the same sequence of collective calls, so no two calls' barriers on a channel are ever in flight
// together.
enum : uint32_t {
    CH_STAGE_MAP = 0,      // + stage index (3): after K_map of a host-pipeline round
    CH_STAGE_RESOLVE = 3,  // + stage index (3): after resolve of a host-pipeline round
    CH_DEV_MAP = 6, CH_DEV_RESOLVE = 7,  // ctmr_process_device
    CH_USER = 8, CH_HIST_A = 9, CH_HIST_B = 10, CH_RESET_A = 11, CH_RESET_B = 12, CH_MAILBOX = 13,
    CH_STAGE_META = 16                   // + stage index (3): after the string-identity insert of a host-pipeline round
};

struct ctmr_ctx {
    int device = 0;
    int sm_count = 132;
    uint32_t flags = 0;
    Stream stream;
    DeviceState st{};
    FilterCfg filter{};
    uint64_t next_index = 0;
    uint64_t stage_entries = 0, stage_bytes = 0;
    std::unique_ptr<Stage[]> stages;  // [kStages], ensure_stages
    // shared region + the views of every rank's region (a single GPU is a group of one)
    DevBuf<uint8_t> shared;
    SharedLayout lay{};
    PeerFlags pf{};
    IssuerRegistry reg{};                  // lives in rank 0's region
    int peer_mode = PEER_NONE;
    IpcMap ipc_base[kMaxWorld];            // the other ranks' regions, opened with cudaIpcOpenMemHandle
    IpcMap ipc_xchg[kMaxWorld];
    // key exchange of a group: peer-visible area (inboxes, result bits, region sizes) + private bookkeeping
    DevBuf<uint8_t> xchg;
    uint64_t X = 0, cfg_round_entries = 0;
    uint32_t exported_world = 0;            // ctmr_peer_export was called for a group of this size (the views follow at attach)
    PeerExchange px{};
    DevBuf<unsigned long long> cursors;     // [kParities][kMaxWorld] records appended per owner (local)
    DevBuf<uint32_t> rev;                   // [kParities][world][X] inbox position -> entry
    DevBuf<uint32_t> in_slot, in_pair;      // [kParities][world][X] owner-side scratch of the inbox records
    unsigned long long epoch[kPeerChannels] = {};
    struct ctmr_group* group = nullptr;    // set when the ctx is a member of an in-process group
    // issuer memo on the host (the registry itself is on the device): DER -> index, digest -> index, index -> digest
    std::unordered_map<std::string, uint32_t> issuer_by_der;
    std::unordered_map<std::string, uint32_t> issuer_by_digest;
    std::vector<std::array<uint8_t, 32>> digests;
    DevBuf<uint32_t> issuer_map_dev;
    uint32_t issuer_map_cap = 0;
    // scratch of the device-resident entry points
    DevBuf<ctmr_key> keys_scratch;
    DevBuf<uint32_t> slot_scratch;
    DevBuf<uint32_t> pair_scratch;
    DevBuf<uint8_t> bits_scratch;
    DevBuf<uint32_t> meta_scratch;  // [2*cap]
    uint64_t scratch_cap = 0;
    DevBuf<uint32_t> order_scratch;  // length-bucketed order of the device entry points (ensure_order)
    uint64_t order_cap = 0;
    DevBuf<unsigned int> len_hist;
    std::unique_ptr<DevicePipeline> dp;  // ctmr_process_device
    int last_sub = 0;
    DevBuf<SmallDev> small;
    std::unique_ptr<FrontEnd> fe;
    uint32_t fe_peer_stopped = 0;  // ranks that stopped (tiles) in the last collective front-end call
    std::string err;
};

struct ctmr_group {
    std::vector<ctmr_ctx*> m;
    uint64_t next_index = 0;
    std::string err;
};

// ---- helpers shared by the ABI translation units --------------------------------------------------------------
namespace ctmr_host {

int fail(ctmr_ctx* ctx, int code, const std::string& msg);

#define CU(ctx, call)                                                                                   \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess) {                                                                        \
            return fail((ctx), e_ == cudaErrorMemoryAllocation ? CTMR_E_NOMEM : CTMR_E_CUDA,             \
                        std::string(#call) + ": " + cudaGetErrorString(e_));                            \
        }                                                                                               \
    } while (0)

uint64_t pow2_at_least(uint64_t v);
int ensure_order(ctmr_ctx* c, uint64_t n);   // c->order_scratch holds >= n entries, c->len_hist exists
// key exchange: allocation for a group of `world` ranks, views of every rank's area
size_t exchange_bytes(uint32_t world, uint64_t X);
int alloc_exchange(ctmr_ctx* c, uint32_t world);
void attach_exchange(ctmr_ctx* c, uint8_t* const* bases, uint32_t world, uint32_t rank);

// One member's part of a round of the key exchange: the GPU (ctx), its slice and where the slice's results and scratch
// live (all device memory, [db.n] each unless noted), its streams, events and barrier channels.
struct RoundMember {
    ctmr_ctx* c = nullptr;
    ctmr_dev_batch db{};  // db.n == 0: an empty slice, which still takes part in every sync
    ctmr_dev_out dout{};  // keys, was_unknown and first_issuer_hour are required; spans and first_* when string identities are wanted
    uint32_t *slot_of = nullptr, *pair_slot = nullptr;
    uint32_t* order = nullptr;           // K_map's length order, with len_hist (256 counters) as scratch
    unsigned int* len_hist = nullptr;
    uint32_t* meta_slots = nullptr;      // [2 * db.n]
    cudaStream_t map_stream = nullptr;   // round_begin, K_map, round_publish
    cudaStream_t reduce_stream = nullptr;  // everything after sync 1; may be map_stream
    // this round's events; reduced and meta_done may be null where nothing waits for them (one member, no chain)
    cudaEvent_t mapped = nullptr, reduced = nullptr, meta_done = nullptr;
    cudaEvent_t prev_reduced = nullptr, prev_meta_done = nullptr;  // optional: the previous round's, to chain on
    cudaEvent_t map_start = nullptr, map_end = nullptr;            // optional: timing events around K_map
    uint32_t ch_map = 0, ch_resolve = 0, ch_meta = 0;              // peer_barrier channels of sync 1, 2 and 3
};
// Issues one round for the W members this process drives: map + route, sync 1, owner passes, sync 2, pull, and with
// want_meta the string identities (insert, sync 3, read-back).  `parity` selects the exchange regions and
// max_per_region bounds one member's slice.  On error *failed names the member that failed.
int run_round(const RoundMember* m, uint32_t W, int parity, uint64_t max_per_region, bool want_meta, ctmr_ctx** failed);
// D2H of entries [0, cnt) of device outputs to entries [lo, lo + cnt) of the caller's outputs: every per-entry array of
// ctmr_out that both sides have, on stream s
int copy_out(ctmr_ctx* c, const ctmr_dev_out& d, uint64_t cnt, const ctmr_out* out, uint64_t lo, cudaStream_t s);
int group_fail(ctmr_group* g, ctmr_ctx* c, int rc);   // c's error becomes g's last error (when both are given); returns rc
// views of the shared regions `bases[0..world)` (this rank's own among them) -> st.peer, pf, reg
void attach_views(ctmr_ctx* c, uint8_t* const* bases, uint32_t world, uint32_t rank);
int peer_barrier(ctmr_ctx* c, uint32_t channel, cudaStream_t s);   // PEER_IPC only; no-op otherwise
int refresh_digests(ctmr_ctx* c);                                   // host memo <- device registry
int lookup_digest(ctmr_ctx* c, const uint8_t digest[32], bool insert, uint32_t* idx_out, bool* found);
int upload_issuer_map(ctmr_ctx* c, const uint32_t* dense, uint32_t n);
int preload_impl(ctmr_ctx* c, int64_t exp_hour, const uint8_t digest[32], const uint8_t* serial_blob, const uint64_t* serial_offsets,
                 uint64_t n, uint64_t first_index);
int ensure_stages(ctmr_ctx* c);
// snapshot pieces (ctmr_api.cu): one shard's tables + histograms, and the registry of the group (rank 0's region)
uint64_t snap_shard_bytes(ctmr_ctx* c);
int snap_shard_save(ctmr_ctx* c, uint8_t* p);
int snap_shard_load(ctmr_ctx* c, const uint8_t* p);
// a snapshot's issuer digests on their way into the registry: allocated before a load overwrites anything
struct RegistryUpload {
    DevBuf<uint8_t> digests;
    DevBuf<uint32_t> idx;
};
int snap_registry_alloc(ctmr_ctx* c, uint64_t n, RegistryUpload& u);
int snap_registry_restore(ctmr_ctx* c, const uint8_t* digests, uint64_t n, const RegistryUpload& u);
int frontend_ensure(ctmr_ctx* c);   // allocates the front end's buffers on first use (ctmr_api.cu)
int tiles_ensure(ctmr_ctx* c);      // ... and the tile buffers + fingerprint table (ctmr_frontend_api.cu), after frontend_ensure
int tiles_clear_fingerprints(ctmr_ctx* c);
int bodies_ensure(ctmr_ctx* c);     // ... and the JSON buffers of ctmr_process_raw_bodies (ctmr_frontend_api.cu), after frontend_ensure
int ensure_scratch(ctmr_ctx* c, uint64_t n);
int ensure_device_path(ctmr_ctx* c, uint64_t n);   // what ctmr_process_device needs for n entries
uint64_t device_round_entries(uint64_t n, uint32_t rounds);   // E of a ctmr_process_device call cut into `rounds` rounds
uint32_t peer_rounds();   // rounds of the collective ctmr_process_device (CTMR_PEER_ROUNDS, env override for experiments)
int pem_ensure(ctmr_ctx* c, PemStage& ps, uint64_t entries, uint64_t der_bytes);
int pem_chunk(ctmr_ctx* c, PemStage& ps, const uint8_t* blob, const uint64_t* offsets, const uint32_t* lens, const uint8_t* select,
              uint64_t cnt, const ctmr_out* out, uint64_t first, uint64_t* base, cudaStream_t s);

}  // namespace ctmr_host
