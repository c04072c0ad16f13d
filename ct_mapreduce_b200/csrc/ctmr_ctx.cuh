// ctmr_ctx.cuh -- internal: the context behind the opaque ctmr_ctx of include/ctmr.h, shared by the translation
// units that implement the C ABI (ctmr_api.cu: lifecycle, issuers, the steps of a round and run_round, which sequences
// one round of the key exchange for all three callers, the ranks' barriers and mailbox, device entry points, the table
// calls of a ctx and a group (read side, preload, eviction, snapshots), front end plumbing;
// ctmr_pipeline.cu: the host-buffer batch pipeline on one GPU, on a group of GPUs, and across processes, and the copy of
// a round's outputs to the host, the group's lifecycle and the peer attach; ctmr_frontend_api.cu: the wire-format front
// end on one GPU and on a group; ctmr_resize.cu: the tables of a ctx or a group in other sizes).
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
#include <functional>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <vector>

#include "ctmr_common.cuh"
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

// where the path writes the results of one slice or chunk of up to cap entries, and the events of its round of the key
// exchange: one per host-pipeline stage and one for the front end
struct PathOut {
    uint64_t cap = 0;
    DevBuf<uint8_t> status, sha, was_unknown, first;
    DevBuf<int64_t> exp_hour;
    DevBuf<uint32_t> serial_off, serial_len;
    DevBuf<uint32_t> spans;       // [4][cap]: issuer name off/len, crldp off/len
    DevBuf<uint8_t> first_meta;   // [2][cap]: first_issuer_dn, first_crldp
    Event mapped;     // recorded after the round's K_map (its inserts have reached the owners' tables)
    Event reduced;    // recorded after the round's owner passes (resolve + pairs of own entries and inbox records)
    Event meta_done;  // recorded after the round's string-identity insert

    int allocate(ctmr_ctx* c, uint64_t entries);  // every buffer and event (ctmr_api.cu)
    // the buffers as the path's outputs: sha256 when the caller asked for it, the spans and first_* when the call computes
    // string identities; keys are the caller's to set
    ctmr_dev_out dev_out(bool sha256, bool meta) const {
        ctmr_dev_out d{};
        d.status = status;
        d.sha256 = sha256 ? sha.get() : nullptr;
        d.exp_hour = exp_hour;
        d.serial_off = serial_off;
        d.serial_len = serial_len;
        d.was_unknown = was_unknown;
        d.first_issuer_hour = first;
        if (meta) {
            d.issuer_name_off = spans;
            d.issuer_name_len = spans + cap;
            d.crldp_off = spans + 2 * cap;
            d.crldp_len = spans + 3 * cap;
            d.first_issuer_dn = first_meta;
            d.first_crldp = first_meta + cap;
        }
        return d;
    }
};

struct Stage {
    Stream stream;
    PathOut out;
    DevBuf<uint8_t> blob;
    DevBuf<uint64_t> offsets;
    DevBuf<uint32_t> issuer_idx;
    DevBuf<ctmr_key> keys;
    DevBuf<uint32_t> slot_of;
    DevBuf<uint32_t> pair_slot;
    DevBuf<uint32_t> order;
    DevBuf<unsigned int> len_hist;
    DevBuf<uint32_t> meta_slots;  // [2*E]
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

// the tree forms of the bodies call (ctmr_process_raw_bodies_tree(s)): each body's status and entry count, read back with
// the chunk's entry count, and the fold windows of the chunk's bodies ([cap_entries] each).  Allocated on the first such
// call.
struct BodyFoldState {
    HostBuf<uint8_t> h_status;
    HostBuf<uint32_t> h_count;
    HostBuf<BodyWindow> h_win;
    DevBuf<BodyWindow> win;
};

// whole get-entries bodies (ctmr_process_raw_bodies): the JSON kernels' buffers for a chunk of up to cap_text / 2 bytes
// and cap_entries bodies and requested entries.  Allocated on the first bodies call.
struct BodyState {
    std::unique_ptr<BodyFoldState> fold;  // bodies_fold_ensure
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
    PathOut out;  // the path's outputs for this chunk; its events serve the rounds of a group or collective call (fe_member)
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
    float fe_ms = 0.f, path_ms = 0.f;
    uint64_t launches = 0;
    PemStage pem;
    std::unique_ptr<TileState> tl;    // tiles_ensure
    std::unique_ptr<TreeState> tree;  // tree_ensure
    std::unique_ptr<BodyState> bd;    // bodies_ensure
};

// ctmr_revoked_known: the double-buffered staging of whole CRLs, the split's per-byte, per-candidate and per-entry
// buffers (allocated on the first call, for chunks of `budget` bytes), and the join's set (grown to the largest chunk).
// A group's members 1.. hold only the set arrays: a copy of member 0's set and their own answers.
struct CrlState {
    uint64_t budget = 0, cap_crls = 0, cap_cand = 0, cap_entries = 0;
    Stream copy_stream;
    DevBuf<uint8_t> stage[2];       // [budget + 64] each
    DevBuf<CrlDesc> desc[2];        // [cap_crls] each
    HostBuf<CrlDesc> h_desc[2];
    Event uploaded[2], consumed[2];
    DevBuf<CrlRes> res;             // [cap_crls]
    DevBuf<uint32_t> cnt16, off16;  // [budget / 16 + 1]: candidates per 16 staged bytes and their exclusive scan
    DevBuf<uint32_t> cpos, ccrl, link, jump[2];  // [cap_cand]
    DevBuf<uint8_t> mark;           // [cap_cand]
    DevBuf<uint8_t> temp;           // cub scans
    size_t temp_bytes = 0;
    // per entry [cap_entries]
    DevBuf<uint32_t> epos, ecrl, eslot, esets;
    DevBuf<uint64_t> eserial_off;
    DevBuf<uint8_t> eserial_len, ereason, estatus, eknown;
    DevBuf<int64_t> erevoked, ehour;
    // the set of a chunk's (issuer, serial) pairs, and per pair the lowest hour and the number of sets holding it
    uint64_t set_cap = 0;
    DevBuf<CrlSetSlot> set;
    DevBuf<int32_t> set_hour, recv_hour;   // recv_*: a group's member 0 receives the other members' answers there
    DevBuf<uint32_t> set_count, recv_count;
    // a rank attached to peers (crl_peer_ensure): the 64-byte records it sends in a round [X], and the owner side's union
    // set of the records every rank sends in a round [union_cap = 2 world X, a power of two] with its answers
    DevBuf<ctmr_key> records;
    uint64_t union_cap = 0;
    DevBuf<CrlSetSlot> union_set;
    DevBuf<int32_t> union_hour;
    DevBuf<uint32_t> union_count;
};

// ctmr_revoked_cascade (ctmr_cascade.cu): one bit per table slot (revoked: the slot's pair is in a chunk's set), the
// registry's digests and the covered-issuer bitmap over dense indices, the three include / test lists of slot indices
// [list_cap] each, one level's bits [bit_words] and on a group's member 0 the receive side of the merge [bit_words].
// Built on first use and grown, all or nothing.
struct CascadeState {
    uint64_t slot_words = 0;
    DevBuf<uint32_t> revoked;            // [slot_words]
    uint32_t issuer_cap = 0;
    DevBuf<uint8_t> dig;                 // [issuer_cap][32]
    DevBuf<uint32_t> covered;            // [issuer_cap / 32 + 1]
    DevBuf<unsigned long long> counters; // [2]: records appended to a list, records counted
    uint64_t list_cap = 0;
    DevBuf<uint32_t> list[3];
    uint64_t bit_words = 0;
    DevBuf<uint32_t> bits, recv;         // recv: a group's member 0 only (0 words elsewhere)
    uint64_t recv_words = 0;
};

// ctmr_revoked_stash (ctmr_cascade.cu): the published filter laid out again in words, each level from a 16-byte boundary,
// its level table, and the 44-byte key bodies of the R records the filter calls not revoked.  Built on first use and
// grown, all or nothing.
struct StashLevel {
    uint64_t word;  // the level's first word in the filter words
    uint32_t m, k;
};
struct StashState {
    uint64_t word_cap = 0;
    DevBuf<uint32_t> words;              // [word_cap]
    uint64_t level_cap = 0;
    DevBuf<StashLevel> levels;           // [level_cap]
    uint64_t body_cap = 0;
    DevBuf<uint32_t> bodies;             // [body_cap][11]: issuer, serial_len, serial[39]
};

// ctmr_revoked_verify (ctmr_cascade.cu): one bit per table slot (listed: a stash lists the slot's pair), the stashes' set,
// the counts and the listed records read back (the filter is StashState's, the slots of the listed records go to the
// cascade's list 1).  Built on first use and grown, all or nothing.
struct VerifyState {
    uint64_t slot_words = 0;
    DevBuf<uint32_t> listed;              // [slot_words]
    DevBuf<unsigned long long> counters;  // [9]: before and since (revoked, missed, valid, blocked), then records listed
    uint64_t set_cap = 0;
    DevBuf<CrlSetSlot> set;               // [set_cap]
    uint64_t rec_cap = 0;
    DevBuf<KnownSlot> recs;               // [rec_cap]: the listed records, tag 1 for an S record, 0 for an R record
};

// the ctx's private device words (one allocation)
struct SmallDev {
    unsigned long long slots_used;   // DeviceState::slots_used points here (no kernel reads it)
    int error_flag;                  // DeviceState::error_flag
    unsigned long long cardinality;  // ctmr_set_cardinality's probe result
    unsigned long long table_count;  // ctmr_table_stats' count
    unsigned long long evict[2];     // ctmr_evict_expired: live, expired
    uint32_t sha_sink;               // ctmr_sha256_ceiling_device's sink
    alignas(16) uint8_t digest[32];  // lookup_digest: one digest to register
    uint32_t idx;                    //   and its index
    int resize_error;                // ctmr_resize's rehash: its own flag, so that a failed resize leaves error_flag as it was
    unsigned long long occupancy[3]; // ctmr_table_occupancy's counts: known, pair, meta
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
    CH_CKPT = 14,                        // ctmr_checkpoint_*: every barrier and agreement of the collective size, save and load
    CH_CRL = 15,                         // ctmr_revoked_known and ctmr_revoked_cascade: the two barriers of each round of a
                                         // collective call, and of each slice of the cascade's OR all-reduce
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
    // delta checkpoints (ctmr_checkpoint.cu), kept by the ctx, by member 0 of a group and by every peer rank: the next
    // index at the last call that removed records other than by eviction (a reset or a load), and the evictions since,
    // as (next index at the call, now) with the indices rising and the nows falling, so that the first mark at or above
    // an index holds the highest now passed from that index on
    uint64_t delta_floor = 0;
    std::vector<std::pair<uint64_t, int64_t>> evict_marks;
    // rollback marks (ctmr_rollback.cu): the starts of the last CTMR_ROLLBACK_MARKS entry-taking calls.  Mark k (counted
    // from the last clear) lives in slot k % CTMR_ROLLBACK_MARKS: its next index on the ctx that holds the delta state,
    // the status counters at the call's start on every member (copied on the device by the call's stream).
    std::vector<uint64_t> mark_index;        // [CTMR_ROLLBACK_MARKS]
    uint64_t marks = 0;                      // marks taken since the last clear; the indices rise
    uint64_t marks_lo = 0;                   // the marks held are marks_lo .. marks - 1 (their slots not overwritten)
    DevBuf<unsigned long long> mark_status;  // [CTMR_ROLLBACK_MARKS][CTMR_ST__COUNT]
    Event mark_taken;                        // recorded after the last mark's copy
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
    bool ipc_exported = false;              // ctmr_peer_export was called: the region is behind a CUDA IPC handle (no resize)
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
    std::unique_ptr<CrlState> crl;  // ctmr_revoked_known (ctmr_crl.cu)
    std::unique_ptr<CascadeState> cascade;  // ctmr_revoked_cascade (ctmr_cascade.cu)
    std::unique_ptr<StashState> stash;      // ctmr_revoked_stash and ctmr_revoked_verify (ctmr_cascade.cu)
    std::unique_ptr<VerifyState> verify;    // ctmr_revoked_verify (ctmr_cascade.cu)
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

// the call computes string identities: the caller asked for one of them
inline bool want_meta(const ctmr_out* o) { return o->first_issuer_dn || o->first_crldp || o->issuer_name_off || o->crldp_off; }
inline int check_pem(ctmr_ctx* c, const ctmr_out* o) {
    if ((o->pem != nullptr) != (o->pem_off != nullptr)) return fail(c, CTMR_E_INVALID, "pem and pem_off go together");
    return CTMR_OK;
}

// The window rule of a group round: the round cuts ONE contiguous window of units from `pos` on, q units per member
// (member r's slice is [pos + r q, pos + (r + 1) q), clipped to `total`), so that every unit keeps its global index.
// q starts at q0 and is halved, rounded up, until fits(r, lo, hi, &ok) leaves ok set for every member's slice.  *q = 0:
// not even one unit per member fits.  An error of fits ends the search and is returned.
template <class Fits>
int split_window(uint64_t total, uint64_t pos, uint32_t W, uint64_t q0, Fits fits, uint64_t* q) {
    for (*q = q0;; *q = (*q + 1) / 2) {
        bool ok = true;
        for (uint32_t r = 0; r < W && ok; ++r) {
            const int rc = fits(r, std::min(total, pos + r * *q), std::min(total, pos + (r + 1) * *q), &ok);
            if (rc) return rc;
        }
        if (ok) return CTMR_OK;
        if (*q == 1) {
            *q = 0;
            return CTMR_OK;
        }
    }
}

// D2H of rows [0, cnt) of the device's `src` to rows [lo, lo + cnt) of the caller's `dst`, `per` elements of dst's type
// a row, on s; nothing when the caller did not ask for the array (dst null) or the device has none (src null)
template <class T>
cudaError_t d2h_rows(T* dst, const void* src, uint64_t lo, uint64_t cnt, cudaStream_t s, uint64_t per = 1) {
    if (!dst || !src) return cudaSuccess;
    return cudaMemcpyAsync(dst + lo * per, src, cnt * per * sizeof(T), cudaMemcpyDeviceToHost, s);
}
// D2H of entries [0, cnt) of device outputs to entries [lo, lo + cnt) of the caller's outputs: every per-entry array of
// ctmr_out that both sides have, on stream s
int copy_out(ctmr_ctx* c, const ctmr_dev_out& d, uint64_t cnt, const ctmr_out* out, uint64_t lo, cudaStream_t s);
// No copy into or out of the caller's buffers may outlive a failed call: waits for streams s[0..n) of c.  c's last
// error stays the failure's.
inline void drain_streams(ctmr_ctx* c, const cudaStream_t* s, int n) {
    const std::string keep = c->err;
    cudaSetDevice(c->device);
    for (int k = 0; k < n; ++k) cudaStreamSynchronize(s[k]);
    c->err = keep;
}
int group_fail(ctmr_group* g, ctmr_ctx* c, int rc);   // c's error becomes g's last error (when both are given); returns rc
// A call through the body a ctx and a group share, body(m, W, next_index, &failed, args...) over the members m[0..W):
// on_ctx passes the ctx alone (a NULL ctx: CTMR_E_INVALID), on_group every member of the group, whose last error becomes
// that of the member the body names (member 0 when none) on failure (a NULL or empty group: bare CTMR_E_INVALID).
template <class Body, class... Args>
int on_ctx(ctmr_ctx* c, Body body, Args... args) {
    if (!c) return fail(nullptr, CTMR_E_INVALID, "bad argument");
    ctmr_ctx* failed = nullptr;
    return body(&c, 1u, &c->next_index, &failed, args...);
}
template <class Body, class... Args>
int on_group(ctmr_group* g, Body body, Args... args) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    ctmr_ctx* failed = nullptr;
    const int rc = body(g->m.data(), (uint32_t)g->m.size(), &g->next_index, &failed, args...);
    return rc ? group_fail(g, failed ? failed : g->m[0], rc) : rc;
}
// the sections of a shared region for these capacities: the tables come last, so every section before SharedLayout::meta
// depends on max_issuers alone (ctmr_resize copies that prefix byte for byte)
SharedLayout make_layout(uint64_t table_slots, uint64_t pair_slots, uint64_t meta_slots, uint32_t max_issuers);
// st.table, pairs, meta, issuer_counts and status_counts -> their sections of c->shared under c->lay
void point_at_region(ctmr_ctx* c);
// views of the shared regions `bases[0..world)` (this rank's own among them) -> st.peer, pf, reg
void attach_views(ctmr_ctx* c, uint8_t* const* bases, uint32_t world, uint32_t rank);
int peer_barrier(ctmr_ctx* c, uint32_t channel, cudaStream_t s);   // PEER_IPC only; no-op otherwise
// c is one rank of a group of processes (ctmr_peer_attach): its front-end, checkpoint, CRL and batch calls are collective
inline bool peer_call(const ctmr_ctx* c) { return c->peer_mode == PEER_IPC && c->st.peer.world > 1; }
// one word from every rank through the mailbox, row[r] = rank r's; the caller then checks the device for a barrier that
// timed out
int peer_mailbox(ctmr_ctx* c, uint64_t mine, uint64_t* row);
// One agreement of a collective call: posts peer_word(mine, payload) and reads every rank's word into row.  Returns, in
// this order: a failed exchange or a barrier that timed out; this rank's own error `mine`, with its error text; the
// failure of the lowest rank whose word failed, CTMR_E_PEER_FAILED (their_code: that rank's own code) with the text
// "<call>rank r's part of this <part>"; CTMR_OK, row then holding every rank's payload.
int peer_agree(ctmr_ctx* c, int mine, uint64_t payload, uint64_t* row, const char* call, const char* part, bool their_code = false);
int refresh_digests(ctmr_ctx* c);                                   // host memo <- device registry
int lookup_digest(ctmr_ctx* c, const uint8_t digest[32], bool insert, uint32_t* idx_out, bool* found);
int upload_issuer_map(ctmr_ctx* c, const uint32_t* dense, uint32_t n);
int ensure_stages(ctmr_ctx* c);
// a snapshot's or checkpoint's issuer digests on their way into the registry of the group (rank 0's region): allocated
// before a load overwrites anything (ctmr_api.cu)
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
int bodies_fold_ensure(ctmr_ctx* c);  // ... and the fold windows of its tree forms, after bodies_ensure
int ensure_scratch(ctmr_ctx* c, uint64_t n);
int ensure_device_path(ctmr_ctx* c, uint64_t n);   // what ctmr_process_device needs for n entries
// known-certificate table, pairs, string identities, per-issuer and status counters and the error flag to zero, on this
// ctx alone (ctmr_reset_device brackets it with the group's barriers)
int reset_tables(ctmr_ctx* c, cudaStream_t s);
// after the registry was replaced: the host memos of it go, and so do the Chain[0] mirror and the tiles' fingerprints
int clear_issuer_memos(ctmr_ctx* c);
// one shard's TTL eviction at now_unix_sec (ctmr_evict_expired), *evicted its expired keys
int evict_shard(ctmr_ctx* c, int64_t now_unix_sec, uint64_t* evicted);
// the delta state of the ctx that holds it (member 0 of a group): records were removed other than by eviction, and the
// state stands at next_index; an eviction at now_unix_sec while the state stood at next_index; the highest now of an
// eviction from `since` on (INT64_MIN when none)
inline void delta_floor_at(ctmr_ctx* c, uint64_t next_index) {
    c->delta_floor = next_index;
    c->evict_marks.clear();
    c->marks = c->marks_lo = 0;  // no rollback reaches across it either
}
// A rollback mark for the members m[0..W) of a call that starts at next_index (ctmr_rollback.cu): each member's status
// counters copied into its ring on the stream `s` (NULL: the member's own stream), then mark_taken recorded there.  A
// call that starts where the newest mark stands keeps that mark (an earlier call at this index may have changed the
// state already).  No host wait.
int note_call_start(ctmr_ctx** m, uint32_t W, uint64_t next_index, cudaStream_t s = nullptr);
// ctmr_process_device; mark: take the call's rollback mark (the public entry on a handle with an index of its own)
int process_device(ctmr_ctx* c, const ctmr_dev_batch* b, const ctmr_dev_out* o, void* stream, bool mark);
inline void note_eviction(ctmr_ctx* c, uint64_t next_index, int64_t now_unix_sec) {
    while (!c->evict_marks.empty() && c->evict_marks.back().second <= now_unix_sec) c->evict_marks.pop_back();
    c->evict_marks.emplace_back(next_index, now_unix_sec);
}
inline int64_t evicted_since(const ctmr_ctx* c, uint64_t since) {
    for (const auto& mk : c->evict_marks)
        if (mk.first >= since) return mk.second;
    return INT64_MIN;
}

// A failure of one ctx, a group or a peer rank in a CRL call.  One ctx or a group stops at the first; a peer rank that
// failed after its first agreement does no more work but still meets every barrier and agreement of the call.  The first
// failure's code and text are kept (for a peer rank, for the final agreement).
struct PeerLocal {
    int code = CTMR_OK;
    std::string err;
    void fail(const ctmr_ctx* c, int rc) {
        if (code || rc == CTMR_OK) return;
        code = rc;
        err = c->err;
    }
};

// The CRL path as ctmr_revoked_cascade and ctmr_revoked_stash use it (ctmr_crl.cu, whose ctmr_revoked_known runs the same
// drivers).  crl_prepare: the checks every CRL call makes before any work (`out` is only tested for NULL; `call` opens the
// error text), then each CRL's dense issuer (CTMR_ISSUER_NONE when the digest is not registered); on a peer rank
// (peer_call) also the split's and the exchange's buffers and *n_chunks, the batch's chunk count, so that every failure
// before any work travels in agreement 1 (*n_chunks is 0 otherwise).
int crl_prepare(ctmr_ctx* c, const ctmr_crl_batch* b, const void* out, const char* call, std::vector<uint32_t>& issuer,
                uint64_t* n_chunks);

// A set of (issuer, serial) pairs on a member's device, mask + 1 slots, and per slot the answer arrays a join fills: the
// lowest hour and the number of sets that hold the pair.
struct CrlSet {
    const CrlSetSlot* slots;
    uint64_t mask;
    int32_t* hour;
    uint32_t* count;
};
using CrlSetVisit = std::function<int(ctmr_ctx* c, const CrlSet& set)>;
// crl_each_set: every chunk through the split, its entries and the set of its (issuer, serial) pairs; status[] gets the
// CTMR_CRL_* of this process's CRLs, and visit(c, set) is issued on c's stream, its device current, while the set is
// intact.  One ctx or a group (peer false; W members): member 0 builds each chunk's set, and every member visits a copy
// on its device (a chunk with no entries: no visit); synchronous, and no upload outlives it.  A peer rank (peer true,
// W == 1), after agreement 1 (row: every rank's chunk count): the steps and rounds of the collective
// ctmr_revoked_known, and in each round the rank visits the union set of every rank's valid records of the round,
// between the round's two barriers.  Failures go to `local`; false: the call stops (one ctx or a group failed, or a
// rank's failure stopped the steps and the ranks go to the final agreement).
bool crl_each_set(ctmr_ctx* const* m, uint32_t W, bool peer, const ctmr_crl_batch* b, const std::vector<uint32_t>& issuer, uint64_t* row,
                  const CrlSetVisit& visit, std::vector<uint8_t>& status, PeerLocal& local);
// crl_peer_finish: a peer rank's end of a CRL call after crl_each_set.  The ctx's copy stream and stream are drained (no
// upload may read the caller's data afterwards), the device is checked for a barrier that timed out, the text of the
// rank's first failure is restored, and the final agreement posts `payload` (row: every rank's).  Returns peer_agree's
// code.
int crl_peer_finish(ctmr_ctx* c, PeerLocal& local, uint64_t payload, uint64_t* row, const char* call);

// Where a table's live slots go when they are compacted in slot order (launch_evict_compact): the exclusive prefix of the
// live slots per tile of kCompactTile, on the host and on the device.  host[tiles()] = the live slots of the table.
struct CompactPlan {
    std::vector<unsigned long long> host;
    DevBuf<unsigned long long> dev;
    uint64_t tiles() const { return host.empty() ? 0 : host.size() - 1; }
    uint64_t live() const { return host.empty() ? 0 : host.back(); }
};
template <class Slot>
int compact_plan(ctmr_ctx* c, const Slot* table, uint64_t n_slots, int64_t now_sec, CompactPlan& p, uint64_t since = 0) {
    const uint64_t tiles = (n_slots + kCompactTile - 1) / kCompactTile;
    DevBuf<uint32_t> counts;
    std::vector<uint32_t> h(tiles);
    CU(c, alloc(counts, tiles));
    CU(c, alloc(p.dev, tiles + 1));
    CU(c, launch_evict_compact(table, n_slots, c->st.epoch, now_sec, 0, tiles, (const unsigned long long*)nullptr, (Slot*)nullptr, counts.get(), c->stream,
                               since));
    CU(c, cudaMemcpyAsync(h.data(), counts, tiles * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    p.host.assign(tiles + 1, 0);
    for (uint64_t t = 0; t < tiles; ++t) p.host[t + 1] = p.host[t] + h[t];
    CU(c, cudaMemcpyAsync(p.dev, p.host.data(), (tiles + 1) * sizeof(unsigned long long), cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return CTMR_OK;
}
uint64_t device_round_entries(uint64_t n, uint32_t rounds);   // E of a ctmr_process_device call cut into `rounds` rounds
uint32_t peer_rounds();   // rounds of the collective ctmr_process_device (CTMR_PEER_ROUNDS, env override for experiments)
int pem_ensure(ctmr_ctx* c, PemStage& ps, uint64_t entries, uint64_t der_bytes);
int pem_chunk(ctmr_ctx* c, PemStage& ps, const uint8_t* blob, const uint64_t* offsets, const uint32_t* lens, const uint8_t* select,
              uint64_t cnt, const ctmr_out* out, uint64_t first, uint64_t* base, cudaStream_t s);

}  // namespace ctmr_host
