// ctmr_kernels.cuh -- launch-side declarations shared by ctmr_kernels.cu and ctmr_api.cu
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ctmr.h"
#include "../../include/ctmr_frontend.h"

namespace ctmr {

// issuerCNFilter, pre-split on ',' by the host (strings.Split, ct-fetch.go:58): prefixes are raw bytes.
struct FilterCfg {
    uint32_t filter_nonempty;  // len(*ctconfig.IssuerCNFilter) != 0
    uint32_t n_prefix;
    uint32_t log_expired;
    uint32_t flags;            // CTMR_F_*
    uint16_t off[33];          // prefix p = bytes[off[p] .. off[p+1])
    uint8_t bytes[446];
};
static_assert(sizeof(FilterCfg) == 16 + 66 + 446, "FilterCfg layout");

// known-certificate slot: 64 bytes = two 32-byte sectors
struct __align__(16) KnownSlot {
    unsigned long long inv_first;  // ~(lowest global entry index seen for this key); 0 = none yet
    unsigned long long tag;        // 0 empty | (hash & ~3)|1 pending | (hash & ~3)|2 ready
    uint32_t body[12];             // exp_hour, issuer, {serial_len, serial[39]}
};
static_assert(sizeof(KnownSlot) == 64, "KnownSlot layout");

struct __align__(16) PairSlot {   // one per Redis set "serials::<expDate>::<issuer>" ever written
    unsigned long long key;        // ((issuer << 32) | (uint32)exp_hour) + 1; 0 = empty
    unsigned long long inv_first;  // ~(lowest index among was-unknown entries of this (issuer, hour))
    unsigned long long count;      // SetCardinality of the set: unique serials inserted and not yet expired
    unsigned long long pad;
};
static_assert(sizeof(PairSlot) == 32, "PairSlot layout");


struct __align__(16) MetaSlot {      // IssuerMetadata string sets: identity = two independent 64-bit hashes
    unsigned long long h1;           // 0 = empty
    unsigned long long h2;           // 0 = not yet published
    unsigned long long inv_first;    // ~(lowest index among new certificates carrying this string)
    unsigned long long pad;
};

// Multi-GPU (SURVEY.md §8(e)): every set "serials::<expDate>::<issuer>" has ONE owner GPU
// (key_owner(exp_hour, issuer, world)), which holds its serials and its (issuer, hour) slot, and does every table
// operation on them with device-scope atomics in its own HBM.  What crosses NVLink is BULK traffic only (measured before
// the port: fine-grained remote atomics are limited by the rate of remote operations and made K_map several times slower):
// K_map appends the 64-byte key record of an entry owned elsewhere to a per-source region of the owner's INBOX
// (coalesced posted writes, cursors in local memory), the owner inserts / resolves its inbox after a barrier, and the
// source pulls the result bits back as contiguous arrays.  The peers' memory is mapped into every rank (peer access
// in one process, CUDA IPC across processes).
constexpr uint32_t kMaxWorld = 8;
constexpr uint32_t kParities = 3;   // exchange buffers in flight: the host pipeline's three stages / two rounds of the device path

// exchange areas of every rank (peer visible).  Region of (parity p, source s) = element offset (p * world + s) * X.
struct PeerExchange {
    ctmr_key* inbox[kMaxWorld];             // [kParities][world][X] key records appended by the sources
    uint8_t* out_wu[kMaxWorld];             // [kParities][world][X] was_unknown of the inbox records, same positions
    uint8_t* out_first[kMaxWorld];          // [kParities][world][X] first_issuer_hour
    unsigned long long* counts[kMaxWorld];  // [kParities][world] records per source region, published by the sources
    uint64_t X;                             // capacity of a region = the most entries one rank maps per round
    uint32_t world, rank;
};

// what K_map needs to route the keys of one round
struct RouteOut {
    ctmr_key* inbox[kMaxWorld];   // owner o's region for THIS source and this round's parity
    unsigned long long* cursor;   // local [world]: records appended per owner so far
    uint32_t* rev;                // local [world][X]: inbox position -> entry of this round (for the pull)
    uint64_t X;
    uint32_t world, rank;
};

struct PeerTables {
    KnownSlot* table[kMaxWorld];
    PairSlot* pairs[kMaxWorld];
    MetaSlot* meta[kMaxWorld];
    uint32_t world;  // 1 = single GPU: device-scope atomics, no peer traffic
    uint32_t rank;
};

// ctx-lifetime issuer registry ON THE DEVICE of rank 0: Issuer.ID digest -> dense index, find-or-insert with
// system-scope atomics, so that every rank of a group gets the same index for the same issuer without any host
// coordination (a key record carries the dense index; owner routing and the full-key compare depend on it).
struct __align__(16) IssuerRegSlot {
    unsigned long long state;  // 0 empty | 1 pending | 2 ready
    uint32_t idx;
    uint32_t pad;
    uint8_t digest[32];
    unsigned long long pad2[2];
};
static_assert(sizeof(IssuerRegSlot) == 64, "IssuerRegSlot layout");

struct IssuerRegistry {
    IssuerRegSlot* slots;          // [mask + 1]
    uint64_t mask;
    unsigned long long* counter;   // number of dense indices handed out
    uint8_t* by_index;             // [max_issuers][32]
    uint32_t max_issuers;
};

// barrier flags and histograms of every rank, for the cross-process barrier and the one-shot all-reduce
struct PeerFlags {
    unsigned long long* flags[kMaxWorld];          // [kPeerChannels][kMaxWorld] epochs, written by the peers
    unsigned long long* issuer_counts[kMaxWorld];  // [max_issuers]
    unsigned long long* status_counts[kMaxWorld];  // [CTMR_ST__COUNT]
    uint32_t world, rank;
    unsigned long long timeout_ns;                 // a barrier wait longer than this raises CTMR_E_PEER_TIMEOUT
};
constexpr uint32_t kPeerChannels = 20;

struct DeviceState {
    KnownSlot* table;          // this rank's shard (== peer.table[peer.rank])
    uint64_t table_mask;       // capacity - 1, identical on every rank
    PairSlot* pairs;
    uint64_t pair_mask;
    PeerTables peer;
    unsigned long long* issuer_counts;  // [max_issuers]
    uint32_t max_issuers;
    unsigned long long* status_counts;  // [CTMR_ST__COUNT]
    unsigned long long* slots_used;     // [1]
    int* error_flag;                    // [1]: 0 ok, CTMR_E_TABLE_FULL...
    MetaSlot* meta;                     // (issuer, kind, bytes) first-seen table
    uint64_t meta_mask;
};

struct MapParams {
    const uint8_t* blob;
    uint64_t blob_bytes;
    const uint64_t* offsets;
    const uint32_t* lens;  // optional explicit lengths (records not contiguous)
    uint64_t n;
    const uint32_t* issuer_idx;
    const uint32_t* issuer_map;
    uint32_t issuer_map_len;
    uint64_t first_index;
    int64_t now_sec;
    uint32_t now_frac_nonzero;
    uint32_t one;  // always 1: a multiplier ptxas cannot fold (see fadd in ctmr_device.cuh)
    uint8_t* status;
    uint8_t* sha256;
    int64_t* exp_hour;
    uint32_t* serial_off;
    uint32_t* serial_len;
    ctmr_key* keys;
    uint32_t* issuer_name_off;
    uint32_t* issuer_name_len;
    uint32_t* crldp_off;
    uint32_t* crldp_len;
    unsigned long long* status_counts;
    const uint32_t* order;             // [n] length-bucketed processing order (NULL = entry order)
    // fused K_insert (slot_of != NULL): keys this rank owns go straight into its table (slot -> slot_of), keys owned
    // elsewhere are appended to the owner's inbox (slot_of = 0xFFFFFFFF)
    KnownSlot* table;
    RouteOut route;
    uint64_t table_mask;
    int* error_flag;
    uint32_t* slot_of;
    FilterCfg filter;
};

cudaError_t launch_map(const MapParams& p, int sm_count, cudaStream_t s);
cudaError_t launch_sha_ceiling(uint32_t iters, int rolled, int ctas_per_sm, int sm_count, uint32_t* sink, cudaStream_t s);
cudaError_t launch_len_order(const uint64_t* offsets, const uint32_t* lens, uint64_t n, uint64_t blob_bytes, unsigned int* hist256, uint32_t* order,
                             int sm_count, cudaStream_t s);
cudaError_t launch_insert(const DeviceState& st, const ctmr_key* keys, uint64_t m, uint32_t* slot_of, cudaStream_t s);
cudaError_t launch_resolve(const DeviceState& st, const ctmr_key* keys, uint64_t m, const uint32_t* slot_of,
                           uint32_t* pair_slot, uint8_t* was_unknown, cudaStream_t s);
cudaError_t launch_resolve_pairs(const DeviceState& st, const ctmr_key* keys, uint64_t m, const uint32_t* pair_slot,
                                 const uint8_t* was_unknown, uint8_t* first_issuer_hour, cudaStream_t s);
// owner side of the exchange: the same three passes over the inbox regions of one parity (record counts on the device)
cudaError_t launch_inbox_insert(const DeviceState& st, const PeerExchange& px, uint32_t parity, uint64_t max_per_region, uint32_t* in_slot,
                                cudaStream_t s);
cudaError_t launch_inbox_resolve(const DeviceState& st, const PeerExchange& px, uint32_t parity, uint64_t max_per_region,
                                 const uint32_t* in_slot, uint32_t* in_pair, cudaStream_t s);
cudaError_t launch_inbox_pairs(const DeviceState& st, const PeerExchange& px, uint32_t parity, uint64_t max_per_region,
                               const uint32_t* in_pair, cudaStream_t s);
// source side: publish the region sizes to the owners (before the barrier), pull the result bits (after the second one)
cudaError_t launch_publish_counts(const PeerExchange& px, uint32_t parity, const unsigned long long* cursor, cudaStream_t s);
cudaError_t launch_pull_bits(const PeerExchange& px, uint32_t parity, const unsigned long long* cursor, const uint32_t* rev,
                             uint64_t max_per_region, uint8_t* was_unknown, uint8_t* first_issuer_hour, cudaStream_t s);
cudaError_t launch_meta_insert(const DeviceState& st, const uint8_t* blob, const uint64_t* offsets, const ctmr_key* keys, uint64_t m,
                               const uint8_t* was_unknown, const uint32_t* name_off, const uint32_t* name_len, const uint32_t* crl_off,
                               const uint32_t* crl_len, uint32_t* meta_slots /* [2*m] scratch */, cudaStream_t s);
cudaError_t launch_meta_resolve(const DeviceState& st, const ctmr_key* keys, uint64_t m, const uint32_t* meta_slots, uint8_t* first_dn,
                                uint8_t* first_crl, cudaStream_t s);
cudaError_t launch_evict_pairs(const DeviceState& st, int64_t now_sec, int sm_count, cudaStream_t s);
cudaError_t launch_issuer_registry(const IssuerRegistry& reg, const uint8_t* digests, const uint8_t* ok, uint32_t n, uint32_t* idx_out,
                                   int* error_flag, cudaStream_t s);
cudaError_t launch_peer_post(const PeerFlags& pf, unsigned long long value, cudaStream_t s);
cudaError_t launch_peer_barrier(const PeerFlags& pf, uint32_t channel, unsigned long long epoch, int* error_flag, cudaStream_t s);
cudaError_t launch_hist_sum(const PeerFlags& pf, uint32_t n_slots, unsigned long long* counts_dst, unsigned long long* status_dst,
                            cudaStream_t s);
cudaError_t launch_issuer_prepare(const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint8_t* digests,
                                  uint8_t* ok, cudaStream_t s);
cudaError_t launch_table_count(const DeviceState& st, unsigned long long* out, int sm_count, cudaStream_t s);
cudaError_t launch_evict_count(const DeviceState& st, int64_t now_sec, unsigned long long* counters /* [2] */, int sm_count, cudaStream_t s);
cudaError_t launch_evict_compact(const DeviceState& st, int64_t now_sec, KnownSlot* keep, unsigned long long* cursor, int sm_count,
                                 cudaStream_t s);
cudaError_t launch_evict_reinsert(const DeviceState& st, const KnownSlot* keep, uint64_t n, cudaStream_t s);
cudaError_t launch_cardinality(const DeviceState& st, int32_t exp_hour, uint32_t issuer, unsigned long long* out,
                               cudaStream_t s);

// ---- CT wire-format front end (ctmr_frontend.cu, include/ctmr_frontend.h) ------------------------
#define CTMR_ISSUER_UNRESOLVED 0xFFFFFFFDu  // internal: Chain[0] present, dense index not looked up yet

struct FeParams {
    const uint8_t* text;        // device copy of the batch's characters (slack of 16 bytes on both sides)
    uint64_t text_bytes;
    const uint64_t* leaf_off;   // [n] string spans inside text
    const uint32_t* leaf_len;
    const uint64_t* extra_off;
    const uint32_t* extra_len;
    uint64_t n;
    // string s = 2*entry + (0: leaf_input, 1: extra_data)
    uint64_t* pad_size;         // [2n+1] decoded size rounded up to 16
    uint64_t* dec_off;          // [2n+1] placement in the decoded arena (exclusive scan of pad_size)
    uint32_t* dec_len;          // [2n]
    uint8_t* str_bad;           // [2n]
    uint8_t* decoded;           // arena
    // per entry
    uint8_t* entry_status;
    uint8_t* entry_type;
    uint64_t* timestamp;
    uint8_t* leaf_src;
    uint32_t* leaf_rel;
    uint32_t* leaf_len_out;
    uint64_t* leaf_abs;         // arena offset of the certificate K_map processes
    uint64_t* chain_abs;        // arena offset / length of Chain[0]
    uint32_t* chain_len;
    uint64_t* tbs_abs;          // precert entries: the leaf's TBSCertificate
    uint32_t* tbs_len;
    uint32_t* issuer_idx;
};

// Device mirror of the issuer registry keyed by the certificate BYTES: Chain[0] repeats for millions of
// entries, so it is hashed, probed and compared in full on the GPU and parsed once per distinct value.
struct IssuerCertSlot {
    uint64_t h;          // 0 = empty
    uint32_t len;
    uint32_t idx;        // dense issuer index or CTMR_ISSUER_BAD
    uint64_t arena_off;  // 16-byte aligned, zero padded to a multiple of 16
    uint64_t pad;
};
struct IssuerCertTable {
    const IssuerCertSlot* slots;
    uint64_t mask;
    const uint8_t* arena;
};

// hash of a byte string = finish(sum over its little-endian 8-byte words (zero padded) of word(w, i), length):
// a commutative sum, so that 32 lanes can each take every 32nd word; the host computes the same value.
__host__ __device__ __forceinline__ uint64_t fe_mix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t issuer_cert_word(uint64_t w, uint32_t i) {
    return fe_mix64(w + 0x9E3779B97F4A7C15ULL * (uint64_t)(i + 1u));
}
__host__ __device__ __forceinline__ uint64_t issuer_cert_finish(uint64_t acc, uint32_t len) {
    return fe_mix64(acc ^ ((uint64_t)len << 32)) | (1ull << 63);  // never 0
}

size_t pem_scan_temp_bytes(uint64_t n_items);
cudaError_t launch_pem_encode(const uint8_t* blob, const uint64_t* offsets, const uint32_t* lens, const uint8_t* select, uint64_t n,
                              uint64_t* sizes, void* scan_temp, size_t scan_temp_bytes, uint64_t* pem_off, uint8_t* pem, uint64_t cap,
                              int* error_flag, int sm_count, cudaStream_t s);
size_t fe_scan_temp_bytes(uint64_t n_items);
cudaError_t launch_fe_decode(const FeParams& p, void* scan_temp, size_t scan_temp_bytes, int sm_count, cudaStream_t s);
cudaError_t launch_fe_frame(const FeParams& p, cudaStream_t s);
cudaError_t launch_fe_issuer(const FeParams& p, const IssuerCertTable& tab, uint64_t* pending, uint64_t pending_mask,
                             uint32_t* unknown_list, uint32_t unknown_cap, unsigned int* unknown_count, int sm_count, cudaStream_t s);
cudaError_t launch_fe_tbs(const FeParams& p, cudaStream_t s);
cudaError_t launch_fe_finish(const FeParams& p, const uint8_t* status, cudaStream_t s);

// ---- whole get-entries response bodies (ctmr_json.cu, ctmr_process_raw_bodies) --------------------------------------
// one body of a chunk as uploaded
struct BodyDesc {
    uint64_t staged_off;  // in BodyParams.text
    uint64_t text_off;    // in ctmr_body_batch.text
    uint32_t len;
    uint32_t max;         // entries requested
    uint32_t slot0;       // first of the body's `max` slots of the walk's spans (sum of max over earlier bodies)
    uint32_t pad;
};
static_assert(sizeof(BodyDesc) == 32, "BodyDesc layout");

// per 64-byte block of the staged text: tokens outside strings (structural characters, opening quotes, bytes of
// scalars), unescaped quotes, backslashes, and characters that make a string invalid
struct BlockMasks {
    unsigned long long tok, quote, bs, bad;
};

struct BodyParams {
    const uint8_t* text;       // staged bodies (16 bytes of slack before, 64 after the stage)
    uint64_t spare;            // unescaped strings go to text + spare + their offset
    const BodyDesc* bodies;    // [n_bodies]
    uint32_t n_bodies;
    unsigned long long* starts;  // [blocks + 1] body start bits
    uint8_t* trans;            // [blocks] carry function of each block (4 x 2 bits)
    uint8_t* carry;            // [blocks] composed functions of the blocks before
    BlockMasks* masks;         // [blocks]
    uint32_t* stack;           // container kinds deeper than 63 levels: bit staged_off + depth
    uint8_t* body_status;      // [n_bodies] CTMR_BODY_*
    uint32_t* body_count;      // [n_bodies + 1] entries of OK bodies (0 otherwise)
    uint32_t* body_base;       // [n_bodies + 1] exclusive scan of body_count
    uint64_t* s_off[2];        // [sum of max] the walk's spans by body slot, staged offsets (~0: absent or null)
    uint32_t* s_len[2];
    uint8_t* s_esc;
    uint64_t* off[2];          // [entries] dense: where fe_decode reads each string (leaf_input, extra_data)
    uint32_t* len[2];
    uint64_t* abs_off[2];      // [entries] dense: the string's offset in the caller's text, its escaped length
    uint32_t* raw_len[2];
    uint8_t* esc;              // [entries] bit 0: leaf_input held a backslash, bit 1: extra_data did
};

size_t json_scan_temp_bytes(uint64_t blocks, uint64_t bodies);
// classify, walk, compact and unescape the n_bodies bodies of `bytes` staged bytes with `sparse` = sum of max slots;
// the entry count is left in body_base[n_bodies].  *launches: kernels issued.
cudaError_t launch_json_bodies(const BodyParams& p, uint64_t bytes, uint64_t sparse, void* temp, size_t temp_bytes, cudaStream_t s,
                               uint32_t* launches);

// ---- static-ct-api data tiles (ctmr_tiles.cu, ctmr_process_tiles) ------------------------------------------------
// one tile of a chunk as uploaded: where it sits in the staging buffer and in the caller's data
struct TileDesc {
    uint64_t staged_off;  // in TileParams.data
    uint64_t data_off;    // in ctmr_tile_batch.data
    uint64_t index;       // N of tile/data/<N>
    uint32_t len;
    uint32_t first;       // chunk-local index of the tile's first entry
    uint32_t width;
    uint32_t pad;
};
static_assert(sizeof(TileDesc) == 40, "TileDesc layout");

// fingerprint -> dense issuer index (ctmr_register_chain_certs): open addressing on the fingerprint's first 8 bytes
struct FpSlot {
    uint32_t w[8];  // SHA-256 fingerprint, bytes in order
    uint32_t idx;   // dense issuer index or CTMR_ISSUER_BAD
    uint32_t used;
    uint64_t pad;
};
static_assert(sizeof(FpSlot) == 48, "FpSlot layout");
struct FpTable {
    const FpSlot* slots;
    uint64_t mask;
};

struct TileParams {
    const uint8_t* data;       // staged tile bytes (16 bytes of slack before, 64 after)
    const TileDesc* tiles;     // [n_tiles]
    uint32_t n_tiles;
    uint64_t n;                // entries = sum of widths
    uint8_t* tile_bad;         // [n_tiles]
    uint64_t* entry_off;       // [n] TileLeaf start in data
    uint32_t* entry_tile;      // [n] chunk-local tile
    uint32_t* te_len;          // [n] bytes of the TimestampedEntry
    uint64_t* leaf_index;      // [n]
    uint64_t* leaf_data_off;   // [n] the path's certificate, offset in the caller's data
    unsigned int* first_stop;  // [1] lowest chunk-local tile holding an unknown Chain[0] fingerprint
    uint8_t* leaf_hash;        // [n][32]
    FeParams fe;               // per-entry outputs shared with the get-entries front end; fe.decoded = data
};

cudaError_t launch_tile_split(const TileParams& p, cudaStream_t s);
cudaError_t launch_tile_frame(const TileParams& p, cudaStream_t s);
cudaError_t launch_tile_issuer(const TileParams& p, const FpTable& tab, cudaStream_t s);
cudaError_t launch_tile_leaf_hash(const TileParams& p, cudaStream_t s);
cudaError_t launch_fingerprints(const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint8_t* fps, cudaStream_t s);

// ---- the logs' Merkle trees (ctmr_merkle.cu, ctmr_process_*_tree / ctmr_process_*_trees) -------------------------------
// The trees of one call live on the device: each caller's ctmr_tree, plus the lowest log position of a leaf that is
// missing in the chunk being folded (~0 when none).
struct TreeDev {
    ctmr_tree t;
    unsigned long long missing;
};

// One tree's part of a chunk: its entries are order[off .. off + cnt) (chunk entries, in log order), entry order[off + j]
// is log position first_pos + j.  The fold takes [t.size, end), where end is the first missing leaf at or above t.size,
// or first_pos + cnt; nothing when t.size < first_pos (an earlier chunk stopped this tree).
struct FoldTree {
    uint64_t first_pos;
    uint32_t tree;  // index into FoldChunk::trees
    uint32_t off;
    uint32_t cnt;   // > 0
    uint32_t skip;  // leaves first_pos .. first_pos + skip - 1 were in the tree before the call (a first tile that holds
                    // its size): the range fold starts after them; the fold into a tree reads t.size instead
};
static_assert(sizeof(FoldTree) == 24, "FoldTree layout");

// One chunk's leaves: leaf hash rows [chunk entries][32].  Entry e has no leaf when flags[e * stride] == match.  The
// chunk folds into n_desc trees; desc is ordered by off, and order (NULL: the identity) lists the chunk's entries grouped
// by tree, `total` of them (entries of no tree are left out).
struct FoldChunk {
    TreeDev* trees;
    const FoldTree* desc;
    uint32_t n_desc;
    uint32_t stride;
    const uint32_t* order;
    uint64_t total;
    const uint8_t* leaves;
    const uint8_t* flags;
    uint32_t match;
};

// get-entries leaves: SHA-256(0x00 || decoded leaf_input) of p.n entries -> rows[n][32]; rows of bad leaf_inputs are not written
cudaError_t launch_raw_leaf_hash(const FeParams& p, uint8_t* rows, cudaStream_t s);
// Folds a chunk into its trees: one launch for the missing leaves, one per level of the widest tree range, for all trees
// (level buffers lvl[2], each [total / 2 + 2 * n_desc][32]), one to commit the new sizes.  hdesc is the host copy of
// f.desc (the level loop's bounds).  Returns the number of launches in *launches.
cudaError_t launch_tree_fold(const FoldChunk& f, const FoldTree* hdesc, uint8_t* const lvl[2], cudaStream_t s, uint32_t* launches);
// the roots of trees[0, n) from their edges, rows of clear bits zeroed
cudaError_t launch_tree_root(TreeDev* trees, uint32_t n, cudaStream_t s);

// ---- the trees of a group call (ctmr_group_process_*_tree(s)): members 1.. fold their chunk into ranges ---------------
// One tree's part of a member's chunk as the canonical decomposition of its leaves [begin, end) into complete subtrees.
// begin = first_pos + skip; end is first_pos + cnt, or the member's first leaf at or above begin that is missing.  At
// level l the range covers nodes [A_l, B_l), A_l = ceil(begin / 2^l), B_l = end >> l; an odd A_l leaves node A_l as
// left[l], an odd B_l leaves node B_l - 1 as right[l], and the pairs between make level l + 1.  Rows of other levels are
// not written.  The home member (member 0, which holds the trees) appends the range when begin is the tree's size.
struct TreeRange {
    uint64_t begin, end;
    uint32_t tree;  // index into the call's trees
    uint32_t pad;
    uint8_t left[64][32];
    uint8_t right[64][32];
};
static_assert(sizeof(TreeRange) == 4120 && sizeof(TreeRange) % 8 == 0, "TreeRange layout: rows stay 8-byte aligned");

// The ranges of members 1..members (of one round) on the home member: member r's n[r - 1] ranges, ordered by tree, at
// recv + (r - 1) * stride.
struct RangeSet {
    const TreeRange* recv;
    uint32_t stride;
    uint32_t members;
    uint32_t n[kMaxWorld];
};

// Folds a chunk into one range per tree, out[i] for f.desc[i] (f.trees is not read): the launches of launch_tree_fold
// (missing leaves, one per level of the widest tree range, commit), with miss[cap] as the missing-leaf words.  miss
// must hold ~0 before the first chunk; each commit leaves it so.
cudaError_t launch_range_fold(const FoldChunk& f, const FoldTree* hdesc, uint8_t* const lvl[2], TreeRange* out, unsigned long long* miss,
                              cudaStream_t s, uint32_t* launches);
// One launch, one thread per tree of trees[0, n): appends the members' ranges of that tree in member order, each only
// when its begin is the tree's size, so that a tree stopped earlier keeps its size.
cudaError_t launch_tree_merge(TreeDev* trees, uint32_t n, const RangeSet& set, cudaStream_t s);

}  // namespace ctmr
