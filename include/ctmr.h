/*
 * ctmr.h -- C ABI of the H100-native CT-entry map/reduce hot path (libctmr.so).
 *
 * This is the drop-in boundary for ONE path of jcjones/ct-mapreduce (@739eda2): the per-entry
 * worker and its two reducers.  A Go host binds these entry points with cgo (INTEGRATION.md shows
 * the stub) and calls them in place of the loop body of
 *     (*LogSyncEngine).insertCTWorker        cmd/ct-fetch/ct-fetch.go:191-245
 *     certIsFilteredOut                      cmd/ct-fetch/ct-fetch.go:44-70
 *     (*FilesystemDatabase).Store            storage/filesystemdatabase.go:158-211
 *     (*KnownCertificates).WasUnknown/Count  storage/knowncertificates.go:38-63
 *     (*IssuerMetadata).Accumulate (the seenExpDateBefore bit)  storage/issuermetadata.go:92-108
 *     NewIssuer/Issuer.ID, NewSerial, NewExpDateFromTime        storage/types.go:109-130,171-178,339-346
 * while storage.StorageBackend, storage.RemoteCache and storage.CertDatabase
 * (storage/types.go:46-102) stay byte-identical on the Go side.
 *
 * Conventions (SURVEY.md §8(b)):
 *   - plain pointers and sizes only; no C++ or torch types; no exceptions cross the ABI.
 *   - functions return 0 (CTMR_OK) or a negative CTMR_E_* batch-level error; the text is
 *     available from ctmr_last_error(ctx) until the next call on that ctx.
 *   - per-entry problems are never return codes: they are status[i] (CTMR_ST_*), exactly like the
 *     reference's log-and-continue (ct-fetch.go:206-209,223-225,230-232).
 *   - the caller owns every input and output buffer; the library never keeps a caller pointer
 *     past return (cgo rule).  Device state lives in an opaque ctmr_ctx.
 *   - one ctmr_ctx per GPU, calls on a ctx are serialised by the caller; batches are ordered:
 *     every entry of call k precedes every entry of call k+1 for first-seen semantics.
 *   - several GPUs: ctmr_group_* (one process drives the GPUs of the box: what the Go host calls) or
 *     ctmr_peer_* (one process per GPU, tables attached through CUDA IPC).  Either way every set
 *     "serials::<expDate>::<issuer>" has one owner GPU, the map kernels insert straight into the owner's
 *     table over NVLink, and WasUnknown / counts are globally exact -- the fan-out is invisible above the ABI.
 *   - there is no CPU fallback: without a CUDA device ctmr_create fails with CTMR_E_NO_DEVICE.
 */
#ifndef CTMR_H
#define CTMR_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTMR_ABI_VERSION 3

/* ---- batch-level return codes ------------------------------------------------------------ */
enum {
    CTMR_OK = 0,
    CTMR_E_INVALID = -1,          /* bad argument */
    CTMR_E_CUDA = -2,             /* CUDA runtime error (text in ctmr_last_error) */
    CTMR_E_NOMEM = -3,            /* host or device allocation failed */
    /* The *_TABLE_FULL codes.  The batch path and preloads place a new record at most 4096 slots (kProbeLimit) past its
     * home slot, and fail with the table's code when the nearest free slot lies further.  Finding a record the table
     * holds has no such limit, and eviction, ctmr_resize and checkpoint loads place records again anywhere in the
     * table: they fail only when it has no free slot (DESIGN.md §3 "Probe rule"). */
    CTMR_E_TABLE_FULL = -4,       /* known-certificate table exhausted (cf. Redis OOM, rediscache.go:61-63) */
    CTMR_E_TOO_MANY_ISSUERS = -5, /* more distinct issuers than config.max_issuers */
    CTMR_E_NO_DEVICE = -6,        /* no usable CUDA device: the product path has no CPU fallback */
    CTMR_E_BATCH_TOO_LARGE = -7,  /* exceeds config.max_batch_* */
    CTMR_E_PAIR_TABLE_FULL = -8,  /* (issuer, expDate) table exhausted: raise config.pair_capacity_log2 */
    CTMR_E_META_TABLE_FULL = -9,  /* IssuerMetadata string-identity table exhausted: raise config.meta_capacity_log2 */
    CTMR_E_PEER_TIMEOUT = -10,    /* a rank of the group did not reach a barrier (a peer failed or the calls diverged) */
    CTMR_E_PEER = -11,            /* peer access / CUDA IPC between the GPUs of a group is not available */
    CTMR_E_UNKNOWN_ISSUER = -12,  /* ctmr_process_tiles: a Chain[0] fingerprint is not registered (ctmr_frontend.h) */
    CTMR_E_PEER_FAILED = -13      /* another rank's part of this collective call failed before any work (ctmr_frontend.h) */
};

/* ---- per-entry status -------------------------------------------------------------------- */
enum {
    CTMR_ST_OK = 0,               /* reached Store (counted by insertCTWorker.Inserted, ct-fetch.go:235) */
    CTMR_ST_PARSE_ERR = 1,        /* "Problem decoding certificate", ct-fetch.go:206-209 */
    CTMR_ST_FILTER_CA = 2,        /* certIsFilteredOut.CA, ct-fetch.go:47-50 */
    CTMR_ST_FILTER_EXPIRED = 3,   /* certIsFilteredOut.expired, ct-fetch.go:52-55 */
    CTMR_ST_FILTER_CN = 4,        /* certIsFilteredOut.cn-filtered, ct-fetch.go:57-68 */
    CTMR_ST_NO_ISSUER = 5,        /* len(Chain) < 1, ct-fetch.go:215-219 */
    CTMR_ST_ISSUER_PARSE_ERR = 6, /* "Problem decoding issuing certificate", ct-fetch.go:221-225 */
    CTMR_ST_SERIAL_TOO_LONG = 7,  /* serial INTEGER longer than CTMR_MAX_SERIAL octets (documented limit) */
    CTMR_ST__COUNT = 8
};

#define CTMR_MAX_SERIAL 39u            /* octets of raw serial a key record holds (RFC 5280 allows 20) */
#define CTMR_ISSUER_NONE 0xFFFFFFFFu   /* issuer_idx value for "entry has no chain" */
#define CTMR_ISSUER_BAD 0xFFFFFFFEu    /* dense index of an issuer certificate that failed to parse */

/* config.flags */
#define CTMR_F_NO_FINGERPRINT 1u /* skip SHA-256(leaf DER); the reference itself never computes it (SURVEY §0 M3) */

typedef struct ctmr_ctx ctmr_ctx;

typedef struct ctmr_config {
    uint32_t struct_size;        /* sizeof(ctmr_config), for ABI evolution */
    int32_t device;              /* CUDA device ordinal */
    uint64_t table_capacity;     /* known-certificate slots (64 B each), rounded up to a power of two */
    uint64_t max_batch_entries;  /* ceiling for one ctmr_process_batch call (sizes device staging); 0 = 1<<20 */
    uint64_t max_batch_bytes;    /* ceiling for the leaf blob of one call; 0 = 2 KiB * max_batch_entries */
    uint32_t max_issuers;        /* distinct issuers over the ctx lifetime; 0 = 65536 */
    uint32_t pair_capacity_log2; /* (issuer, exp-hour) first-seen table, log2 slots; 0 = 24 */
    const uint8_t* issuer_cn_filter; /* raw config value issuerCNFilter (config/config.go:193): split on ',' */
    uint32_t issuer_cn_filter_len;   /*   without trimming, HasPrefix on raw CN bytes (ct-fetch.go:57-63)      */
    uint32_t log_expired_entries;    /* config logExpiredEntries (config/config.go:188) */
    uint32_t flags;                  /* CTMR_F_* */
    uint32_t meta_capacity_log2;     /* IssuerMetadata string-identity table (issuer DN / CRL-DP bytes), log2 slots; 0 = 20, max 26 */
    uint64_t max_round_entries;      /* groups only: the most entries one GPU maps per round of ctmr_process_device
                                      * (= ceil(4n / (4R - 3)), R = ctmr_peer_rounds()); sizes the key-exchange regions (78 bytes x
                                      * GPUs x 3 per entry).  0 = the host pipeline's stage size (max_batch_entries) */
} ctmr_config;

/* Caller-allocated per-entry outputs, each [n]; any pointer may be NULL to skip that copy-back. */
typedef struct ctmr_out {
    uint8_t* status;            /* CTMR_ST_* */
    uint8_t* sha256;            /* [n][32] SHA-256 of the leaf DER (crypto/sha256.Sum256(cert.Raw)) */
    int64_t* exp_hour;          /* floor(NotAfter/3600 s): NewExpDateFromTime, storage/types.go:339-346 */
    uint32_t* serial_off;       /* raw serial content octets (NewSerial, storage/types.go:171-178):   */
    uint32_t* serial_len;       /*   offset inside the entry's DER, and length                          */
    uint8_t* was_unknown;       /* KnownCertificates.WasUnknown result, storage/knowncertificates.go:38-55 */
    uint8_t* first_issuer_hour; /* 1 iff Accumulate would return seenExpDateBefore == false (issuermetadata.go:95-108) */
    /* IssuerMetadata's string reducers (SURVEY.md §8(f)-1): spans of the two strings Accumulate looks at, and
     * first-seen bits so that the host only formats / parses them for candidates, not for every new certificate */
    uint32_t* issuer_name_off;  /* issuer Name (full TLV) inside the entry's DER: source of Issuer.String() (issuermetadata.go:94) */
    uint32_t* issuer_name_len;
    uint32_t* crldp_off;        /* cRLDistributionPoints extnValue content (issuermetadata.go:111), len 0 = absent */
    uint32_t* crldp_len;
    uint8_t* first_issuer_dn;   /* 1 iff was_unknown and no earlier new certificate of this issuer had the same Name bytes */
    uint8_t* first_crldp;       /* 1 iff was_unknown, extension present, and its bytes are new for this issuer */
    /* PEM of the NEW certificates, encoded on the device (SURVEY.md §8(f)-3): what Store hands to
     * StorageBackend.StoreCertificatePEM (storage/filesystemdatabase.go:171-175,197-198), i.e.
     * pem.EncodeToMemory(&pem.Block{Type: "CERTIFICATE", Bytes: cert.Raw}).  Optional as a group. */
    uint8_t* pem;               /* [pem_cap] texts of the entries with was_unknown == 1, back to back in entry order */
    uint64_t pem_cap;           /* too small => CTMR_E_BATCH_TOO_LARGE */
    uint64_t* pem_off;          /* [n+1]: entry i's text = pem[pem_off[i] .. pem_off[i+1]), empty unless new */
} ctmr_out;

/* ---- lifecycle ---------------------------------------------------------------------------- */
uint32_t ctmr_abi_version(void);
int ctmr_create(const ctmr_config* cfg, ctmr_ctx** out);      /* replaces GetConfiguredStorage wiring, engine/engine.go:19-48 */
void ctmr_destroy(ctmr_ctx* ctx);
const char* ctmr_last_error(ctmr_ctx* ctx);                   /* ctx may be NULL: error of the last failed ctmr_create */

/* Pinned host memory for batch packing (the Go batcher packs entries straight into it). */
void* ctmr_host_alloc(size_t bytes);
void ctmr_host_free(void* p);

/* ---- issuers ------------------------------------------------------------------------------ */
/* Parses n issuer certificates (x509.ParseCertificate(Chain[0]), ct-fetch.go:221), computes
 * Issuer.ID() digests (SHA-256 of RawSubjectPublicKeyInfo, storage/types.go:124-130,155-159) on the
 * GPU and assigns ctx-lifetime dense indices in order of first appearance.  HOST buffers.
 * dense_idx_out[k] = dense index, or CTMR_ISSUER_BAD when certificate k does not parse. */
int ctmr_register_issuers(ctmr_ctx* ctx, const uint8_t* issuer_blob, const uint64_t* issuer_offsets /* [n+1] */,
                          uint32_t n, uint32_t* dense_idx_out);
/* digest (32 octets) of a dense index; base64url of it is Issuer.ID() */
int ctmr_issuer_digest(ctmr_ctx* ctx, uint32_t dense_idx, uint8_t digest_out[32]);
uint32_t ctmr_issuer_count(ctmr_ctx* ctx);

/* ---- the hot path, HOST buffers (what the Go shim calls) ----------------------------------- */
/* One call = one batch drained from entryChan (ct-fetch.go:132,191).  blob holds the n leaf DERs
 * back to back (entry i = blob[offsets[i] .. offsets[i+1])); issuer_* hold the batch's distinct
 * Chain[0] certificates and issuer_idx[i] selects one (CTMR_ISSUER_NONE = no chain).
 * now_unix_ns replaces time.Now() at ct-fetch.go:52.  Copies host->device, runs the kernels,
 * copies the requested outputs back; synchronous.
 * After a failure (rc != 0) the outputs are undefined and part of the batch may already be in the tables; the
 * call's entry indices are consumed either way, so replaying the batch is safe in the reference's own sense
 * (idempotent replays, SURVEY §5): entries that were inserted read as known, never as unknown twice.  A replay does
 * not issue the write-back of those entries: ctmr_rollback to the call's start first (see "rollback"). */
int ctmr_process_batch(ctmr_ctx* ctx, const uint8_t* blob, const uint64_t* offsets /* [n+1] */, uint64_t n,
                       const uint8_t* issuer_blob, const uint64_t* issuer_offsets /* [n_issuers+1] */,
                       uint32_t n_issuers, const uint32_t* issuer_idx /* [n] */, int64_t now_unix_ns,
                       ctmr_out* out);

/* ---- reducers' read side ------------------------------------------------------------------- */
/* Per-issuer unique-certificate counts = sum over expDates of KnownCertificates.Count()
 * (cmd/storage-statistics/storage-statistics.go:44-53).  *n in: capacity, out: issuers written. */
int ctmr_issuer_counts(ctmr_ctx* ctx, uint8_t* digests /* [cap][32] */, uint64_t* counts /* [cap] */, size_t* n);
/* SetCardinality("serials::<expDate>::<issuer>"), storage/knowncertificates.go:57-63 */
int ctmr_set_cardinality(ctmr_ctx* ctx, int64_t exp_hour, const uint8_t issuer_digest[32], uint64_t* count_out);
/* entries per status since create, indexed by CTMR_ST_* (the certIsFilteredOut.* / Inserted counters) */
int ctmr_status_counters(ctmr_ctx* ctx, uint64_t out[CTMR_ST__COUNT]);
int ctmr_table_stats(ctmr_ctx* ctx, uint64_t* slots_used, uint64_t* capacity);

/* ---- warm start / checkpoint (SURVEY.md §8(f)-4) -------------------------------------------- */
/* Seed the known-certificate table from pre-existing state, e.g. the members of the Redis set
 * "serials::<expDate>::<issuer>" read back with KnownCertificates.Known() (storage/knowncertificates.go:65-96):
 * `n` serials, serial i = serial_blob[serial_offsets[i] .. serial_offsets[i+1]).  Preloaded keys count as
 * seen before every batch: WasUnknown answers false for them, per-issuer counts include them, and the
 * (issuer, expDate) pair counts as already allocated.  HOST buffers. */
int ctmr_preload_known(ctmr_ctx* ctx, int64_t exp_hour, const uint8_t issuer_digest[32], const uint8_t* serial_blob,
                       const uint64_t* serial_offsets /* [n+1] */, uint64_t n);
/* Redis TTLs: WasUnknown puts EXPIREAT(expDate) on every "serials::<expDate>::<issuer>" set
 * (storage/knowncertificates.go:44-47,98-104; expDate = hour-truncated NotAfter, storage/types.go:371-373), so
 * as time passes whole sets vanish from the reference's state.  This call applies that to the device state:
 * every set with expDate <= now is dropped (its serials are unknown again, it stops counting towards
 * ctmr_issuer_counts / ctmr_set_cardinality, its slots are reclaimed).  IssuerMetadata's seenExpDateBefore memo
 * is process memory in the reference and is kept.  Call it between batches, e.g. once per hour. */
int ctmr_evict_expired(ctmr_ctx* ctx, int64_t now_unix_sec, uint64_t* evicted_out);
/* Snapshot of the derived device state (tables, histograms, issuer registry, next entry index) into a
 * caller buffer, and its restoration into a ctx created with the same capacities.  ctmr_snapshot_size
 * gives the bytes needed.  The reference's analogue is the state it keeps in Redis between runs
 * (storage/rediscache.go); its own resume logic is cmd/ct-fetch/ct-fetch.go:288-300.
 * To move the state into other capacities or another number of GPUs, use ctmr_checkpoint_* below. */
int ctmr_snapshot_size(ctmr_ctx* ctx, uint64_t* bytes);
int ctmr_snapshot_save(ctmr_ctx* ctx, uint8_t* buf, uint64_t cap, uint64_t* written);
int ctmr_snapshot_load(ctmr_ctx* ctx, const uint8_t* buf, uint64_t bytes);

/* ---- portable checkpoint -------------------------------------------------------------------- */
/* The live content of the state (not its slot layout), loadable into ANY shape: one ctx, a group of any size, or peer
 * ranks of any world size, of any capacities that hold the content.  A checkpoint is one or more PARTS: a ctx or a group
 * saves one part; a ctx attached to peers saves its own, so a world-rank deployment saves `world` parts.  A load takes
 * every part of one checkpoint, in any order.  HOST buffers.
 *
 * Part layout (little-endian): a 128-byte header -- magic "CTMRCKP1", u32 part index, u32 part count, u64 n_issuers,
 * u64 next_index, u64 status counters [CTMR_ST__COUNT] of this part, u64 keys, pairs, string identities, u64 0 -- then
 * the registry digests [n_issuers][32] in dense-index order (every part carries the same list), the ready key slots
 * (64 B each, as they lie in the table: inv_first keeps the first-seen index), the (issuer, hour) slots (32 B: key,
 * inv_first, count) and the string identities (32 B).  Bytes = 128 + 32 n_issuers + 64 keys + 32 (pairs + strings).
 * Two saves of one state are byte-equal.
 *
 * Save compacts the tables through a bounded staging buffer (no second table-sized allocation).  Load replaces the
 * target's state: its tables are cleared, the registry rebuilt (digest i gets index i again), every member / rank
 * inserts the records it owns under the TARGET's world (per-issuer counts are rebuilt from the keys), member 0 / rank 0
 * holds the status counters (the sum over the parts), and the next index is the checkpoint's.  Like
 * ctmr_snapshot_load, the Chain[0] mirror and the tiles' fingerprints are cleared: chain certificates are registered
 * again and get the same dense indices.  Failures:
 *   CTMR_E_INVALID          bad magic, truncation, parts that disagree (count, index given twice or missing,
 *                           registry, next index), a NULL part: the target is untouched
 *   CTMR_E_TOO_MANY_ISSUERS the registry exceeds the target's max_issuers: the target is untouched
 *   CTMR_E_TABLE_FULL / CTMR_E_PAIR_TABLE_FULL / CTMR_E_META_TABLE_FULL (a target table too small), and
 *   CTMR_E_INVALID for a record out of range (issuer >= n_issuers, serial longer than CTMR_MAX_SERIAL, a slot not
 *   ready): the target is as after a reset with the checkpoint's registry, its next index unchanged
 * On a ctx attached to peers the three calls are COLLECTIVE.  Save: a barrier, each rank writes its own part, a barrier.
 * Load: the ranks agree on their checks before any change (a rank whose checks fail returns its error, the others
 * CTMR_E_PEER_FAILED, nothing changes), and on the outcome of their inserts (a failure on one rank is every rank's).
 * A member ctx of an in-process group is refused: use ctmr_group_checkpoint_*. */
int ctmr_checkpoint_size(ctmr_ctx* ctx, uint64_t* bytes);
int ctmr_checkpoint_save(ctmr_ctx* ctx, uint8_t* buf, uint64_t cap, uint64_t* written);
int ctmr_checkpoint_load(ctmr_ctx* ctx, const uint8_t* const* parts, const uint64_t* part_bytes, uint32_t n_parts);

/* ---- delta checkpoint --------------------------------------------------------------------------------------------- */
/* The records added since an earlier checkpoint, and their application on top of the state that checkpoint gave.  Every
 * record keeps its first-seen index (eviction, resize and loads keep it), so the records added since a checkpoint taken
 * at next index N are the live ones first seen at or above N.  A delta save reads the whole table on the device and
 * copies only those records to the host.  HOST buffers.
 *
 * Part layout: the checkpoint's, with its own 128-byte header -- magic "CTMRDLT1", u16 part index, u16 part count,
 * u32 n_issuers, u64 since, u64 next_index, i64 evict_now, u64 status counters [CTMR_ST__COUNT] of this part (totals,
 * not increments), u64 keys, pairs, string identities -- then the WHOLE registry [n_issuers][32] in dense-index order,
 * the ready key slots, the (issuer, hour) slots and the string identities whose first-seen index is >= since (64, 32
 * and 32 B as in a checkpoint).  Bytes = 128 + 32 n_issuers + 64 keys + 32 (pairs + strings).  evict_now is the highest
 * now_unix_sec passed to ctmr_evict_expired while the state stood at next index >= since (INT64_MIN: none); an
 * eviction before `since` is already in the state the delta goes on, and repeating it would drop the keys stored after
 * it.  A ctx or a group saves one part; a rank attached to peers saves its own, collectively, as ctmr_checkpoint_save.
 * Two saves of one state with the same since are byte-equal.  In both headers the next index is the u64 at byte 24, so
 * the since of the next delta can be read from the last part saved (a group has no ctmr_next_index).  Deltas follow the
 * handle's next index: ctmr_map_device / ctmr_process_device take their indices from the caller and do not move it.
 *
 * Save refusals (CTMR_E_INVALID, nothing written): since > next index; since below the DELTA FLOOR, the next index at
 * the last call that removed records other than by eviction (ctmr_reset_device / ctmr_group_reset, ctmr_snapshot_load,
 * ctmr_checkpoint_load, and a failed ctmr_checkpoint_apply, which leaves a reset state).  A delta cannot express a
 * reset: take a full checkpoint there.  ctmr_resize and a successful apply keep every record and its index, and do not
 * move the floor.
 *
 * Apply puts one delta (every part of it, any order) on top of the target's state; the target may have any shape and
 * capacities.  Every check runs before anything changes: magic and truncation, part count and indices, the same since,
 * next index and registry in every part, the target's next index == since (deltas go on in order, with no gap), the
 * target's registry a prefix of the delta's, the registry within max_issuers.  Then: the new digests are registered in
 * order (digest i keeps index i); if evict_now (the highest over the parts) is above every eviction the target made at
 * its current index, every member evicts at evict_now; the records go in as a load puts them (each member / rank keeps
 * the ones it owns); every (issuer, hour) count and the per-issuer histogram are rebuilt from the live keys; the status
 * counters (on member 0 / rank 0) and the next index become the delta's.  The Chain[0] mirror and the fingerprints stay.
 * Failures: a failed check (CTMR_E_INVALID; CTMR_E_TOO_MANY_ISSUERS) changes nothing; CTMR_E_*TABLE_FULL or a record out
 * of range during the inserts leaves the target as after a reset, with the delta's registry: resize, then replay the
 * base checkpoint and its deltas.  On peer ranks apply is collective with ctmr_checkpoint_load's two agreements.
 *
 * The contract: a full checkpoint C0 at next index N0, deltas D1 (since N0) ... Dk (since N(k-1)) saved later, with any
 * calls between them (batches, front-end calls, preloads, evictions, resizes).  ctmr_checkpoint_load(C0) and
 * ctmr_checkpoint_apply(D1) ... (Dk) into any shape give every later call the result that loading a full checkpoint
 * taken at Dk's point gives in that shape: every ctmr_out field and front-end output, ctmr_issuer_counts,
 * ctmr_set_cardinality, ctmr_status_counters, ctmr_next_index and the CRL calls; the checkpoint records, parsed and
 * sorted, are equal.  A member ctx of an in-process group is refused: use ctmr_group_checkpoint_*. */
int ctmr_checkpoint_delta_size(ctmr_ctx* ctx, uint64_t since, uint64_t* bytes);
int ctmr_checkpoint_delta_save(ctmr_ctx* ctx, uint64_t since, uint8_t* buf, uint64_t cap, uint64_t* written);
int ctmr_checkpoint_apply(ctmr_ctx* ctx, const uint8_t* const* parts, const uint64_t* part_bytes, uint32_t n_parts);

/* ---- resize ------------------------------------------------------------------------------------------------------- */
/* The known-certificate, (issuer, expDate) and string-identity tables in other sizes, rehashed on the device: what
 * checkpoint save, destroy, create, checkpoint load and registering the chain certificates again would do, without
 * leaving the GPU.  0 keeps a table's current size; table_capacity is rounded up to a power of two as in ctmr_create.
 *
 * Equivalence.  After ctmr_resize(ctx, T, P, M) returns CTMR_OK, every later call returns exactly what it would return on
 * a ctx created with capacities (T, P, M) and the same other config, loaded with ctmr_checkpoint_load from a
 * ctmr_checkpoint_save taken just before the resize: every ctmr_out field, the front-end calls, ctmr_issuer_counts,
 * ctmr_set_cardinality, ctmr_status_counters, ctmr_next_index, ctmr_revoked_known, the cascade and the stash.  Checkpoint
 * records (parsed and sorted) are equal; slot order, and so the checkpoint bytes, may differ.
 * Kept state.  Everything else stays as it was: the issuer registry (same dense indices), the registered chain
 * certificates, the Chain[0] mirror, the tiles' fingerprint table and the staging buffers.  Unlike the checkpoint route,
 * nothing is registered again.
 * Records.  A resize carries what a checkpoint carries: the ready known-certificate slots of the current epoch with their
 * first-seen index, every occupied (issuer, expDate) slot (an evicted set's, count 0, included) and every occupied
 * string-identity slot.  Slots left by earlier epochs (ctmr_reset_device) are empty and are not carried.  The per-issuer
 * counts are rebuilt from the keys, as a checkpoint load rebuilds them.
 * Shrinking is allowed.  A target too small for its records fails with the table's own CTMR_E_TABLE_FULL,
 * CTMR_E_PAIR_TABLE_FULL or CTMR_E_META_TABLE_FULL.
 * All or nothing.  On any failure (CTMR_E_NOMEM for the new tables, a *_TABLE_FULL, a CUDA error) the ctx or every member
 * of the group is left exactly as it was: the same tables, a checkpoint byte-equal to the one before, usable; the rehash
 * raises no flag that ctmr_check_device would report later.
 * Peak memory.  The old and the new tables exist together; a group builds every member's new tables before it frees any
 * old ones, so the peak on a device is old plus new for every member on it.  A shape that does not fit is CTMR_E_NOMEM
 * with nothing changed: move the state through ctmr_checkpoint_save / ctmr_checkpoint_load instead, which holds it in
 * host memory between the two tables.
 * Refusals (CTMR_E_INVALID, nothing touched): a NULL ctx; a member ctx of a group (use ctmr_group_resize); table_capacity
 * above 2^32 - 16 slots once rounded, pair_capacity_log2 above 32, meta_capacity_log2 above 26 (ctmr_create's limits);
 * a ctx on which ctmr_peer_export was called.  Its whole shared region, tables included, is behind a CUDA IPC handle whose
 * size the other ranks check at ctmr_peer_attach, and the table size must be the same on every rank: a rank resizes
 * before it exports, and ranks attached to each other resize through the checkpoint route.  The refusal comes before any
 * barrier, so no rank waits for it.
 * Not collective and not automatic: a full table still fails its batch with *_TABLE_FULL.  Watch ctmr_table_occupancy and
 * resize, or resize after a *_TABLE_FULL and replay the batch (safe by ctmr_process_batch's replay rule).
 * Cost: one pass over each old table and one scattered insert per record (DESIGN.md §3 "Resize"). */
int ctmr_resize(ctmr_ctx* ctx, uint64_t table_capacity, uint32_t pair_capacity_log2, uint32_t meta_capacity_log2);
/* used (live slots of the current epoch) and capacity (slots) of the three tables, in the order known-certificate,
 * (issuer, expDate), string identities; either array may be NULL.  One count pass per table.  A member ctx of a group
 * reports its own shard; ctmr_group_table_occupancy sums over the members. */
int ctmr_table_occupancy(ctmr_ctx* ctx, uint64_t used[3], uint64_t capacity[3]);

/* ---- rollback ----------------------------------------------------------------------------------------------------- */
/* Takes the device state back to the start of an earlier entry-taking call, so that "undo that call, run it again" gives
 * exactly the outputs of a clean run: the same was_unknown bits, the same write-back and the same indices.  Use it after a
 * failed batch (part of it may already be in the tables: its entries would read as known on a replay, and their
 * SetInsert and PEM write would never be issued) and when a tree root does not match the log's STH.
 *
 * Semantics.  After ctmr_rollback(ctx, N) returns CTMR_OK the ctx is in exactly the state a checkpoint taken when the
 * next index was N would load to, followed by ctmr_evict_expired(now) with the highest now evicted since N:
 *   - every key, (issuer, expDate) and string-identity slot whose first-seen index is >= N is gone; every other slot is
 *     unchanged, its first-seen index included;
 *   - every (issuer, expDate) count and the per-issuer histogram equal those of the remaining live keys;
 *   - the status counters equal their values at the start of the call that began at N;
 *   - the next index is N.
 * Not indexed, so kept: the issuer registry, the registered chain certificates, the Chain[0] mirror and the caller's
 * ctmr_tree structs (keep a copy of the trees from before the call and restore it).
 *
 * Valid targets.  N is the next index at the start of an entry-taking call of this ctx or group, failed calls included:
 * ctmr_process_batch, every front-end call (ctmr_frontend.h), ctmr_process_device and ctmr_preload_known.  Each call
 * start is a MARK: its next index and the status counters, copied on the device on the call's stream (no host wait).
 * The ctx keeps the last CTMR_ROLLBACK_MARKS marks; calls that start at the same index keep the first one's.
 * ctmr_process_device takes its indices from the caller and does not move the handle's next index, so its mark is at
 * the handle's next index: a rollback to it undoes the device call (its records at or above that index, its status
 * counts) only once a later host-buffer, front-end or preload call has moved the index past it.  A caller of the device
 * path alone reaches no earlier state this way (N == the next index does nothing); it keeps its own checkpoints.  The
 * chunks of a front-end call and a group's members take no mark of their own.
 * N == the current next index is valid and does nothing.  Refusals (CTMR_E_INVALID, nothing touched): N above the next
 * index, N not a mark, N below the delta floor (see "delta checkpoint"), a mark that has dropped out of the ring, a NULL
 * ctx, a member ctx of a group (use ctmr_group_rollback).  A reset, ctmr_snapshot_load and ctmr_checkpoint_load (and a
 * failed ctmr_checkpoint_apply) clear the marks as they move the delta floor; ctmr_resize keeps them.  Afterwards the
 * marks above N are gone, the eviction history at or above N counts as made at N (a later delta's evict_now stays
 * right), and the delta floor is unchanged.
 * Group.  The group's next index is the one checked; each member restores its own shard and status counters.
 * Peer ranks (ctmr_peer_attach, world > 1): COLLECTIVE.  The ranks agree on their checks first (every rank needs a mark
 * at N; a rank whose check fails returns its error, the others CTMR_E_PEER_FAILED, nothing changes); each rank then
 * rolls its own shard back, and a final agreement makes a failure on one rank every rank's.
 * Failures.  Every check comes before any work.  Among them, after waiting for the device, the error flag of each
 * member is read and cleared as ctmr_check_device does: a flag raised by an earlier call that nobody checked (an
 * asynchronous ctmr_process_device) is returned as that call's failure, with nothing rolled back; call again.  The
 * deletion works in place: a CUDA error after it started leaves that member's tables undefined and raises its error
 * flag (ctmr_check_device reports it), as eviction does; load a checkpoint.  On peer ranks the ranks whose own deletion
 * succeeded stand at N (next index, marks, tables) even when another rank's failed and they return CTMR_E_PEER_FAILED.
 * Cost: one pass over each table, then per cluster of occupied slots that holds a removed record, one walk over the
 * cluster from its first removed slot (DESIGN.md §3 "Rollback"). */
#define CTMR_ROLLBACK_MARKS 4096u
int ctmr_rollback(ctmr_ctx* ctx, uint64_t next_index);

/* ---- revoked known certificates (CRLite's join of CRLs with the serials:: sets) ------------------- */
/* Which revoked serials of an issuer's CRLs are known certificates, and in which "serials::<expDate>::<issuer>" set
 * (storage/knowncertificates.go:28-55)?  A CRL entry carries no expiry, so the set cannot be named; the call parses the
 * CRLs on the GPU (DESIGN.md "Revoked known certificates") and answers every entry from one pass over the table per chunk.
 *
 * Rules (RFC 5280 §5.1).  CertificateList ::= SEQUENCE { tbsCertList, AlgorithmIdentifier, BIT STRING } with nothing after
 * the signatureValue and nothing after the outer SEQUENCE.  TBSCertList: version INTEGER OPTIONAL (absent = v1, else 1 =
 * v2), signature AlgorithmIdentifier, issuer Name, thisUpdate Time, nextUpdate Time OPTIONAL, revokedCertificates SEQUENCE
 * OF entry OPTIONAL (absent = no entries), [0] EXPLICIT crlExtensions OPTIONAL, nothing after.  An entry is SEQUENCE {
 * userCertificate INTEGER (at least one octet), revocationDate Time, crlEntryExtensions Extensions OPTIONAL } with nothing
 * after it; a reasonCode (2.5.29.21) must be an ENUMERATED of one octet.  TLV headers and Time follow the certificate
 * walker (single-octet tags, minimal definite lengths; UTCTime pivots at 50, GeneralizedTime accepted).  Signatures are
 * not verified: tbs_off / tbs_len give the host the signed bytes.  Parity with Go's x509.ParseDERCRL /
 * ParseRevocationList is not pinned (as for ct-go in the front end): serials need not be minimal INTEGERs here.
 *
 * Match.  An entry is joined when its CRL is CTMR_CRL_OK and the entry is CTMR_RV_OK: its serial's raw content octets
 * must equal a key's raw serial (NewSerial, storage/types.go:171-178) under the dense issuer of issuer_digest.  Minimal
 * encodings of one integer are equal bytes; a non-minimal encoding on either side (00 01 against 01) does not match.
 *
 * Sizing.  The smallest entry is 18 bytes (SEQUENCE 2 + INTEGER 3 + a UTCTime without seconds 13), so entry_cap =
 * (total CRL bytes) / 18 always suffices.  With a smaller entry_cap the call writes only n_entries (the count needed) and
 * returns CTMR_E_BATCH_TOO_LARGE.  The CRLs are staged in chunks of whole CRLs of at most min(config.max_batch_bytes
 * as the pipeline caps it, 256 MiB) bytes, each chunk one pass over the table; a CRL larger than a chunk is
 * CTMR_E_BATCH_TOO_LARGE before any work.
 *
 * Read-only: no index is taken and no table, counter or registry changes, so the call may come between any other calls.
 * A member ctx of a group is refused with CTMR_E_INVALID: use ctmr_group_revoked_known.
 *
 * On a ctx attached to peers (ctmr_peer_attach, world > 1) the call is COLLECTIVE: every rank makes the same sequence of
 * collective calls (a mismatch is undefined), each with its OWN batch, which may be empty (n_crls == 0).  Each rank gets
 * the answers for its own CRLs only, and every output is what the call on one ctx holding the union of all ranks' tables
 * gives for that batch: known_exp_hour is the lowest hour over every rank's sets and known_sets the sum over the ranks.
 * The other ranks' batches make no difference to it.  Issuer digests are looked up in the shared registry (one that
 * only another rank registered is found), and the call stays read-only on every rank.  Failures:
 *   - the checks above (a NULL batch or output, a CRL outside data or larger than a chunk) run on every rank before any
 *     work; if one fails anywhere, that rank returns its error and the others CTMR_E_PEER_FAILED, n_entries is 0 and
 *     nothing else is written;
 *   - a later failure on any rank (CUDA, an allocation, a barrier that timed out) is every rank's: that rank returns its
 *     error, the others CTMR_E_PEER_FAILED, and the outputs are undefined;
 *   - entry_cap too small is the rank's own: it still answers the other ranks' entries and returns
 *     CTMR_E_BATCH_TOO_LARGE with the count needed, while the others succeed.
 * A rank whose binding refuses its arguments before calling must still make the call (a NULL batch will do).  Cost: a
 * CRL entry has no expiry, so an entry's sets may lie on any rank; every rank's records go to every rank, config.
 * max_round_entries (X, at least max_batch_entries) per rank and round, and each round is one pass over each rank's
 * shard.  A chunk takes ceil(the most entries any rank has in its chunk at that step / X) rounds (DESIGN.md "Revoked
 * known certificates").
 * Out of scope: signature verification, fetching, and the semantics of delta and indirect CRLs beyond crl_flags and
 * CTMR_RV_INDIRECT. */
enum { CTMR_CRL_OK = 0, CTMR_CRL_BAD = 1,          /* CertificateList / TBSCertList framing or fields */
       CTMR_CRL_BAD_ENTRIES = 2,                   /* revokedCertificates does not split into well-formed entries */
       CTMR_CRL_UNKNOWN_ISSUER = 3 };              /* digest not in the registry: parsed, nothing joined */
enum { CTMR_RV_OK = 0, CTMR_RV_INDIRECT = 1,       /* certificateIssuer entry extension (2.5.29.29): not joined */
       CTMR_RV_SERIAL_TOO_LONG = 2 };              /* longer than CTMR_MAX_SERIAL: no key can hold it */
#define CTMR_CRL_F_DELTA 1u                        /* crl_flags: deltaCRLIndicator (2.5.29.27) */
#define CTMR_CRL_F_IDP 2u                          /* crl_flags: issuingDistributionPoint (2.5.29.28) */

typedef struct ctmr_crl_batch {                    /* HOST buffers */
    const uint8_t* data; uint64_t data_bytes;
    const uint64_t* crl_off; const uint64_t* crl_len;   /* [n_crls] DER CertificateList */
    const uint8_t* issuer_digest;                       /* [n_crls][32] Issuer.ID() digest whose crl:: set named the URL */
    uint64_t n_crls;
} ctmr_crl_batch;

typedef struct ctmr_crl_out {                      /* caller-allocated, any pointer may be NULL */
    uint8_t* crl_status; uint8_t* crl_flags;       /* [n_crls] bit 0 deltaCRLIndicator, bit 1 issuingDistributionPoint */
    int64_t* this_update; int64_t* next_update;    /* unix seconds; next_update INT64_MIN when absent */
    uint64_t* tbs_off; uint32_t* tbs_len;          /* tbsCertList span: the host verifies the signature without a parse */
    uint64_t* issuer_name_off; uint32_t* issuer_name_len;
    uint64_t* crl_first; uint32_t* crl_entries;    /* the CRL's entries in the per-entry arrays */
    uint64_t* serial_off; uint8_t* serial_len;     /* [entry_cap] absolute in data: INTEGER content octets */
    int64_t* revoked_at; uint8_t* reason;          /* reasonCode (2.5.29.21), 0xFF when absent */
    uint8_t* entry_status;                         /* CTMR_RV_* */
    uint8_t* known;                                /* 1 iff a set serials::<h>::<issuer> in the table holds the serial */
    int64_t* known_exp_hour;                       /* the lowest such h (0 when not known) */
    uint32_t* known_sets;                          /* how many such h (more than 1 = serial reuse) */
    uint64_t entry_cap;
    uint64_t n_entries;                            /* written; on CTMR_E_BATCH_TOO_LARGE the count needed */
} ctmr_crl_out;
/* Per CRL: CTMR_CRL_BAD and CTMR_CRL_BAD_ENTRIES CRLs have no entries (crl_entries 0) and only crl_status is meaningful;
 * CTMR_CRL_OK and CTMR_CRL_UNKNOWN_ISSUER CRLs list every entry in order, entries of the CRLs back to back in CRL order.
 * serial_len saturates at 255: a serial of 256 or more content octets (always CTMR_RV_SERIAL_TOO_LONG, never joined)
 * reports 255, and its serial_off is still exact.
 * On a failed call (rc != 0) the outputs other than n_entries are undefined. */
int ctmr_revoked_known(ctmr_ctx* ctx, const ctmr_crl_batch* batch, ctmr_crl_out* out);

/* ---- CRLite filter cascade (the revoked / not-revoked Bloom cascade of the covered issuers) ------------------------- */
/* Builds CRLite's filter cascade straight from the table: only the serialized filter reaches the host (DESIGN.md
 * "Revoked cascade").  Same batch and match rule as ctmr_revoked_known; the batch holds the CRLs the caller accepts (their
 * signatures already verified, INTEGRATION.md §2d).
 *
 * Sets.  An issuer is COVERED when its digest appears in the batch, it is in the registry, and every one of its CRLs in the
 * batch is CTMR_CRL_OK (an issuer with a bad CRL must not claim its certificates valid).  A LIVE key record is a ready key
 * whose set has exp_hour * 3600 > now_unix_sec (the sets ctmr_evict_expired(now) keeps).  Of the live records of covered
 * issuers, R = those whose (issuer, raw serial) equals a CTMR_RV_OK entry of a CTMR_CRL_OK CRL (byte for byte, under
 * every hour), S = all the others.  Sizes count key records: a serial under two hours counts twice (a group's counts are
 * sums over its shards).
 *
 * Key and hash.  x = digest(32) || serial content octets (Issuer.ID()'s digest, then NewSerial's bytes).  Level l
 * (1-based) with m_l bits and k_l functions sets or tests the bits
 *     b_i = LE32(SHA-256(salt || LE32(i) || u8(l) || x)[0..4]) mod m_l,   i = 0 .. k_l - 1.
 * salt_len <= 32 (every message fits two SHA-256 blocks); a longer salt is CTMR_E_INVALID.
 *
 * Sizing: host IEEE double, in exactly this order, with C log, pow, sqrt and ceil:
 *     p_1 = 0.5 if |R| == 0 or |S| == 0, else min(0.5, |R| / (sqrt(2) * |S|));   p_l = 0.5 for l >= 2
 *     k_l = max(1, ceil(log(1 / p_l) / log(2)))
 *     m_l = max(8, ceil(-k_l * n_l / log(1 - pow(p_l, 1.0 / k_l))))   n_l = records included at level l
 * m_l >= 2^32 is CTMR_E_BATCH_TOO_LARGE (with bytes = 0).
 *
 * Build.  Level 1 includes I_1 = R and is tested against E_1 = S.  F_l = the records of E_l that level l contains (all
 * k_l bits set).  The cascade stops at the first empty F_l; otherwise I_{l+1} = F_l, E_{l+1} = I_l.  More than 255 levels
 * is CTMR_E_INVALID (the level is one octet): build again with another salt.
 *
 * Layout, integers little-endian:
 *     header      u16 2 (version), u8 0 (not inverted), u8 salt_len, salt[salt_len]
 *     each level  u8 2 (hash: SHA-256, first 32 bits), u32 m_l, u32 k_l, u8 l, ceil(m_l / 8) bytes of bits
 * Bit j is (byte[j >> 3] >> (j & 7)) & 1; the unused high bits of the last byte are zero.
 *
 * Query.  Walk the levels from 1 and stop at the first that does not contain x: x is revoked iff that level's number is
 * even.  If all L levels contain x, it is revoked iff L is odd.
 *
 * This follows Mozilla's filter-cascade version 2 as restated here.  Byte parity with filter-cascade or rust-cascade is
 * NOT pinned (neither is available to this build): this header and tests/cascade_model.py pin the format.
 *
 * The output is deterministic: it depends neither on table layout, group size nor thread order.  With cap too small (buf
 * may be NULL) the call returns CTMR_E_BATCH_TOO_LARGE and writes `bytes` and nothing else; a second call with that cap
 * returns exactly those bytes.  Read-only, like ctmr_revoked_known: no index is taken and no table, counter or registry
 * changes.  Argument checks are ctmr_revoked_known's (a NULL batch or output, a CRL outside data or larger than a chunk),
 * plus the salt's.  A member ctx of a group is refused with CTMR_E_INVALID (use ctmr_group_revoked_cascade).  Cost: one
 * pass over the table per CRL chunk, two more for level 1, and device scratch of one bit per table slot plus the include
 * lists and one level's bits (DESIGN.md "Revoked cascade").
 *
 * On a ctx attached to peers (world > 1) the call is COLLECTIVE: every rank makes it with its own batch, which may be
 * empty (n_crls == 0), and every rank passes the same now_unix_sec and the same salt.  The result is what the call on one
 * ctx would give that holds the union of every rank's table (every rank's checkpoint part loaded) and is passed the
 * concatenated batch, rank 0's CRLs first, then rank 1's, and so on: bytes, buf, issuers, levels, revoked and valid are
 * identical on every rank, and crl_status covers the rank's own CRLs.  Coverage is global: an issuer is covered when it
 * is registered, its digest appears in some rank's batch, and every CRL of it in every rank's batch is CTMR_CRL_OK (a
 * bad CRL on one rank uncovers its issuer on every rank); an issuer registered only by another rank is found, as in
 * ctmr_revoked_known.  Read-only on every rank.  Failures follow ctmr_revoked_known's peer rules:
 *   - the checks before any work (a NULL batch or output, a CRL outside data or larger than a chunk, salt_len > 32, a
 *     NULL salt with salt_len > 0) run on every rank: a rank that fails one returns its error, the others return
 *     CTMR_E_PEER_FAILED, and bytes is 0; nothing else is written;
 *   - a now_unix_sec or salt not equal to rank 0's: that rank returns CTMR_E_INVALID and the others CTMR_E_PEER_FAILED,
 *     before any work (R, S and every bit depend on them);
 *   - a later failure on any rank (CUDA, an allocation, a barrier timeout) is every rank's; outputs are undefined;
 *   - a cap too small on any rank (or a NULL buf) is CTMR_E_BATCH_TOO_LARGE on every rank, and every rank writes only
 *     bytes, which is the same everywhere.  Unlike ctmr_revoked_known's entry_cap, which only affects its own rank: the
 *     retry with the reported size is a collective call, so every rank retries together;
 *   - m_l >= 2^32 and more than 255 levels are as above; the sizes are agreed, so every rank reaches them together.
 * The collective form moves every rank's CRL entries to every rank through the exchange area and merges each level's
 * bits with an OR all-reduce there; DESIGN.md "Revoked cascade" gives its cost. */
typedef struct ctmr_cascade_out {   /* caller-allocated; HOST buffers */
    uint8_t* buf; uint64_t cap;     /* the serialized cascade */
    uint64_t bytes;                 /* written; on CTMR_E_BATCH_TOO_LARGE the bytes needed */
    uint8_t* crl_status;            /* [n_crls] CTMR_CRL_*, as ctmr_revoked_known; may be NULL */
    uint32_t issuers;               /* issuers covered */
    uint32_t levels;
    uint64_t revoked, valid;        /* key records in R and in S */
} ctmr_cascade_out;
int ctmr_revoked_cascade(ctmr_ctx* ctx, const ctmr_crl_batch* batch, int64_t now_unix_sec,
                         const uint8_t* salt, uint32_t salt_len, ctmr_cascade_out* out);

/* ---- CRLite stash (the revoked known certificates a published filter and its stashes miss) ------------------------- */
/* Between full filters CRLite publishes stashes: per issuer, the serials revoked since the filter.  This call computes the
 * next stash from the table and what was already published, with no state kept between runs; only the candidates the
 * filter misses reach the host (DESIGN.md "Revoked stash").
 *
 * Sets.  Covered issuers, live records and R are ctmr_revoked_cascade's with the same batch and now_unix_sec.  For each
 * key record of R, with x = digest || serial:
 *   in_filter   query(filter, x) is revoked (the query rule above, with the filter's own salt);
 *   in_stashes  otherwise, and an earlier stash lists (digest, serial);
 *   new         every other record of R.  The stash lists the distinct (digest, serial) pairs of the new records: a serial
 *               under two hours is one entry.
 * Counts are key records, as in the cascade: revoked == in_filter + in_stashes + (new key records).
 *
 * Stash layout, integers little-endian: any number of units back to back, each
 *     u32 n, u8 32 (hash length), digest[32], then n entries of u8 len, serial[len].
 * Byte parity with Firefox's cert_storage loader is NOT pinned: this header and tests/stash_model.py pin the format.  The
 * concatenation of stashes is a stash, so `stashes` is every stash published since `filter`, back to back (may be empty).
 * The output is deterministic: units in ascending order of digest bytes, only issuers with at least one entry; each
 * issuer's serials in ascending lexicographic byte order, a serial before any longer one it is a prefix of.  An empty
 * stash is 0 bytes and succeeds with any cap and a NULL buf.
 *
 * Checks before any work, each CTMR_E_INVALID (both inputs come from outside the library):
 *   - the filter must follow the layout above exactly: at least 4 bytes; version 2, not inverted, salt_len <= 32; at least
 *     one level; each level hash byte 2, 1 <= k <= 64, m >= 8, a level byte equal to its 1-based position, all
 *     ceil(m / 8) bytes present with the unused high bits of the last zero; nothing after the last level.  k <= 64 is a
 *     bound the build never reaches (its p_1 >= 1 / (sqrt(2) * slots)); it stops a crafted filter from making each
 *     thread hash without limit;
 *   - a stash unit whose hash length is not 32, and a stash truncated anywhere; a NULL filter or stashes with a nonzero
 *     length.  Entries longer than CTMR_MAX_SERIAL and digests not in the registry are accepted: they never match;
 *   - ctmr_revoked_cascade's: a NULL batch or output, a CRL outside data or larger than a chunk.
 *
 * The cap rule is the cascade's: with cap too small (buf may be NULL) the call returns CTMR_E_BATCH_TOO_LARGE and writes
 * `bytes` and nothing else; a second call with that cap returns exactly those bytes.  Read-only, like the other CRL calls.
 * A member ctx of a group is refused with CTMR_E_INVALID (use ctmr_group_revoked_stash), and so is a ctx attached to
 * peers (world > 1): every rank refuses before any barrier, so none waits.  Cost: the cascade's mark and split, then one
 * thread per record of R walking the filter's levels, and the candidates the filter misses read back and sorted on the
 * host (DESIGN.md "Revoked stash").
 * Out of scope: un-revocations (a stash only adds); which issuers the old filter covered (every issuer covered now is
 * answered by the filter's query, and a newly enrolled issuer wants a new full filter); signature verification. */
typedef struct ctmr_stash_out {     /* caller-allocated; HOST buffers */
    uint8_t* buf; uint64_t cap;     /* the serialized stash */
    uint64_t bytes;                 /* written; on CTMR_E_BATCH_TOO_LARGE the bytes needed */
    uint8_t* crl_status;            /* [n_crls] CTMR_CRL_*, as ctmr_revoked_known; may be NULL */
    uint32_t issuers;               /* issuers covered (the cascade's rule) */
    uint32_t stash_issuers;         /* issuer units written */
    uint64_t revoked;               /* key records in R (the cascade's |R| for this batch and now) */
    uint64_t in_filter;             /* of them: the filter answers revoked */
    uint64_t in_stashes;            /* of the rest: an earlier stash lists their (issuer, serial) */
    uint64_t serials;               /* (issuer, serial) entries written */
} ctmr_stash_out;
int ctmr_revoked_stash(ctmr_ctx* ctx, const ctmr_crl_batch* batch, int64_t now_unix_sec,
                       const uint8_t* filter, uint64_t filter_bytes,
                       const uint8_t* stashes, uint64_t stash_bytes, ctmr_stash_out* out);

/* ---- CRLite verify (a published filter and its stashes checked against the table) --------------------------------- */
/* Checks a filter, with the stashes published since it, against the table before it is published or while it is in
 * use: every live record of a covered issuer is queried, and only the records answered wrongly reach the host
 * (DESIGN.md "Revoked verify").  Filter.verify(include, exclude) of Mozilla's filter-cascade, with R and S from the table.
 *
 * Sets.  Covered issuers, live records, R and S are ctmr_revoked_cascade's for the same batch and now_unix_sec.  Records
 * of issuers that are not covered are neither verified nor counted.
 *
 * Answer.  x = digest || serial.  A record is ANSWERED REVOKED when the query rule above, with the filter's own salt,
 * says revoked, or when any stash in `stashes` lists (digest, serial) (the stash layout above; `stashes` may be empty).
 * Counts are key records: a serial under two hours is two records, each with its own first index.
 *
 * Age.  A record is counted in `before` when its first-seen global index is below covered_below, and in `since`
 * otherwise.  The index is the one the table keeps per key (eviction, resize and checkpoint loads keep it; preloads take
 * indices from next_index).  Pass ctmr_next_index, read when the filter was built, to tell the records the filter was
 * built over from the ones that arrived later; UINT64_MAX puts every record in `before`.
 *
 * List.  Every `before` record that is missed or blocked, ordered by digest bytes, then serial (ascending bytes, a prefix
 * before any longer serial), then exp_hour.  That triple is unique per key record, so the output is deterministic: it
 * depends neither on slot order, shard count nor thread order.  If list_cap is too small, or list is NULL while records
 * are to be listed, the call returns CTMR_E_BATCH_TOO_LARGE and writes n_list and nothing else (ctmr_revoked_known's
 * entry_cap rule).
 *
 * Checks before any work, each CTMR_E_INVALID: ctmr_revoked_stash's checks of the filter (including k <= 64) and of the
 * stashes, ctmr_revoked_cascade's (a NULL batch or output, a CRL outside data or larger than a chunk).  Stash entries of
 * unregistered digests or longer than CTMR_MAX_SERIAL are accepted and never match.  Read-only, like the other CRL calls.
 * A member ctx of a group is refused with CTMR_E_INVALID (use ctmr_group_revoked_verify).  Cost: the cascade's mark and
 * split, one more mark pass for the stashes, and one pass over the table that hashes the covered live records the
 * stashes do not list (DESIGN.md "Revoked verify").
 *
 * On a ctx attached to peers (world > 1) the call is COLLECTIVE and follows ctmr_revoked_cascade's peer rules: every rank
 * passes its own CRLs (possibly none) and the same now_unix_sec, covered_below, filter and stashes.  Counts and list are
 * identical on every rank: what one ctx holding every rank's table gives for the CRLs of all ranks in rank order;
 * crl_status covers the rank's own CRLs.  A rank whose now_unix_sec, covered_below, filter or stashes differ from rank
 * 0's returns CTMR_E_INVALID and the others CTMR_E_PEER_FAILED, before any work.  A list_cap too small on any rank is
 * CTMR_E_BATCH_TOO_LARGE on every rank, each writing only n_list; later failures are every rank's.
 * Out of scope: un-revocations in stashes; which issuers the old filter covered (the issuers covered now are verified). */
typedef struct ctmr_verify_counts {  /* key records, counted as the cascade counts them */
    uint64_t revoked;                /* in R, answered revoked */
    uint64_t missed;                 /* in R, answered not revoked */
    uint64_t valid;                  /* in S, answered not revoked */
    uint64_t blocked;                /* in S, answered revoked */
} ctmr_verify_counts;
typedef struct ctmr_verify_miss {    /* one listed key record: 96 bytes */
    uint8_t  digest[32];             /* Issuer.ID() digest */
    int64_t  exp_hour;
    uint64_t first_index;            /* the record's first-seen global index */
    uint8_t  serial_len;
    uint8_t  serial[CTMR_MAX_SERIAL]; /* zero padded */
    uint8_t  blocked;                /* 0: an R record answered not revoked; 1: an S record answered revoked */
    uint8_t  pad[7];
} ctmr_verify_miss;
typedef struct ctmr_verify_out {     /* caller-allocated; HOST buffers */
    uint8_t* crl_status;             /* [n_crls] CTMR_CRL_*, as ctmr_revoked_known; may be NULL */
    uint32_t issuers;                /* covered (the cascade's rule) */
    uint32_t levels;                 /* levels of the filter */
    ctmr_verify_counts before;       /* records first seen at a global index < covered_below */
    ctmr_verify_counts since;        /* the others */
    ctmr_verify_miss* list; uint64_t list_cap;
    uint64_t n_list;                 /* written; on CTMR_E_BATCH_TOO_LARGE the count needed */
} ctmr_verify_out;
int ctmr_revoked_verify(ctmr_ctx* ctx, const ctmr_crl_batch* batch, int64_t now_unix_sec,
                        const uint8_t* filter, uint64_t filter_bytes, const uint8_t* stashes, uint64_t stash_bytes,
                        uint64_t covered_below, ctmr_verify_out* out);

/* ---- device-resident entry points ---------------------------------------------------------- */
/* Same path with every buffer already in HBM on ctx's device (benchmarks, multi-GPU orchestration,
 * hosts that receive entries by GPUDirect).  `stream` is a cudaStream_t passed as void*; NULL =
 * the ctx's own stream.  Asynchronous: the caller synchronises the stream. */

/* 64-byte key record: what WasUnknown is keyed on (SURVEY §0 M4): expDate hour, issuer, raw serial. */
typedef struct ctmr_key {
    uint64_t index;      /* global entry index: lowest index of equal keys wins "was unknown" */
    int32_t exp_hour;
    uint32_t issuer;     /* dense issuer index */
    uint8_t serial_len;
    uint8_t serial[CTMR_MAX_SERIAL]; /* zero padded */
    uint32_t valid;      /* 1 when the entry reached Store (status OK) */
    uint32_t pad;
} ctmr_key;

typedef struct ctmr_dev_batch {
    const uint8_t* blob;        /* device; readable up to blob_bytes rounded up to 16 */
    uint64_t blob_bytes;
    const uint64_t* offsets;    /* device [n+1] */
    uint64_t n;
    const uint32_t* issuer_idx; /* device [n]; NULL = every entry has no chain */
    const uint32_t* issuer_map; /* device [*]: batch-local -> dense index, or NULL when issuer_idx is dense */
    uint32_t issuer_map_len;
    uint32_t reserved;
    uint64_t first_index;       /* global index of entry 0 */
    int64_t now_unix_ns;
    const uint32_t* lens;       /* device [n] or NULL.  When set, entry i = blob[offsets[i] .. offsets[i]+lens[i]):
                                 * records need not be contiguous and offsets needs only n elements (this is how
                                 * the wire-format front end, ctmr_frontend.h, hands over leaves it decoded in place) */
} ctmr_dev_batch;

typedef struct ctmr_dev_out { /* device pointers, each [n]; NULL = not produced */
    uint8_t* status;
    uint8_t* sha256;
    int64_t* exp_hour;
    uint32_t* serial_off;
    uint32_t* serial_len;
    uint8_t* was_unknown;
    uint8_t* first_issuer_hour;
    ctmr_key* keys; /* [n] key records (valid=0 for entries that did not reach Store) */
    uint32_t* issuer_name_off; /* as in ctmr_out; first_* are produced by ctmr_process_device only */
    uint32_t* issuer_name_len;
    uint32_t* crldp_off;
    uint32_t* crldp_len;
    uint8_t* first_issuer_dn;
    uint8_t* first_crldp;
} ctmr_dev_out;

/* map half: DER walk + filter + SHA-256 -> status, exp_hour, serial span, fingerprint, key records */
int ctmr_map_device(ctmr_ctx* ctx, const ctmr_dev_batch* batch, const ctmr_dev_out* out, void* stream);
/* reduce half over m key records in any order WITHIN the call: insert, resolve lowest-index-wins, per-issuer
 * counts.  Across calls the ordering contract of the path holds: every index of a later call must be higher than
 * every index of an earlier call (a lower index arriving later would find itself "first" a second time). */
int ctmr_reduce_device(ctmr_ctx* ctx, const ctmr_key* keys, uint64_t m, uint8_t* was_unknown /* [m] */,
                       uint8_t* first_issuer_hour /* [m] */, void* stream);
/* map + reduce on one GPU */
int ctmr_process_device(ctmr_ctx* ctx, const ctmr_dev_batch* batch, const ctmr_dev_out* out, void* stream);

/* CUDA-event timings of the last ctmr_process_device call, valid once its stream has been synchronised:
 * map_ms = span of the K_map launches (first start to last end), total_ms = whole call */
int ctmr_profile_last(ctmr_ctx* ctx, float* map_ms, float* total_ms);

/* copy the per-issuer histogram (uint64 [n_slots], dense index order) and the status counters
 * (uint64 [CTMR_ST__COUNT]) of THIS GPU into device buffers (a group merges them with ctmr_peer_allreduce_histogram_device) */
int ctmr_read_histogram_device(ctmr_ctx* ctx, uint64_t* counts_dst, uint32_t n_slots, uint64_t* status_dst,
                               void* stream);
/* forget everything: known-certificate table, first-seen pairs, per-issuer and status counters
 * (the issuer registry is kept).  The analogue of FLUSHDB on the reference's Redis. */
int ctmr_reset_device(ctmr_ctx* ctx, void* stream);
/* fails with CTMR_E_TABLE_FULL / CTMR_E_CUDA if any asynchronous launch since the last check failed */
int ctmr_check_device(ctmr_ctx* ctx, void* stream);

/* ---- several GPUs, ONE process (what a Go host uses: SURVEY.md §8(b) "fan-out inside the library") ------------ */
/* The worker pool of StartDatabaseThreads (cmd/ct-fetch/ct-fetch.go:140-145) becomes one call per drained batch:
 * the group cuts the batch into rounds of n_devices slices by entry index (entry i keeps global index
 * next_index + i, so the result equals the sequential numThreads=1 run over the batch in its given order), every
 * GPU maps its slice and hands each key to the set's owner GPU over NVLink, events separate the appends from the
 * owners' insert/resolve and that from the pull of the result bits, and the outputs land in the caller's arrays in
 * entry order.  cfg->device is ignored;
 * `devices` may name a device more than once (several shards on one GPU: how the path is tested on a 1-GPU box). */
typedef struct ctmr_group ctmr_group;
int ctmr_group_create(const ctmr_config* cfg, const int32_t* devices, uint32_t n_devices, ctmr_group** out);
void ctmr_group_destroy(ctmr_group* g);
const char* ctmr_group_last_error(ctmr_group* g);
uint32_t ctmr_group_size(ctmr_group* g);
ctmr_ctx* ctmr_group_member(ctmr_group* g, uint32_t rank); /* read-side access to one shard; owned by the group */
/* same arguments and outputs as ctmr_process_batch; globally exact across the GPUs of the group */
int ctmr_group_process_batch(ctmr_group* g, const uint8_t* blob, const uint64_t* offsets, uint64_t n, const uint8_t* issuer_blob,
                             const uint64_t* issuer_offsets, uint32_t n_issuers, const uint32_t* issuer_idx, int64_t now_unix_ns,
                             ctmr_out* out);
int ctmr_group_issuer_counts(ctmr_group* g, uint8_t* digests, uint64_t* counts, size_t* n);   /* summed over the shards */
int ctmr_group_set_cardinality(ctmr_group* g, int64_t exp_hour, const uint8_t issuer_digest[32], uint64_t* count_out);
int ctmr_group_status_counters(ctmr_group* g, uint64_t out[CTMR_ST__COUNT]);
int ctmr_group_table_stats(ctmr_group* g, uint64_t* slots_used, uint64_t* capacity);
int ctmr_group_preload_known(ctmr_group* g, int64_t exp_hour, const uint8_t issuer_digest[32], const uint8_t* serial_blob,
                             const uint64_t* serial_offsets, uint64_t n);
int ctmr_group_evict_expired(ctmr_group* g, int64_t now_unix_sec, uint64_t* evicted_out);
int ctmr_group_reset(ctmr_group* g);
/* snapshot of the whole group (every shard + the one issuer registry); restores into a group of the same size and
 * capacities (a set's owner depends on the group size).  For another size or other capacities: ctmr_group_checkpoint_*. */
int ctmr_group_snapshot_size(ctmr_group* g, uint64_t* bytes);
int ctmr_group_snapshot_save(ctmr_group* g, uint8_t* buf, uint64_t cap, uint64_t* written);
int ctmr_group_snapshot_load(ctmr_group* g, const uint8_t* buf, uint64_t bytes);
/* portable checkpoint of the whole group: one part (every shard's records); loads any checkpoint (ctmr_checkpoint_*) */
int ctmr_group_checkpoint_size(ctmr_group* g, uint64_t* bytes);
int ctmr_group_checkpoint_save(ctmr_group* g, uint8_t* buf, uint64_t cap, uint64_t* written);
int ctmr_group_checkpoint_load(ctmr_group* g, const uint8_t* const* parts, const uint64_t* part_bytes, uint32_t n_parts);
/* delta checkpoint of the whole group (one part; member 0 holds the delta floor and the evictions), and a delta applied
 * onto it (ctmr_checkpoint_delta_*, ctmr_checkpoint_apply) */
int ctmr_group_checkpoint_delta_size(ctmr_group* g, uint64_t since, uint64_t* bytes);
int ctmr_group_checkpoint_delta_save(ctmr_group* g, uint64_t since, uint8_t* buf, uint64_t cap, uint64_t* written);
int ctmr_group_checkpoint_apply(ctmr_group* g, const uint8_t* const* parts, const uint64_t* part_bytes, uint32_t n_parts);
/* ctmr_resize of every shard, all or nothing: each member's tables get the given size (0 keeps it), every member's new
 * tables are built and rehashed before any old ones go, and a failure of one member leaves every member unchanged */
int ctmr_group_resize(ctmr_group* g, uint64_t table_capacity, uint32_t pair_capacity_log2, uint32_t meta_capacity_log2);
int ctmr_group_table_occupancy(ctmr_group* g, uint64_t used[3], uint64_t capacity[3]);   /* summed over the shards */
/* ctmr_rollback of the group to its own next index N: every member's shard and status counters back to the mark at N */
int ctmr_group_rollback(ctmr_group* g, uint64_t next_index);
/* ctmr_revoked_known over every shard: member 0 parses the CRLs and builds the set of (issuer, serial) pairs, each member
 * scans its own table against a bulk copy of it, and member 0 merges the answers (lowest hour, sum of sets). */
int ctmr_group_revoked_known(ctmr_group* g, const ctmr_crl_batch* batch, ctmr_crl_out* out);
/* ctmr_revoked_cascade over every shard, the same bytes as one ctx: member 0 parses the CRLs and builds the set, each
 * member marks and compacts its own shard, and each level's partial bit arrays are merged on member 0 with peer copies
 * and copied back to every member before the members test their own records.  No atomic crosses a GPU. */
int ctmr_group_revoked_cascade(ctmr_group* g, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* salt,
                               uint32_t salt_len, ctmr_cascade_out* out);
/* ctmr_revoked_stash over every shard, the same bytes as one ctx: the cascade's mark and split on every member, each
 * member queries the filter for its own R records, and the host merges the candidates. */
int ctmr_group_revoked_stash(ctmr_group* g, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* filter,
                             uint64_t filter_bytes, const uint8_t* stashes, uint64_t stash_bytes, ctmr_stash_out* out);
/* ctmr_revoked_verify over every shard, the same counts and list as one ctx: the cascade's mark and split and the
 * stashes' mark on every member, each member verifies its own shard, and the host sums the counts and merges the lists. */
int ctmr_group_revoked_verify(ctmr_group* g, const ctmr_crl_batch* batch, int64_t now_unix_sec, const uint8_t* filter,
                              uint64_t filter_bytes, const uint8_t* stashes, uint64_t stash_bytes, uint64_t covered_below,
                              ctmr_verify_out* out);

/* ---- several GPUs, one PROCESS PER GPU (torchrun-style launches; SURVEY.md §8(e)) ------------------------------ */
/* Every rank creates its ctx with the same capacities, exports a handle, gathers all handles by whatever means the
 * launcher offers (torch.distributed all_gather in this repository) and attaches them.  From then on
 * ctmr_process_device, ctmr_process_batch, ctmr_reset_device, ctmr_peer_* and the nine front-end calls of
 * ctmr_frontend.h (ctmr_process_raw, ctmr_process_tiles, ctmr_process_raw_bodies and their _tree / _trees forms; their
 * contract is stated there) are COLLECTIVE: every rank must make the same sequence of calls; any front-end call matches any other.
 * Inside them the ranks meet at barriers kept in peer memory (no host round trip, no
 * NCCL on the data path); the global index of entry j of rank r's round k is first_index + (k * world + r) * E + j,
 * i.e. the result equals the sequential run over the rounds in rank order.  E = entries per rank and round: the host
 * pipeline's stage size for ctmr_process_batch; for ctmr_process_device (every rank passes the same n, R =
 * ctmr_peer_rounds() >= 4) E = ceil(4n / (4R - 3)), i.e. R - 1 full rounds and a last one a quarter as long. */
#define CTMR_PEER_HANDLE_BYTES 256u
/* allocates this rank's key-exchange area for a group of `world` ranks and exports it together with the tables */
int ctmr_peer_export(ctmr_ctx* ctx, uint32_t world, uint8_t handle_out[CTMR_PEER_HANDLE_BYTES]);
int ctmr_peer_attach(ctmr_ctx* ctx, uint32_t rank, uint32_t world, const uint8_t* handles /* [world][CTMR_PEER_HANDLE_BYTES] */);
/* *next_index = the global index the next ctmr_process_batch or front-end call on this ctx starts at: what the earlier
 * calls used up, on a ctx of a multi-process group by the collective rules.  A ctmr_process_device call whose entries
 * must follow them passes first_index >= this.  CTMR_E_INVALID for a member of an in-process group (the group holds the
 * index). */
int ctmr_next_index(ctmr_ctx* ctx, uint64_t* next_index);
/* barrier over the group on `stream` (device side; returns immediately) */
int ctmr_peer_barrier_device(ctmr_ctx* ctx, void* stream);
/* all-reduce(sum) of [per-issuer unique counts || status counters] over peer memory, bracketed by barriers: the
 * merge of the per-GPU histograms at the end of a chunk.  Device buffers, uint64 [n_slots] and [CTMR_ST__COUNT]. */
int ctmr_peer_allreduce_histogram_device(ctmr_ctx* ctx, uint64_t* counts_dst, uint32_t n_slots, uint64_t* status_dst, void* stream);
/* the collective ctmr_process_device always runs ctmr_peer_rounds() rounds (CTMR_PEER_ROUNDS unless the environment
 * variable of the same name overrides it for experiments; identical on every rank) */
#define CTMR_PEER_ROUNDS 8u
uint32_t ctmr_peer_rounds(void);
/* E of a collective ctmr_process_device call over n entries per rank: what config.max_round_entries must cover and what
 * the global-index formula above uses (R - 1 rounds of E entries and a short last one) */
uint64_t ctmr_peer_round_entries(uint64_t n);

/* ---- host placement -------------------------------------------------------------------------------- */
/* Binds the calling thread to the CPUs of the NUMA node `device` hangs off (sysfs), so that pinned buffers it
 * allocates and first touches afterwards are node-local: with 8 GPUs reading host memory at PCIe rate, remote-node
 * buffers halve the end-to-end rate.  Returns the node, or -1 when the topology cannot be read (no change made). */
int ctmr_bind_host_to_device(int32_t device);

/* ---- measurement tooling -------------------------------------------------------------------- */
/* Register-only SHA-256 microbenchmark: every lane chains `iters` compressions (K_map's own function, no
 * memory traffic) at `ctas_per_sm` x 256 threads per SM.  The measured INT-pipe ceiling of the fingerprint. */
int ctmr_sha256_ceiling_device(ctmr_ctx* ctx, uint32_t iters, uint32_t rolled, uint32_t ctas_per_sm, float* ms_out,
                               uint64_t* blocks_out);

/* ---- synthetic corpus on the device (bench/test tooling; ctmr_synth.h) ---------------------- */
struct ctmr_synth_cfg;
/* pass 1: offsets[0..n] (device) of entries [first, first+n); returns total bytes via *total_bytes */
int ctmr_synth_offsets_device(const struct ctmr_synth_cfg* cfg, uint64_t first, uint64_t n, uint64_t* offsets,
                              uint64_t* total_bytes, void* stream);
/* pass 2: write the DER bytes and (optionally) the issuer index of each entry */
int ctmr_synth_write_device(const struct ctmr_synth_cfg* cfg, uint64_t first, uint64_t n, const uint64_t* offsets,
                            uint8_t* blob, uint32_t* issuer_idx, void* stream);
/* generator-side truth for size-independent checks: cert id, notAfter, basicConstraints mode */
int ctmr_synth_truth_device(const struct ctmr_synth_cfg* cfg, uint64_t first, uint64_t n, uint64_t* cert_id,
                            int64_t* not_after, uint8_t* bc_mode, void* stream);

/* host-side: DER of the n_issuers synthetic CA certificates; returns total bytes, fills
 * offsets[0..n_issuers]; writes bytes when blob != NULL and cap suffices */
uint64_t ctmr_synth_issuers_host(const struct ctmr_synth_cfg* cfg, uint64_t* offsets, uint8_t* blob, uint64_t cap);

/* host-side: RFC 6962 get-entries response bodies (JSON, base64 leaf_input / extra_data; every third entry a
 * precert_entry, chains of one or two certificates) for entries [first, first+n) in pages of `page` entries -- input
 * for ctmr_process_raw (ctmr_frontend.h).  Returns the bytes needed; writes the text and the string spans when
 * text != NULL and cap suffices. */
uint64_t ctmr_synth_raw_pages_host(const struct ctmr_synth_cfg* cfg, uint64_t first, uint64_t n, uint32_t page, uint8_t* text,
                                   uint64_t cap, uint64_t* leaf_off, uint32_t* leaf_len, uint64_t* extra_off, uint32_t* extra_len);

/* host-side: static-ct-api data tiles first_tile .. first_tile + n_tiles - 1 (256 entries each) of the same entries as
 * ctmr_synth_raw_pages_host (entry i = 256 * N + j of tile N), for input to ctmr_process_tiles (ctmr_frontend.h).
 * issuer_fps ([cfg->n_issuers][32]) are the fingerprints of the synthetic issuers, passed in by the caller.  Returns the
 * bytes needed; writes the tiles back to back and their spans when data != NULL and cap suffices. */
uint64_t ctmr_synth_tiles_host(const struct ctmr_synth_cfg* cfg, uint64_t first_tile, uint64_t n_tiles, const uint8_t* issuer_fps,
                               uint8_t* data, uint64_t cap, uint64_t* tile_off, uint32_t* tile_len);

#ifdef __cplusplus
}
#endif
#endif /* CTMR_H */
