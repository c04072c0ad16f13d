/*
 * ctmr_frontend.h -- CT wire-format front end of libctmr (SURVEY.md §8(f)-2): the step BEFORE the
 * hot path.  The host ships the base64 strings of RFC 6962 §4.6 get-entries responses as they came off
 * the wire; the GPU decodes them, undoes the TLS framing, identifies Chain[0], and feeds the leaves to
 * the same map/reduce kernels as ctmr_process_batch -- no per-entry parse on the host.
 *
 * What it replaces in the reference (jcjones/ct-mapreduce):
 *   - the base64 decode of "leaf_input" / "extra_data" that encoding/json performs inside
 *     ct-go jsonclient for LogClient.GetRawEntries (cmd/ct-fetch/ct-fetch.go:424);
 *   - ct.LogEntryFromLeaf(index, &entry) (cmd/ct-fetch/ct-fetch.go:452): tls.Unmarshal of the
 *     MerkleTreeLeaf (RFC 6962 §3.4), of the CertificateChain / PrecertChainEntry in extra_data
 *     (§4.6), MerkleTreeLeaf.X509Certificate() / .Precertificate() and the "entry dropped" decision
 *     at ct-fetch.go:453-460;
 *   - the entry-type switch of insertCTWorker (ct-fetch.go:198-204): X509 entries use the leaf
 *     certificate, precert entries use PrecertChainEntry.pre_certificate (Precert.Submitted);
 *   - x509.ParseCertificate(Chain[0]) + NewIssuer (ct-fetch.go:215-225, storage/types.go:109-130),
 *     done once per distinct Chain[0] instead of once per entry;
 *   and then everything ctmr_process_batch replaces (include/ctmr.h).
 *
 * github.com/google/certificate-transparency-go v1.1.0 (go.mod:10) is not vendored under the reference,
 * so the TLS rules are restated from RFC 6962 and that version's published struct tags; see
 * oracle/ctmr_oracle_frontend.c ("parity unpinned" for ct-go specifics, pinned against RFC 6962 vectors
 * built in tests/test_frontend_oracle.py).
 */
#ifndef CTMR_FRONTEND_H
#define CTMR_FRONTEND_H

#include "ctmr.h"

#ifdef __cplusplus
extern "C" {
#endif

/* per-entry outcome of the front end ("Erroneous certificate", ct-fetch.go:453-460, unless noted) */
enum {
    CTMR_FE_OK = 0,
    CTMR_FE_BAD_BASE64 = 1,   /* a string is not padded standard base64 (in the reference the whole page fails in
                                 encoding/json and GetRawEntries returns the error, ct-fetch.go:425-443) */
    CTMR_FE_BAD_LEAF = 2,     /* leaf_input is not a v1 timestamped MerkleTreeLeaf, or has trailing data */
    CTMR_FE_UNKNOWN_TYPE = 3, /* entry_type is neither x509_entry(0) nor precert_entry(1) */
    CTMR_FE_BAD_EXTRA = 4,    /* extra_data is not the chain structure its entry type requires */
    CTMR_FE_BAD_CERT = 5,     /* x509: the leaf certificate, precert: the TBSCertificate of the leaf, has a fatal
                                 parse error ("failed to parse (pre)certificate in MerkleTreeLeaf") */
    CTMR_FE_BAD_TILE = 6,     /* static-ct-api data tile that does not split into exactly `width` well-framed TileLeafs
                                 (ctmr_process_tiles): every entry of the tile gets it */
    CTMR_FE_BAD_INDEX = 7     /* TileLeaf whose leaf_index extension is missing, repeated, not 5 bytes long or not
                                 256 * N + j (ctmr_process_tiles) */
};

#define CTMR_ENTRY_X509 0u
#define CTMR_ENTRY_PRECERT 1u
#define CTMR_ENTRY_OTHER 0xFFu

/* n entries of one or more get-entries pages.  HOST buffers.  String i's characters are
 * text[off[i] .. off[i]+len[i]): the contents of the JSON strings, quotes excluded, JSON escapes (if a
 * log emitted any -- base64 needs none) already undone by the caller.  Strings may lie anywhere in
 * `text`, in any order, e.g. in place inside the raw HTTP bodies. */
typedef struct ctmr_raw_batch {
    const uint8_t* text;
    uint64_t text_bytes;
    const uint64_t* leaf_input_off; /* [n] */
    const uint32_t* leaf_input_len; /* [n] characters */
    const uint64_t* extra_data_off; /* [n] */
    const uint32_t* extra_data_len; /* [n] */
    uint64_t n;
    int64_t now_unix_ns;            /* replaces time.Now() at ct-fetch.go:52 */
} ctmr_raw_batch;

/* Caller-allocated outputs, each [n]; any pointer may be NULL. */
typedef struct ctmr_raw_out {
    ctmr_out path;            /* exactly the outputs of ctmr_process_batch; entries with entry_status != 0 and
                                 x509 entries whose leaf does not parse carry status CTMR_ST_PARSE_ERR */
    uint8_t* entry_status;    /* CTMR_FE_* */
    uint8_t* entry_type;      /* CTMR_ENTRY_* (LogEntryType, RFC 6962 §3.1) */
    uint64_t* timestamp_ms;   /* TimestampedEntry.timestamp (feeds uint64ToTimestamp, ct-fetch.go:478) */
    uint32_t* issuer;         /* dense issuer index of Chain[0] (ctmr_issuer_digest), CTMR_ISSUER_NONE, CTMR_ISSUER_BAD */
    /* where the certificate the path processed lies, so that the host can cut the DER of the few NEW
     * certificates out of its own copy of the text without a device round trip (PEM for
     * StoreCertificatePEM, filesystemdatabase.go:197-202): */
    uint8_t* leaf_src;        /* 0: inside the decoded leaf_input, 1: inside the decoded extra_data */
    uint32_t* leaf_off;       /* byte offset inside that decoded string */
    uint32_t* leaf_len;
} ctmr_raw_out;

/* Decode + frame + identify issuers + map + reduce.  Synchronous.  Entries take the global indices
 * following those of earlier ctmr_process_batch / ctmr_process_raw calls on this ctx.
 *
 * Chain[0] is identified on the GPU through a per-ctx mirror keyed by the certificate's bytes: it holds
 * 2 x config.max_issuers distinct Chain[0] DERs.  Every distinct DER takes a slot, also a reissue of a
 * known key and a DER that does not parse (which resolves to CTMR_ISSUER_BAD), so the mirror can fill
 * before the issuer registry does.  A batch that meets one DER more fails with CTMR_E_TOO_MANY_ISSUERS;
 * the DERs already held keep resolving in later calls. */
int ctmr_process_raw(ctmr_ctx* ctx, const ctmr_raw_batch* batch, ctmr_raw_out* out);

/* The same on every GPU of a group (ctmr_group_create, ctmr.h): each round takes one chunk per GPU out of ONE contiguous
 * window of the batch, every GPU decodes and frames its chunk, Chain[0] certificates resolve against the group's issuer
 * registry, and the path runs as one round of the group's key exchange -- entry i keeps global index next_index + i, so
 * the outputs equal those of ctmr_process_raw on one GPU for the same pages. */
int ctmr_group_process_raw(ctmr_group* g, const ctmr_raw_batch* batch, ctmr_raw_out* out);

/* ---- whole get-entries response bodies ----------------------------------------------------------------------------
 * The HTTP bodies as they came off the wire: the GPU validates each body as JSON and finds its entries with the rules
 * of Go 1.13 encoding/json decoding it into ct-go's GetEntriesResponse (Unmarshal runs checkValid over the whole body
 * first; reference cmd/ct-fetch/ct-fetch.go:424):
 *   - validity (RFC 8259 as Go's scanner checks it): structure, the literals, number syntax, the escapes
 *     \" \\ \/ \b \f \n \r \t \uXXXX, no raw byte below 0x20 inside a string, only space, tab, LF and CR as whitespace,
 *     nothing but whitespace after the value.  An empty body or a UTF-8 BOM is invalid; invalid UTF-8 is not;
 *   - types: the top level is an object or null (no entries); "entries" is an array or null; an element is an object or
 *     null (an entry with both strings empty); "leaf_input" / "extra_data" are strings or null (empty).  Members of any
 *     other name, at any depth and of any type, are skipped;
 *   - keys are unescaped before they match: "leaf_input" and "extra_data" ASCII case-insensitively ('_' exactly),
 *     "entries" as encoding/json's equalFoldRight does ('s' also matches U+017F).  Inside an element the last of a
 *     repeated key wins and a missing key means empty;
 *   - a string holding escapes is unescaped, and '\r' / '\n' are dropped as base64.StdEncoding skips them, before the
 *     decode; a non-ASCII character makes the string CTMR_FE_BAD_BASE64.
 * The entries of the OK bodies, in (body, position) order, then go through exactly what ctmr_process_raw does with
 * their strings. */
enum {
    CTMR_BODY_OK = 0,
    CTMR_BODY_BAD_JSON = 1,          /* checkValid fails */
    CTMR_BODY_BAD_TYPE = 2,          /* valid JSON that does not fit GetEntriesResponse */
    CTMR_BODY_TOO_MANY = 3,          /* more entries than body_max */
    CTMR_BODY_REPEATED_ENTRIES = 4   /* a second top-level "entries" member: encoding/json decodes the later array into the
                                        elements the earlier one filled; decode such a body on the host (ctmr_process_raw) */
};

/* n_bodies bodies; HOST buffers.  Body b is text[body_off[b] .. body_off[b] + body_len[b]); bodies may lie anywhere in
 * text, also back to back. */
typedef struct ctmr_body_batch {
    const uint8_t* text;
    uint64_t text_bytes;
    const uint64_t* body_off;  /* [n_bodies] */
    const uint32_t* body_len;  /* [n_bodies] */
    const uint32_t* body_max;  /* [n_bodies] entries requested (end - start + 1 of the get-entries call) */
    uint64_t n_bodies;
    int64_t now_unix_ns;
} ctmr_body_batch;

/* Caller-allocated outputs; any pointer may be NULL.  Per-entry arrays hold sum of body_max entries, of which
 * [0, n_entries) are written (raw.path.pem_off n_entries + 1). */
typedef struct ctmr_body_out {
    ctmr_raw_out raw;          /* as ctmr_process_raw writes them for the entries found */
    uint8_t* body_status;      /* [n_bodies] CTMR_BODY_*; a body that is not OK contributes no entry */
    uint64_t* body_first;      /* [n_bodies] position of the body's first entry in the per-entry arrays */
    uint32_t* body_entries;    /* [n_bodies] */
    uint64_t* leaf_input_off;  /* [entries] the string as found: offset in text (quotes excluded) and length, escapes */
    uint32_t* leaf_input_len;  /*           included, so that the host can cut a new certificate out of its own text */
    uint64_t* extra_data_off;  /*           (0 and 0 for a missing or null string) */
    uint32_t* extra_data_len;
    uint8_t* escaped;          /* [entries] bit 0: leaf_input held an escape, bit 1: extra_data did */
    uint64_t n_entries;        /* written */
} ctmr_body_out;

/* Find the entries of every body, then decode + frame + identify issuers + map + reduce them as ctmr_process_raw does.
 * Synchronous.  The entries take consecutive global indices in (body, position) order after those of earlier calls;
 * a successful call advances the next index by n_entries.  After a failure once a chunk has reached the path, it
 * advances by the sum of body_max, so that a retry never reuses an index.  A body longer than half the front end's
 * character budget, or with more requested entries than its entry budget, is CTMR_E_BATCH_TOO_LARGE before any work.
 * On a group member this call is refused; on a ctx attached to peers it is collective, with the rules of the front-end
 * calls below (chunks of at most E entries requested). */
int ctmr_process_raw_bodies(ctmr_ctx* ctx, const ctmr_body_batch* batch, ctmr_body_out* out);
/* The same on every GPU of a group: the outputs equal those of ctmr_process_raw_bodies on one GPU. */
int ctmr_group_process_raw_bodies(ctmr_group* g, const ctmr_body_batch* batch, ctmr_body_out* out);
/* CUDA-event time of the JSON kernels (classify, walk, compaction, unescape) in the last bodies call on this ctx, summed
 * over its chunks, in milliseconds: a part of the frontend_ms that ctmr_frontend_profile_last reports */
int ctmr_bodies_profile_last(ctmr_ctx* ctx, float* json_ms);

/* CUDA-event timings of the last front-end call (raw or tiles): front-end kernels (decode, framing, issuer
 * identification; for tiles the split, framing, fingerprint look-up and leaf hashes; for the tree forms also the leaf
 * hashes and the Merkle fold) and the map/reduce that
 * followed, summed over its chunks, in milliseconds */
int ctmr_frontend_profile_last(ctmr_ctx* ctx, float* frontend_ms, float* path_ms, uint64_t* frontend_launches);

/* ---- static-ct-api data tiles (C2SP static-ct-api) --------------------------------------------------------------
 * A data tile holds up to 256 TileLeafs back to back, no separators (big-endian, TLS vectors, RFC 5246 §4):
 *   TileLeaf := TimestampedEntry (RFC 6962 §3.4)
 *               [ ASN.1Cert pre_certificate ]                  opaque<1..2^24-1>, precert_entry only
 *               Fingerprint certificate_chain<0..2^16-1>       byte length a multiple of 32
 * A Fingerprint is SHA-256 of a chain certificate's DER (the log serves the DER at issuer/<hex>).  The
 * TimestampedEntry's CtExtensions must carry exactly one leaf_index extension (type 0, 5 bytes, uint40) equal to
 * 256 * N + j for entry j of tile N.  An entry is processed as the get-entries entry with
 * leaf_input = 00 00 || TimestampedEntry and the chain DERs behind the fingerprints; Chain[0] is the certificate
 * behind the first fingerprint. */

/* n_tiles tiles; HOST buffers.  Tile t is data[tile_off[t] .. tile_off[t] + tile_len[t]) with tile_width[t] entries
 * (1..256: 256 for a full tile, W for a partial tile .p/W), and is tile number tile_index[t] of its log.  Tiles need not
 * be consecutive and may come from several logs.  The entries of the batch are the tiles' entries in tile order. */
typedef struct ctmr_tile_batch {
    const uint8_t* data;
    uint64_t data_bytes;
    const uint64_t* tile_off;    /* [n_tiles] */
    const uint32_t* tile_len;    /* [n_tiles] */
    const uint64_t* tile_index;  /* [n_tiles] N of tile/data/<N> */
    const uint16_t* tile_width;  /* [n_tiles] */
    uint64_t n_tiles;
    int64_t now_unix_ns;
} ctmr_tile_batch;

/* Caller-allocated outputs; per-entry arrays [n = sum of widths], any pointer may be NULL.  Only entries and tiles
 * before tiles_done are written. */
typedef struct ctmr_tile_out {
    ctmr_out path;            /* as ctmr_raw_out.path; pem_off has n + 1 entries */
    uint8_t* entry_status;    /* CTMR_FE_* (OK, BAD_CERT, BAD_TILE, BAD_INDEX) */
    uint8_t* entry_type;      /* CTMR_ENTRY_*; CTMR_ENTRY_OTHER for entries of a bad tile */
    uint64_t* timestamp_ms;
    uint32_t* issuer;         /* dense index of Chain[0], CTMR_ISSUER_NONE, CTMR_ISSUER_BAD */
    uint64_t* leaf_index;     /* the leaf_index extension's value (0 when absent or malformed) */
    uint64_t* leaf_off;       /* absolute offset in batch.data of the certificate the path processed (x509: the leaf,
                                 precert: pre_certificate), so the host can cut its DER; 0 with leaf_len 0 when dropped */
    uint32_t* leaf_len;
    uint8_t* leaf_hash;       /* [n][32] RFC 6962 §2.1 leaf hash SHA-256(00 || 00 00 || TimestampedEntry); zero for
                                 entries of a bad tile */
    uint8_t* tile_status;     /* [n_tiles] CTMR_FE_OK or CTMR_FE_BAD_TILE */
    uint8_t* missing_fp;      /* [missing_cap][32] */
    uint32_t missing_cap;
    uint64_t tiles_done;      /* written: tiles completed (n_tiles unless the call returned CTMR_E_UNKNOWN_ISSUER) */
    uint32_t n_missing;       /* written: fingerprints listed in missing_fp */
} ctmr_tile_out;

/* Split + frame + fingerprint -> dense index + map + reduce.  Synchronous.  Entries take the global indices following
 * those of earlier ctmr_process_batch / ctmr_process_raw / ctmr_process_tiles calls on this ctx.
 *
 * Chain[0] is looked up by fingerprint in a per-ctx table filled by ctmr_register_chain_certs; nothing is resolved on a
 * guess.  When tile k is the first tile holding a Chain[0] fingerprint the table does not know, tiles [0, k) are
 * completed with full outputs and indices, tiles_done = k, the distinct unknown fingerprints of tile k (sorted, at most
 * missing_cap) go to missing_fp, and the call returns CTMR_E_UNKNOWN_ISSUER; no entry of tile k or later touches the
 * tables or takes an index.  Register those certificates and call again with tiles [k, n_tiles): the combined result
 * equals one call made with every certificate registered beforehand.  A width outside 1..256 or a tile outside data is
 * CTMR_E_INVALID before any work; a tile larger than the front end's staging budget is CTMR_E_BATCH_TOO_LARGE. */
int ctmr_process_tiles(ctmr_ctx* ctx, const ctmr_tile_batch* batch, ctmr_tile_out* out);

/* The same on a group: each round takes one chunk of whole tiles per GPU out of ONE contiguous window of the batch and
 * runs as one round of the group's key exchange, so the outputs equal those of ctmr_process_tiles on one GPU. */
int ctmr_group_process_tiles(ctmr_group* g, const ctmr_tile_batch* batch, ctmr_tile_out* out);

/* CUDA-event time of tile_split (the serial per-tile walk) in the last ctmr_process_tiles call on this ctx, summed over
 * its chunks, in milliseconds: a part of the frontend_ms that ctmr_frontend_profile_last reports */
int ctmr_tiles_profile_last(ctmr_ctx* ctx, float* split_ms);

/* Chain certificates blob[offsets[k] .. offsets[k+1]) for k < n: SHA-256 fingerprint computed on the GPU, the certificate
 * registered as with ctmr_register_issuers (dense index, or CTMR_ISSUER_BAD when it does not parse), and
 * fingerprint -> dense index recorded in the ctx's fingerprint table.  The table holds 2 x config.max_issuers
 * fingerprints (CTMR_E_TOO_MANY_ISSUERS beyond that; a certificate that fails that way is not registered).  Like the
 * Chain[0] mirror it is cleared by ctmr_snapshot_load and is not part of a snapshot: register the certificates again
 * after a restore (they get the same dense indices).  fp_out ([n][32]) may be NULL. */
int ctmr_register_chain_certs(ctmr_ctx* ctx, const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint32_t* dense_out,
                              uint8_t* fp_out);
/* The same for every member of a group, from the group's one issuer registry. */
int ctmr_group_register_chain_certs(ctmr_group* g, const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint32_t* dense_out,
                                    uint8_t* fp_out);

/* ---- the log's Merkle tree (RFC 6962 §2.1) -----------------------------------------------------------------------------
 * A log signs only the root hash of its tree head (get-sth SHA256RootHash, a static-ct-api checkpoint's root hash): the
 * entries a client ingested are the log's entries when the Merkle tree over them has that root.  These calls fold every
 * entry of a batch into the tree on the GPU, next to the rest of the front end's work.
 *
 * The Merkle tree over the leaves [0, size) of ONE log, held as its right edge (compact range).  The struct holds no
 * pointers, so a Go caller may pass it from Go memory.  The root is r = edge[lowest set bit of size], then for each
 * higher set bit k in ascending order r = SHA-256(0x01 || edge[k] || r). */
typedef struct ctmr_tree {
    uint64_t size;          /* in/out: leaves folded in so far */
    uint8_t  edge[64][32];  /* in/out: for every bit k set in size, the MTH of the 2^k leaves
                               [(size >> (k+1)) << (k+1), that + 2^k); rows of clear bits are ignored on input, zero on output */
    uint8_t  root[32];      /* out: MTH(D[0:size]) after the call; SHA-256("") for size 0 */
} ctmr_tree;

/* ctmr_process_raw, and the batch's entries folded into *tree as leaves tree->size, tree->size + 1, ... of the log.  Every
 * output, the return code and the indices are those of ctmr_process_raw.  The leaf hash is SHA-256(0x00 || decoded
 * leaf_input); it needs no parse, so BAD_LEAF, UNKNOWN_TYPE, BAD_EXTRA and BAD_CERT entries fold too.  Only an entry whose
 * leaf_input is not base64 has no leaf: the fold stops before it and tree->size says where.  tree->size + n must not wrap
 * around 2^64 (CTMR_E_INVALID).  On an error *tree is left as it was passed in.  As with ctmr_process_raw, the batch's n
 * global indices are taken after any failure, this one included, so that a retry does not reuse them. */
int ctmr_process_raw_tree(ctmr_ctx* ctx, const ctmr_raw_batch* batch, ctmr_raw_out* out, ctmr_tree* tree);

/* ctmr_process_tiles, and the batch's entries folded into *tree.  Before any work, with no index taken and *tree untouched
 * (CTMR_E_INVALID otherwise): the tiles are consecutive (tile_index[t+1] == tile_index[t] + 1), every tile but the last is
 * full (width 256), 256 * tile_index[0] <= tree->size <= 256 * tile_index[0] + tile_width[0], and the last leaf index fits
 * 64 bits.  Leaves of the first tile below tree->size are already in the tree and are skipped.  A bad tile
 * (CTMR_FE_BAD_TILE) stops the fold at its first leaf not yet in the tree; the rest of the batch is processed as usual.
 * On the stop at an unknown Chain[0] (CTMR_E_UNKNOWN_ISSUER) *tree is written and holds the completed tiles.  Resume
 * from tiles_done in one of two ways:
 *   - tree->size >= 256 * tile_index[tiles_done]: no bad tile stopped the fold.  Call ctmr_process_tiles_tree again
 *     with the same tree;
 *   - tree->size is below that: a bad tile among the completed tiles stopped the fold, and the tree is final for this
 *     batch.  Call ctmr_process_tiles for the rest; a tree call would fail the size rule above.
 * Either way the tree and every output equal those of one call made with every certificate registered first.  On any
 * other error *tree is left as it was passed in. */
int ctmr_process_tiles_tree(ctmr_ctx* ctx, const ctmr_tile_batch* batch, ctmr_tile_out* out, ctmr_tree* tree);

/* ---- the Merkle trees of several logs in one call ---------------------------------------------------------------------
 * A client that syncs many logs at once drains the entries of all of them into one batch.  These calls fold each entry
 * into the tree of its own log; everything else -- outputs, return codes, global indices, PEM, the tiles' stop and
 * resume -- is exactly that of ctmr_process_raw / ctmr_process_tiles.
 *
 * Routing: entry i (pages), or every entry of tile t (tiles), is the next leaf of trees[entry_log[i]] (trees[tile_log[t]]);
 * CTMR_NO_TREE folds it into no tree.  The entries of one log appear in the batch in log order; they may be interleaved
 * with other logs' in any way (page by page, entry by entry, tile by tile).  Each tree keeps the rules of the one-tree
 * call on its own entries: the leaf hash is SHA-256(0x00 || decoded leaf_input), only bad base64 has no leaf and stops
 * that tree's fold (no other tree's), and size + (entries of that log) must not wrap around 2^64 (pages); the log's tiles
 * in batch order are consecutive, all full but its last, the tree's size lies inside its first tile (leaves below it are
 * skipped), its last leaf index fits 64 bits, and a bad tile stops only its own log's fold (tiles).
 *
 * Before any work, with no index taken and no tree touched, CTMR_E_INVALID for: trees NULL with n_trees > 0, entry_log /
 * tile_log NULL with entries / tiles in the batch, n_trees > CTMR_MAX_TREES, a log id >= n_trees that is not
 * CTMR_NO_TREE, or a broken per-log rule.  Every tree passed in gets its root written, also a tree of no entry in the
 * batch; rows of clear bits come back zero.  On CTMR_E_UNKNOWN_ISSUER (tiles) every tree is written back holding the
 * completed tiles; on any other error every tree is left as passed in.  A member of a group is refused. */
#define CTMR_NO_TREE 0xFFFFFFFFu
#define CTMR_MAX_TREES 1024u   /* well above the number of logs any CT log list names */

int ctmr_process_raw_trees(ctmr_ctx* ctx, const ctmr_raw_batch* batch, ctmr_raw_out* out,
                           const uint32_t* entry_log /* [n] */, ctmr_tree* trees, uint32_t n_trees);

/* Resume after CTMR_E_UNKNOWN_ISSUER from tiles_done: a log whose written-back tree->size is below 256 * tile_index of its
 * first tile in the rest of the batch was stopped by a bad tile, and its tree is final for this batch: pass that log's
 * remaining tiles as CTMR_NO_TREE.  Every other log resumes with its tree.  The trees and every output then equal those
 * of one call made with every certificate registered first. */
int ctmr_process_tiles_trees(ctmr_ctx* ctx, const ctmr_tile_batch* batch, ctmr_tile_out* out,
                             const uint32_t* tile_log /* [n_tiles] */, ctmr_tree* trees, uint32_t n_trees);

/* ---- the trees on a group ----------------------------------------------------------------------------------------------
 * The four tree calls on every GPU of a group (ctmr_group_create, ctmr.h).  Every output, return code, global index,
 * PEM text, tiles_done, missing_fp and n_missing is that of ctmr_group_process_raw / ctmr_group_process_tiles on the
 * same group, and every tree is that of the matching one-ctx call on the same batch, with all of its rules: the argument
 * and per-log checks before any work (no index taken, no tree touched), the leaves that stop a fold, the leaves of a
 * first tile below size, the trees written back at CTMR_E_UNKNOWN_ISSUER with the same resume rules, and every tree left
 * as passed in on any other error.  A member ctx keeps refusing the one-ctx tree forms: a group's trees go through the
 * group handle.
 *
 * In each round the first GPU of the group folds its chunk into the trees; every other GPU folds its chunk into a
 * compact range per tree (at most 64 left and 64 right nodes), and the first GPU appends those ranges in member order
 * after the round. */
int ctmr_group_process_raw_tree(ctmr_group* g, const ctmr_raw_batch* batch, ctmr_raw_out* out, ctmr_tree* tree);
int ctmr_group_process_tiles_tree(ctmr_group* g, const ctmr_tile_batch* batch, ctmr_tile_out* out, ctmr_tree* tree);
int ctmr_group_process_raw_trees(ctmr_group* g, const ctmr_raw_batch* batch, ctmr_raw_out* out,
                                 const uint32_t* entry_log /* [n] */, ctmr_tree* trees, uint32_t n_trees);
int ctmr_group_process_tiles_trees(ctmr_group* g, const ctmr_tile_batch* batch, ctmr_tile_out* out,
                                   const uint32_t* tile_log /* [n_tiles] */, ctmr_tree* trees, uint32_t n_trees);

/* ---- the trees from whole get-entries bodies ---------------------------------------------------------------------------
 * ctmr_process_raw_bodies / ctmr_group_process_raw_bodies, and each body's entries folded into its log's tree.  Every
 * output, the return code, the global indices, body statuses, spans, PEM and string identities are those of the plain
 * bodies call on the same batch.  body_start[b] is the start of the get-entries request that body b answers: entry j of
 * the body is log position body_start[b] + j.  The one-tree forms fold every body into *tree; the routed forms fold body
 * b into trees[body_log[b]], none for CTMR_NO_TREE.
 *
 * Before any work, with no index taken and no tree touched, CTMR_E_INVALID for: body_start NULL with bodies in the
 * batch, body_log NULL in the routed forms, a log id >= n_trees that is not CTMR_NO_TREE, n_trees > CTMR_MAX_TREES, and
 * per log in batch order: starts that decrease, a first body with start > tree.size, a start + body_max that wraps
 * around 2^64.
 *
 * A log may answer a get-entries request with fewer entries than were asked for, so the bodies of a client that
 * pipelines its requests may leave gaps or overlap.  Each tree walks its log's bodies in batch order with end = its size
 * at the start of the call:
 *   - a body that is not CTMR_BODY_OK stops the fold at end: its entries' positions are unknown;
 *   - a body with start > end is a gap: the fold stops at end;
 *   - otherwise its entries below end are already in the tree and are skipped unchecked, the rest are appended (the
 *     first one whose leaf_input is not base64 stops the fold there), and end = max(end, start + entries).
 * A stop is final for the call: tree->size says where to fetch again.  The leaf hash is that of the pages form
 * (SHA-256(0x00 || decoded leaf_input)), so BAD_LEAF, BAD_EXTRA, UNKNOWN_TYPE and BAD_CERT entries fold.  Every tree
 * passed in gets its root written; on any error every tree is left as passed in.  A member of a group is refused the
 * one-ctx forms. */
int ctmr_process_raw_bodies_tree(ctmr_ctx* ctx, const ctmr_body_batch* batch, ctmr_body_out* out,
                                 const uint64_t* body_start /* [n_bodies] */, ctmr_tree* tree);
int ctmr_process_raw_bodies_trees(ctmr_ctx* ctx, const ctmr_body_batch* batch, ctmr_body_out* out,
                                  const uint32_t* body_log /* [n_bodies] */, const uint64_t* body_start /* [n_bodies] */,
                                  ctmr_tree* trees, uint32_t n_trees);
int ctmr_group_process_raw_bodies_tree(ctmr_group* g, const ctmr_body_batch* batch, ctmr_body_out* out,
                                       const uint64_t* body_start /* [n_bodies] */, ctmr_tree* tree);
int ctmr_group_process_raw_bodies_trees(ctmr_group* g, const ctmr_body_batch* batch, ctmr_body_out* out,
                                        const uint32_t* body_log /* [n_bodies] */, const uint64_t* body_start /* [n_bodies] */,
                                        ctmr_tree* trees, uint32_t n_trees);

/* ---- one process per GPU: the front end as a collective call ------------------------------------------------------------
 * On a ctx attached to peers (ctmr_peer_attach, ctmr.h, world > 1) ctmr_process_raw, ctmr_process_raw_bodies,
 * ctmr_process_tiles, ctmr_process_raw_tree, ctmr_process_tiles_tree, ctmr_process_raw_trees, ctmr_process_tiles_trees,
 * ctmr_process_raw_bodies_tree and ctmr_process_raw_bodies_trees are COLLECTIVE.
 * Each rank passes its own batch, and each front-end call on one rank must meet a front-end call on every other rank.
 * The entry points may differ between the ranks of one call (pages on one rank, tiles with trees on another): their
 * collective steps are the same.  A front-end call met by ctmr_process_batch, ctmr_process_device or any other
 * collective call on another rank is undefined, as is any other mismatch of the collective sequence.
 *
 * Agreement.  Each rank checks its arguments (the rules of its entry point, trees included), builds what the call
 * needs and cuts its whole batch into chunks exactly as on one GPU, E entries at most per chunk, before any upload:
 * bad spans, widths or tree rules are CTMR_E_INVALID and an entry or tile beyond the staging budget is
 * CTMR_E_BATCH_TOO_LARGE at this point.  E is the front end's entry budget (config.max_batch_entries), which the
 * key-exchange regions always hold; when ranks were created with different budgets the largest is used in the index
 * rule.  The ranks then exchange, through peer memory, their chunk counts, whether they want the string identities
 * (first_issuer_dn / first_crldp) and whether their checks failed.  If any rank's checks failed, every rank returns
 * before any index is taken or any table or tree changes: that rank with its own error, the others with
 * CTMR_E_PEER_FAILED.  So an argument mistake that the library sees on one rank -- a NULL batch, output or tree
 * included -- never leaves the others waiting at a barrier.  A rank that skips the call, for instance because its own
 * code refused the arguments before calling, does: such a rank still makes the call (a NULL batch will do), so that
 * the others return CTMR_E_PEER_FAILED.
 *
 * Rounds and indices.  Otherwise every rank runs R = the largest chunk count (at least 1) rounds of the key exchange;
 * a rank that has run out of chunks runs its remaining rounds empty.  Entry j of rank r's chunk in round k takes the
 * global index next_index + (k * world + r) * E + j, the rule of the collective ctmr_process_batch, so the result
 * equals the sequential run over the rounds, inside a round the ranks in order.  Every rank advances its next index by
 * R * world * E once the agreement has succeeded, whatever happens after, and by nothing when it failed
 * (ctmr_next_index reads it, e.g. to place a later ctmr_process_device call's first_index).  When any rank
 * wants the string identities every rank computes them (its entries then count for the first-seen rules) and
 * returns them where its caller asked.
 *
 * Stops and failures after the agreement.  A tiles stop at an unknown Chain[0] fingerprint ends the rank's part at the
 * stop tile, as on one GPU (tiles_done, missing_fp, CTMR_E_UNKNOWN_ISSUER); the rank runs its remaining rounds empty.
 * A front or back half that fails with a library error does the same and returns that error at the end of the call:
 * CTMR_E_TOO_MANY_ISSUERS (the issuer registry or the Chain[0] mirror is full), CTMR_E_BATCH_TOO_LARGE (pem_cap too
 * small), and a table that filled up (CTMR_E_TABLE_FULL, CTMR_E_PAIR_TABLE_FULL, CTMR_E_META_TABLE_FULL).  A CUDA error
 * (CTMR_E_CUDA, CTMR_E_NOMEM of a device allocation) that leaves the GPU unable to run the remaining barriers ends the
 * rank's part at once, and the other ranks wait until CTMR_E_PEER_TIMEOUT, as in every collective call.
 *
 * Resume.  The call ends with one more exchange, so that every rank knows how many ranks stopped at an unknown
 * fingerprint: ctmr_peer_frontend_stopped.  A resume loop keeps calling on every rank while it is non-zero; a rank with
 * nothing left passes an empty batch.  A rank whose own call failed is not counted (it has nothing to resume), but
 * while the count is non-zero the others call again, so it joins those calls with an empty batch before it gives up.
 *
 * Trees.  Each rank folds its own batch's entries into its own caller-held trees, with the one-GPU rules: log order is
 * batch order on that rank, and global indices do not enter the tree.  Members of an in-process group (ctmr_group_*)
 * keep refusing the one-ctx tree forms; the group's own tree calls are above. */

/* *ranks = the ranks that stopped at an unknown Chain[0] fingerprint (CTMR_E_UNKNOWN_ISSUER) in the last collective
 * front-end call on this ctx; 0 after a call that failed before any work.  CTMR_E_INVALID on a ctx not attached to
 * peers. */
int ctmr_peer_frontend_stopped(ctmr_ctx* ctx, uint32_t* ranks);

#ifdef __cplusplus
}
#endif
#endif /* CTMR_FRONTEND_H */
