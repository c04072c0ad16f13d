/*
 * ctmr_oracle.h -- CPU ORACLE for the CT-entry map/reduce hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This is a plain-C restatement of the reference's algorithm for the one path this repository
 * accelerates (SURVEY.md §8): cmd/ct-fetch/ct-fetch.go:44-70,180-246 (worker + filter),
 * storage/filesystemdatabase.go:158-240 (Store), storage/types.go:104-178,333-384 (Issuer ID,
 * raw serial, hour truncation), storage/knowncertificates.go:28-63 (set key, first-insert-true),
 * storage/issuermetadata.go:92-138 (first-seen expDate memo), storage/mockcache.go:38-61,120-122
 * (set semantics) and cmd/storage-statistics/storage-statistics.go:36-82 (per-issuer counts).
 * The X.509 parse itself lives in a third-party dependency that is NOT in the reference repository:
 * github.com/google/certificate-transparency-go v1.1.0 (go.mod:10), packages x509/asn1/pkix; it
 * is restated here from RFC 5280 §4.1 / X.690 DER plus the Go behaviours the call sites rely on.
 *
 * Nothing in the product path (ct_mapreduce_b200/, include/) may call into this file.  Only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it,
 * and there only as the checker / the timed CPU arm.
 *
 * Parity pinning (SURVEY.md §8(c)): the leaves are pinned by the reference's own known-answer
 * tests (tests/test_oracle_kat.py): storage/types_test.go:41-57 (SHA-256 + base64url),
 * :81-101 (raw serial 00aa from PEM kLeadingZeroes), :203-252 (ExpDate), knowncertificates_test.go
 * :11-55,:85-110 (set semantics, key string), issuermetadata_test.go:100-136 (seenBefore).  The
 * COMPOSED map path (insertCTWorker -> certIsFilteredOut -> Store) has no test in the reference
 * and the Go toolchain is absent here, so for CommonName / NotAfter / IsCA extraction the status
 * is "parity unpinned" against Go; those fields are cross-checked against Python `cryptography`
 * (an independent X.509 parser) in tests/test_oracle_vs_cryptography.py.
 */
#ifndef CTMR_ORACLE_H
#define CTMR_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* per-entry status, same numeric values as include/ctmr.h */
enum {
    ORA_ST_OK = 0,
    ORA_ST_PARSE_ERR = 1,        /* ct-fetch.go:206-209 */
    ORA_ST_FILTER_CA = 2,        /* ct-fetch.go:47-50  */
    ORA_ST_FILTER_EXPIRED = 3,   /* ct-fetch.go:52-55  */
    ORA_ST_FILTER_CN = 4,        /* ct-fetch.go:57-68  */
    ORA_ST_NO_ISSUER = 5,        /* ct-fetch.go:215-219 */
    ORA_ST_ISSUER_PARSE_ERR = 6, /* ct-fetch.go:221-225 */
    ORA_ST_SERIAL_TOO_LONG = 7   /* never produced by the oracle (the reference has no limit); the GPU path declines serials > 39 octets */
};

typedef struct ora_cert {
    uint32_t tbs_off, tbs_len;         /* RawTBSCertificate (full TLV) */
    uint32_t serial_off, serial_len;   /* INTEGER content octets, types.go:171-178 */
    uint32_t issuer_off, issuer_len;   /* issuer Name, full TLV */
    uint32_t cn_off, cn_len;           /* last 2.5.4.3 string value of the issuer; has_cn=0 -> "" */
    uint32_t spki_off, spki_len;       /* RawSubjectPublicKeyInfo (full TLV), types.go:112 */
    uint32_t crldp_off, crldp_len;     /* extnValue content of cRLDistributionPoints, 0 if absent */
    int64_t not_before, not_after;     /* unix seconds */
    int32_t has_cn;
    int32_t bc_valid, is_ca;           /* BasicConstraintsValid / IsCA (ct-fetch.go:47) */
} ora_cert;

void ora_sha256(const uint8_t* msg, size_t len, uint8_t out[32]);
size_t ora_b64url(const uint8_t* in, size_t n, char* out); /* padded URL alphabet; NUL-terminates */
int ora_parse_cert(const uint8_t* der, size_t len, ora_cert* out); /* 0 = ok, <0 = parse error */
int ora_parse_tbs(const uint8_t* tbs, size_t len, ora_cert* out);  /* ct-go x509.ParseTBSCertificate; offsets relative to tbs */

void ora_issuer_id(const uint8_t* spki, size_t len, uint8_t digest[32], char id[45]);
int64_t ora_exp_hour(int64_t not_after_sec);
void ora_expdate_id(int64_t exp_hour, char out[14]);
void ora_day_id(int64_t not_after_sec, char out[11]);

/* 0 = kept, else ORA_ST_FILTER_* ; filter = raw issuerCNFilter config string */
int ora_filter(const uint8_t* der, const ora_cert* c, const uint8_t* filter, size_t filter_len, int log_expired,
               int64_t now_unix_ns);

/* ---- sets with MockRemoteCache semantics (mockcache.go:38-61,120-122) ---- */
typedef struct ora_cache ora_cache;
ora_cache* ora_cache_new(void);
void ora_cache_free(ora_cache*);
int ora_cache_set_insert(ora_cache*, const char* key, size_t key_len, const uint8_t* member, size_t member_len);
uint64_t ora_cache_set_cardinality(ora_cache*, const char* key, size_t key_len);
/* sorted members of one set, concatenated as (u32 len, bytes)*; returns count */
uint64_t ora_cache_set_list(ora_cache*, const char* key, size_t key_len, uint8_t* buf, size_t buf_cap, size_t* used);

/* ---- KnownCertificates over that cache (knowncertificates.go) ---- */
size_t ora_serials_key(int64_t exp_hour, const char* issuer_id, char* out, size_t cap);
int ora_was_unknown(ora_cache*, int64_t exp_hour, const char* issuer_id, const uint8_t* serial, size_t serial_len);

/* ---- the composed path: insertCTWorker + Store, sequential (numThreads=1) ---- */
typedef struct ora_db ora_db;
ora_db* ora_db_new(const uint8_t* filter, size_t filter_len, int log_expired);
void ora_db_free(ora_db*);

typedef struct ora_out {
    uint8_t* status;          /* [n] */
    uint8_t* sha256;          /* [n][32]  SHA-256 of the leaf DER (north_star output, M3) */
    int64_t* exp_hour;        /* [n] valid when leaf parsed */
    uint32_t* serial_off;     /* [n] offset inside the entry's DER */
    uint32_t* serial_len;     /* [n] */
    uint8_t* was_unknown;     /* [n] knowncertificates.go:38-55 */
    uint8_t* first_issuer_hour; /* [n] !seenExpDateBefore, issuermetadata.go:95-108 */
    /* IssuerMetadata string reducers (issuermetadata.go:110-135), may be NULL as a group */
    uint32_t* issuer_name_off;  /* [n] issuer Name TLV span */
    uint32_t* issuer_name_len;
    uint32_t* crldp_off;        /* [n] cRLDistributionPoints extnValue content span */
    uint32_t* crldp_len;
    uint8_t* first_issuer_dn;   /* [n] new certificate whose (issuer, Name bytes) was not seen on an earlier new certificate */
    uint8_t* first_crldp;       /* [n] same for (issuer, cRLDistributionPoints bytes) */
} ora_out;

/* issuer_idx[i] == 0xFFFFFFFF means len(Chain) < 1.  nthreads>1 parallelises the map half only. */
int ora_db_process(ora_db*, const uint8_t* blob, const uint64_t* offsets, uint64_t n, const uint8_t* issuer_blob,
                   const uint64_t* issuer_offsets, uint32_t n_issuers, const uint32_t* issuer_idx,
                   int64_t now_unix_ns, int nthreads, ora_out* out);

/* issuer ids (raw 32-byte digests) and Count()-sum per issuer, sorted by digest; returns count */
uint64_t ora_db_issuer_counts(ora_db*, uint8_t* ids32, uint64_t* counts, uint64_t cap);
uint64_t ora_db_set_cardinality(ora_db*, int64_t exp_hour, const uint8_t issuer_digest[32]);
void ora_db_filter_counters(ora_db*, uint64_t out[8]); /* indexed by status code */
uint64_t ora_db_evict_expired(ora_db*, int64_t now_unix_sec); /* Redis TTLs firing: sets with expDate <= now vanish */

/* timed CPU arm: map-only over a batch (parse + filter + both SHA-256), returns entries kept */
uint64_t ora_map_only(const uint8_t* blob, const uint64_t* offsets, uint64_t n, const uint8_t* filter,
                      size_t filter_len, int log_expired, int64_t now_unix_ns, int nthreads, uint8_t* sha_out);

/* ---- CT wire-format front end (ctmr_oracle_frontend.c; SURVEY.md §8(f)-2) ---- */
enum { /* same numeric values as CTMR_FE_* in include/ctmr_frontend.h */
    ORA_FE_OK = 0, ORA_FE_BAD_BASE64 = 1, ORA_FE_BAD_LEAF = 2, ORA_FE_UNKNOWN_TYPE = 3, ORA_FE_BAD_EXTRA = 4, ORA_FE_BAD_CERT = 5
};
typedef struct ora_entry {
    uint64_t timestamp_ms;            /* TimestampedEntry.timestamp */
    uint32_t entry_type;              /* 0 x509_entry, 1 precert_entry, 0xFF anything else */
    uint32_t leaf_src;                /* certificate insertCTWorker processes: 0 = inside leaf_input, 1 = inside extra_data */
    uint32_t leaf_off, leaf_len;
    uint32_t chain0_off, chain0_len;  /* Chain[0] inside extra_data; len 0 = empty chain */
    uint32_t chain_count;
    uint32_t tbs_off, tbs_len;        /* precert entries: TBSCertificate inside leaf_input */
} ora_entry;
long ora_b64_decode(const uint8_t* in, size_t n, uint8_t* out, size_t cap); /* base64.StdEncoding; -1 = corrupt input */
int ora_entry_from_leaf(const uint8_t* leaf_input, size_t nl, const uint8_t* extra_data, size_t ne, ora_entry* e); /* ORA_FE_* */

/* synthetic corpus (ct_mapreduce_b200/csrc/ctmr_synth.h) on the CPU */
struct ctmr_synth_cfg;
uint64_t ora_synth_lengths(const struct ctmr_synth_cfg*, uint64_t first, uint64_t n, uint64_t* offsets_out /* n+1 */);
void ora_synth_write(const struct ctmr_synth_cfg*, uint64_t first, uint64_t n, const uint64_t* offsets, uint8_t* blob);
void ora_synth_issuer_idx(const struct ctmr_synth_cfg*, uint64_t first, uint64_t n, uint32_t* idx_out);
uint64_t ora_synth_issuers(const struct ctmr_synth_cfg*, uint64_t* offsets_out /* n_issuers+1 */, uint8_t* blob, size_t cap);

#ifdef __cplusplus
}
#endif
#endif
