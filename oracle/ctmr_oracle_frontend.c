/*
 * ctmr_oracle_frontend.c -- CPU ORACLE for the CT wire-format front end (SURVEY.md §8(f)-2).
 * TEST INFRASTRUCTURE ONLY: nothing under ct_mapreduce_b200/ or include/ may call into it.
 *
 * Restates what happens to one get-entries entry between the HTTP body and the worker's channel
 * in the reference:
 *   - encoding/json decodes "leaf_input" / "extra_data" ([]byte fields of ct.LeafEntry) with
 *     base64.StdEncoding, inside ct-go jsonclient under LogClient.GetRawEntries
 *     (cmd/ct-fetch/ct-fetch.go:424);
 *   - ct.LogEntryFromLeaf (cmd/ct-fetch/ct-fetch.go:452): tls.Unmarshal of MerkleTreeLeaf, then of
 *     CertificateChain or PrecertChainEntry, "trailing data" errors, X509Certificate() /
 *     Precertificate() parses; fatal errors drop the entry (ct-fetch.go:453-460);
 *   - insertCTWorker's entry-type switch (ct-fetch.go:198-204) picks the certificate to process and
 *     Chain[0] is the issuer (ct-fetch.go:215-221).
 *
 * github.com/google/certificate-transparency-go v1.1.0 (go.mod:10) is NOT in the reference repository, so the
 * structures are restated from RFC 6962 §3.4 / §4.6 and RFC 5246 §4 (TLS presentation language) with the
 * struct tags that release publishes in types.go:
 *     MerkleTreeLeaf   { Version tls.Enum `maxval:255`; LeafType tls.Enum `maxval:255`;
 *                        TimestampedEntry *TimestampedEntry `selector:LeafType,val:0` }
 *     TimestampedEntry { Timestamp uint64; EntryType tls.Enum `maxval:65535`;
 *                        X509Entry *ASN1Cert `selector:EntryType,val:0`;
 *                        PrecertEntry *PreCert `selector:EntryType,val:1`;
 *                        JSONEntry *JSONDataEntry `selector:EntryType,val:32768`;
 *                        Extensions CTExtensions `minlen:0,maxlen:65535` }
 *     ASN1Cert         { Data []byte `minlen:1,maxlen:16777215` }
 *     PreCert          { IssuerKeyHash [32]byte; TBSCertificate []byte `minlen:1,maxlen:16777215` }
 *     CertificateChain { Entries []ASN1Cert `minlen:0,maxlen:16777215` }
 *     PrecertChainEntry{ PreCertificate ASN1Cert; CertificateChain []ASN1Cert `minlen:0,maxlen:16777215` }
 * Parity status: "parity unpinned" against ct-go itself (no Go toolchain, source absent); pinned against
 * hand-built RFC 6962 vectors and Python's base64 / struct in tests/test_frontend_oracle.py.
 */
#include <stdlib.h>
#include <string.h>

#include "ctmr_oracle.h"

/* base64.StdEncoding.DecodeString as reached from encoding/json: padded, standard alphabet.  (Go's decoder
 * also skips '\r' and '\n'; a JSON string cannot contain them raw, so the case does not arise here and both
 * this oracle and the GPU reject them.)  Returns decoded length, or -1. */
long ora_b64_decode(const uint8_t* in, size_t n, uint8_t* out, size_t cap) {
    static int8_t lut[256];
    static int init = 0;
    if (!init) {
        memset(lut, -1, sizeof lut);
        const char* al = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
        for (int i = 0; i < 64; ++i) lut[(uint8_t)al[i]] = (int8_t)i;
        init = 1;
    }
    if (n % 4) return -1;
    size_t o = 0;
    for (size_t i = 0; i < n; i += 4) {
        int pad = 0;
        uint32_t v = 0;
        for (int k = 0; k < 4; ++k) {
            uint8_t ch = in[i + k];
            if (ch == '=' && i + 4 == n && k >= 2 && (k == 3 || in[i + 3] == '=')) {
                ++pad;
                v <<= 6;
                continue;
            }
            if (lut[ch] < 0) return -1;
            v = (v << 6) | (uint32_t)lut[ch];
        }
        const int nb = 3 - pad;
        if (o + (size_t)nb > cap) return -1;
        if (nb > 0) out[o++] = (uint8_t)(v >> 16);
        if (nb > 1) out[o++] = (uint8_t)(v >> 8);
        if (nb > 2) out[o++] = (uint8_t)v;
    }
    return (long)o;
}

static uint32_t be24(const uint8_t* d) { return ((uint32_t)d[0] << 16) | ((uint32_t)d[1] << 8) | d[2]; }

/* []ASN1Cert filling d[q..end) exactly; first element reported */
static int walk_chain(const uint8_t* d, size_t q, size_t end, uint32_t* first_off, uint32_t* first_len, uint32_t* count) {
    *first_off = *first_len = *count = 0;
    while (q < end) {
        if (q + 3 > end) return -1;
        uint32_t l = be24(d + q);
        if (l == 0 || l > end - q - 3) return -1;
        if (*count == 0) { *first_off = (uint32_t)(q + 3); *first_len = l; }
        ++*count;
        q += 3 + (size_t)l;
    }
    return 0;
}

/* One entry, already base64-decoded.  Returns ORA_FE_*; fills *e for ORA_FE_OK (and entry_type / timestamp
 * whenever the leaf header could be read). */
int ora_entry_from_leaf(const uint8_t* li, size_t nl, const uint8_t* ed, size_t ne, ora_entry* e) {
    memset(e, 0, sizeof *e);
    e->entry_type = 0xFF;
    if (nl < 12 || li[1] != 0) return ORA_FE_BAD_LEAF; /* LeafType selector has only val:0 */
    for (int k = 0; k < 8; ++k) e->timestamp_ms = (e->timestamp_ms << 8) | li[2 + k];
    uint32_t t = ((uint32_t)li[10] << 8) | li[11];
    size_t q = 12;
    if (t == 0) e->entry_type = 0;
    else if (t == 1) { e->entry_type = 1; q += 32; }
    else return ORA_FE_UNKNOWN_TYPE; /* 0x8000 (JSON) unmarshals but LogEntryFromLeaf rejects it; others fail in Unmarshal */
    if (q + 3 > nl) return ORA_FE_BAD_LEAF;
    uint32_t l = be24(li + q);
    if (l == 0 || l > nl - q - 3) return ORA_FE_BAD_LEAF;
    size_t body = q + 3;
    q = body + l;
    if (q + 2 > nl) return ORA_FE_BAD_LEAF;
    size_t xl = ((size_t)li[q] << 8) | li[q + 1];
    if (q + 2 + xl != nl) return ORA_FE_BAD_LEAF; /* short, or "trailing data after MerkleTreeLeaf" */
    size_t q2 = 0;
    if (e->entry_type == 0) {
        e->leaf_src = 0; e->leaf_off = (uint32_t)body; e->leaf_len = l;
    } else {
        e->tbs_off = (uint32_t)body; e->tbs_len = l;
        if (ne < 3) return ORA_FE_BAD_EXTRA;
        uint32_t pl = be24(ed);
        if (pl == 0 || pl > ne - 3) return ORA_FE_BAD_EXTRA;
        e->leaf_src = 1; e->leaf_off = 3; e->leaf_len = pl;
        q2 = 3 + (size_t)pl;
    }
    if (q2 + 3 > ne) return ORA_FE_BAD_EXTRA;
    if (q2 + 3 + (size_t)be24(ed + q2) != ne) return ORA_FE_BAD_EXTRA;
    if (walk_chain(ed, q2 + 3, ne, &e->chain0_off, &e->chain0_len, &e->chain_count)) return ORA_FE_BAD_EXTRA;
    if (e->entry_type == 1) { /* MerkleTreeLeaf.Precertificate(): x509.ParseTBSCertificate */
        ora_cert c;
        if (ora_parse_tbs(li + e->tbs_off, e->tbs_len, &c)) return ORA_FE_BAD_CERT;
    } else { /* MerkleTreeLeaf.X509Certificate(): x509.ParseCertificate */
        ora_cert c;
        if (ora_parse_cert(li + e->leaf_off, e->leaf_len, &c)) return ORA_FE_BAD_CERT;
    }
    return ORA_FE_OK;
}
