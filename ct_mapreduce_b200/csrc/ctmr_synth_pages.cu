// ctmr_synth_pages.cu -- HOST-side synthesis of RFC 6962 get-entries response bodies and of static-ct-api data tiles around
// the synthetic corpus
// (bench / test tooling for the CT wire-format front end; nothing here runs on the GPU or inside a timed region).
// Byte-identical to tools/bench_frontend.py's Python construction (tests/test_frontend_oracle.py checks that), but
// threaded and ~100x faster, so that a benchmark does not spend its GPU-box minutes building input.
#include <algorithm>
#include <array>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../include/ctmr.h"
#include "ctmr_synth.h"

namespace {

// FIPS 180-4 SHA-256 on the host: PreCert.issuer_key_hash of the synthetic entries is SHA-256 of the issuer
// certificate (any 32 bytes would do for the path; the Python generator uses this value)
struct Sha256 {
    uint32_t h[8];
    static uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
    static void block(uint32_t* h, const uint8_t* p) {
        static const uint32_t K[64] = {
            0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be,
            0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa,
            0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85,
            0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3,
            0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f,
            0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
        uint32_t w[64];
        for (int i = 0; i < 16; ++i) w[i] = ((uint32_t)p[4 * i] << 24) | ((uint32_t)p[4 * i + 1] << 16) | ((uint32_t)p[4 * i + 2] << 8) | p[4 * i + 3];
        for (int i = 16; i < 64; ++i) {
            const uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3), s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
            w[i] = w[i - 16] + s0 + w[i - 7] + s1;
        }
        uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
        for (int i = 0; i < 64; ++i) {
            const uint32_t t1 = hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + K[i] + w[i];
            const uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
            hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
        h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
    }
    static void digest(const uint8_t* msg, size_t n, uint8_t out[32]) {
        uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
        size_t i = 0;
        for (; i + 64 <= n; i += 64) block(h, msg + i);
        uint8_t tail[128] = {0};
        const size_t rem = n - i;
        std::memcpy(tail, msg + i, rem);
        tail[rem] = 0x80;
        const size_t tl = rem + 9 <= 64 ? 64 : 128;
        const uint64_t bits = (uint64_t)n * 8;
        for (int k = 0; k < 8; ++k) tail[tl - 1 - k] = (uint8_t)(bits >> (8 * k));
        block(h, tail);
        if (tl == 128) block(h, tail + 64);
        for (int k = 0; k < 8; ++k) { out[4 * k] = (uint8_t)(h[k] >> 24); out[4 * k + 1] = (uint8_t)(h[k] >> 16); out[4 * k + 2] = (uint8_t)(h[k] >> 8); out[4 * k + 3] = (uint8_t)h[k]; }
    }
};

size_t b64_len(size_t n) { return (n + 2) / 3 * 4; }

uint8_t* b64_put(uint8_t* o, const uint8_t* d, size_t n) {
    static const char A[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    size_t i = 0;
    for (; i + 3 <= n; i += 3) {
        const uint32_t w = ((uint32_t)d[i] << 16) | ((uint32_t)d[i + 1] << 8) | d[i + 2];
        *o++ = A[w >> 18]; *o++ = A[(w >> 12) & 63]; *o++ = A[(w >> 6) & 63]; *o++ = A[w & 63];
    }
    if (n - i == 1) {
        const uint32_t w = (uint32_t)d[i] << 16;
        *o++ = A[w >> 18]; *o++ = A[(w >> 12) & 63]; *o++ = '='; *o++ = '=';
    } else if (n - i == 2) {
        const uint32_t w = ((uint32_t)d[i] << 16) | ((uint32_t)d[i + 1] << 8);
        *o++ = A[w >> 18]; *o++ = A[(w >> 12) & 63]; *o++ = A[(w >> 6) & 63]; *o++ = '=';
    }
    return o;
}

void put24(std::vector<uint8_t>& v, size_t n) { v.push_back((uint8_t)(n >> 16)); v.push_back((uint8_t)(n >> 8)); v.push_back((uint8_t)n); }
void put_opaque24(std::vector<uint8_t>& v, const uint8_t* d, size_t n) { put24(v, n); v.insert(v.end(), d, d + n); }

// header length of the DER TLV at p (definite lengths as the generator writes them)
size_t der_hdr(const uint8_t* p) { return p[1] < 0x80 ? 2 : 2 + (p[1] & 0x7f); }
size_t der_len(const uint8_t* p) {
    if (p[1] < 0x80) return p[1];
    size_t n = 0;
    for (int k = 0; k < (p[1] & 0x7f); ++k) n = (n << 8) | p[2 + k];
    return n;
}

struct Issuers {
    std::vector<std::vector<uint8_t>> der;
    std::vector<std::array<uint8_t, 32>> key_hash;
};

// Synthetic entry i, the part both formats share (the construction of tools/bench_frontend.py: every third entry a
// precert_entry, chains of one or two certificates, timestamps 1 690 000 000 000 + i): the leaf certificate, and the
// TimestampedEntry up to its CtExtensions (timestamp, entry_type, ASN.1Cert or PreCert) in `te`.
struct SynthEntry {
    uint32_t chain[2];  // issuers of Chain[0] and Chain[1]
    int n_chain;
    bool precert;
};

SynthEntry synth_entry(const ctmr_synth_cfg* cfg, const Issuers& iss, uint64_t i, std::vector<uint8_t>& leaf, std::vector<uint8_t>& te) {
    ctmr_synth_plan pl;
    ctmr_synth_plan_make(cfg, i, &pl);
    leaf.resize(ctmr_synth_cert_len(cfg, i));
    ctmr_synth_cert_write(cfg, &pl, leaf.data());
    SynthEntry e{{pl.issuer, (pl.issuer + 1) % cfg->n_issuers}, 1 + (int)(i % 2), i % 3 == 0};
    te.clear();
    const uint64_t ts = 1690000000000ull + i;
    for (int b = 7; b >= 0; --b) te.push_back((uint8_t)(ts >> (8 * b)));
    te.push_back(0); te.push_back(e.precert ? 1 : 0);
    if (e.precert) {  // PreCert: issuer_key_hash, TBSCertificate
        te.insert(te.end(), iss.key_hash[e.chain[0]].begin(), iss.key_hash[e.chain[0]].end());
        const uint8_t* tbs = leaf.data() + der_hdr(leaf.data());
        put_opaque24(te, tbs, der_hdr(tbs) + der_len(tbs));
    } else {
        put_opaque24(te, leaf.data(), leaf.size());
    }
    return e;
}

// leaf_input / extra_data of synthetic entry i as a get-entries entry: no CtExtensions, the chain as DERs
void make_entry(const ctmr_synth_cfg* cfg, const Issuers& iss, uint64_t i, std::vector<uint8_t>& leaf, std::vector<uint8_t>& li,
                std::vector<uint8_t>& ed) {
    std::vector<uint8_t> te;
    const SynthEntry e = synth_entry(cfg, iss, i, leaf, te);
    std::vector<uint8_t> chain;
    for (int m = 0; m < e.n_chain; ++m) put_opaque24(chain, iss.der[e.chain[m]].data(), iss.der[e.chain[m]].size());
    li.assign({0, 0});  // v1, timestamped_entry
    li.insert(li.end(), te.begin(), te.end());
    li.push_back(0); li.push_back(0);  // no CtExtensions
    ed.clear();
    if (e.precert) put_opaque24(ed, leaf.data(), leaf.size());  // PrecertChainEntry.pre_certificate
    put_opaque24(ed, chain.data(), chain.size());
}

// TileLeaf of synthetic entry i (static-ct-api data tiles): the same TimestampedEntry with a leaf_index extension, the
// pre_certificate of a precert entry, and the chain as fingerprints
void make_tile_leaf(const ctmr_synth_cfg* cfg, const Issuers& iss, const uint8_t* fps, uint64_t i, std::vector<uint8_t>& leaf,
                    std::vector<uint8_t>& out) {
    const SynthEntry e = synth_entry(cfg, iss, i, leaf, out);
    const uint8_t ext[10] = {0, 8, 0, 0, 5, (uint8_t)(i >> 32), (uint8_t)(i >> 24), (uint8_t)(i >> 16), (uint8_t)(i >> 8), (uint8_t)i};
    out.insert(out.end(), ext, ext + 10);  // CtExtensions: one leaf_index extension
    if (e.precert) put_opaque24(out, leaf.data(), leaf.size());
    out.push_back(0); out.push_back((uint8_t)(32 * e.n_chain));
    for (int m = 0; m < e.n_chain; ++m) out.insert(out.end(), fps + 32ull * e.chain[m], fps + 32ull * e.chain[m] + 32);
}

Issuers make_issuers(const ctmr_synth_cfg* cfg) {
    Issuers iss;
    iss.der.resize(cfg->n_issuers);
    iss.key_hash.resize(cfg->n_issuers);
    for (uint32_t k = 0; k < cfg->n_issuers; ++k) {
        ctmr_synth_issuer_plan ip;
        ctmr_synth_issuer_plan_make(cfg, k, &ip);
        iss.der[k].resize(ip.total);
        ctmr_synth_issuer_write(cfg, &ip, iss.der[k].data());
        Sha256::digest(iss.der[k].data(), iss.der[k].size(), iss.key_hash[k].data());
    }
    return iss;
}

}  // namespace

extern "C" {

/* Bodies {"entries":[{"leaf_input":"..","extra_data":".."},...]} of `page` entries each, back to back, for entries
 * [first, first+n).  Returns the bytes needed; writes text / spans only when text != NULL and cap suffices. */
uint64_t ctmr_synth_raw_pages_host(const struct ctmr_synth_cfg* cfg, uint64_t first, uint64_t n, uint32_t page, uint8_t* text, uint64_t cap,
                                   uint64_t* leaf_off, uint32_t* leaf_len, uint64_t* extra_off, uint32_t* extra_len) {
    if (!cfg || page == 0) return 0;
    const Issuers iss = make_issuers(cfg);
    static const char kOpen[] = "{\"entries\":[", kLeaf[] = "{\"leaf_input\":\"", kExtra[] = "\",\"extra_data\":\"", kEnd[] = "\"}", kClose[] = "]}";
    const uint64_t n_pages = (n + page - 1) / page;
    // pass 1 (threaded): per-page sizes; pass 2: write at the prefix offsets
    const unsigned T = std::max(1u, std::min(std::thread::hardware_concurrency(), 64u));
    std::vector<uint64_t> page_bytes(n_pages + 1, 0);
    auto for_pages = [&](auto&& fn) {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < T; ++t)
            th.emplace_back([&, t] {
                std::vector<uint8_t> leaf, li, ed;
                for (uint64_t p = t; p < n_pages; p += T) fn(p, leaf, li, ed);
            });
        for (auto& x : th) x.join();
    };
    for_pages([&](uint64_t p, std::vector<uint8_t>& leaf, std::vector<uint8_t>& li, std::vector<uint8_t>& ed) {
        uint64_t bytes = sizeof kOpen - 1 + sizeof kClose - 1;
        const uint64_t lo = p * page, hi = std::min<uint64_t>(n, lo + page);
        for (uint64_t j = lo; j < hi; ++j) {
            make_entry(cfg, iss, first + j, leaf, li, ed);
            bytes += sizeof kLeaf - 1 + b64_len(li.size()) + sizeof kExtra - 1 + b64_len(ed.size()) + sizeof kEnd - 1 + (j + 1 < hi ? 1 : 0);
        }
        page_bytes[p + 1] = bytes;
    });
    for (uint64_t p = 0; p < n_pages; ++p) page_bytes[p + 1] += page_bytes[p];
    const uint64_t total = page_bytes[n_pages];
    if (!text || cap < total) return total;
    for_pages([&](uint64_t p, std::vector<uint8_t>& leaf, std::vector<uint8_t>& li, std::vector<uint8_t>& ed) {
        uint8_t* o = text + page_bytes[p];
        auto lit = [&](const char* s, size_t k) { std::memcpy(o, s, k); o += k; };
        lit(kOpen, sizeof kOpen - 1);
        const uint64_t lo = p * page, hi = std::min<uint64_t>(n, lo + page);
        for (uint64_t j = lo; j < hi; ++j) {
            make_entry(cfg, iss, first + j, leaf, li, ed);
            lit(kLeaf, sizeof kLeaf - 1);
            if (leaf_off) { leaf_off[j] = (uint64_t)(o - text); leaf_len[j] = (uint32_t)b64_len(li.size()); }
            o = b64_put(o, li.data(), li.size());
            lit(kExtra, sizeof kExtra - 1);
            if (extra_off) { extra_off[j] = (uint64_t)(o - text); extra_len[j] = (uint32_t)b64_len(ed.size()); }
            o = b64_put(o, ed.data(), ed.size());
            lit(kEnd, sizeof kEnd - 1);
            if (j + 1 < hi) *o++ = ',';
        }
        lit(kClose, sizeof kClose - 1);
    });
    return total;
}

/* static-ct-api data tiles first_tile .. first_tile + n_tiles - 1 of the same entries, back to back (ctmr.h) */
uint64_t ctmr_synth_tiles_host(const struct ctmr_synth_cfg* cfg, uint64_t first_tile, uint64_t n_tiles, const uint8_t* issuer_fps,
                               uint8_t* data, uint64_t cap, uint64_t* tile_off, uint32_t* tile_len) {
    if (!cfg || !issuer_fps || n_tiles == 0) return 0;
    const Issuers iss = make_issuers(cfg);
    const unsigned T = std::max(1u, std::min(std::thread::hardware_concurrency(), 64u));
    std::vector<uint64_t> off(n_tiles + 1, 0);
    auto for_tiles = [&](auto&& fn) {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < T; ++t)
            th.emplace_back([&, t] {
                std::vector<uint8_t> leaf, tl;
                for (uint64_t x = t; x < n_tiles; x += T) fn(x, leaf, tl);
            });
        for (auto& x : th) x.join();
    };
    for_tiles([&](uint64_t x, std::vector<uint8_t>& leaf, std::vector<uint8_t>& tl) {
        uint64_t bytes = 0;
        for (uint64_t j = 0; j < 256; ++j) {
            make_tile_leaf(cfg, iss, issuer_fps, 256 * (first_tile + x) + j, leaf, tl);
            bytes += tl.size();
        }
        off[x + 1] = bytes;
    });
    for (uint64_t x = 0; x < n_tiles; ++x) off[x + 1] += off[x];
    const uint64_t total = off[n_tiles];
    if (!data || cap < total) return total;
    for_tiles([&](uint64_t x, std::vector<uint8_t>& leaf, std::vector<uint8_t>& tl) {
        uint8_t* o = data + off[x];
        for (uint64_t j = 0; j < 256; ++j) {
            make_tile_leaf(cfg, iss, issuer_fps, 256 * (first_tile + x) + j, leaf, tl);
            std::memcpy(o, tl.data(), tl.size());
            o += tl.size();
        }
        if (tile_off) tile_off[x] = off[x];
        if (tile_len) tile_len[x] = (uint32_t)(off[x + 1] - off[x]);
    });
    return total;
}

}  // extern "C"
