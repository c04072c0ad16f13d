// ctmr_frontend.cu -- kernels of the CT wire-format front end (include/ctmr_frontend.h, SURVEY §8(f)-2).
//
//   K_fe_sizes   thread per string   decoded length from the character count and the '=' padding
//   (cub scan)                       16-byte aligned placement of every decoded string in one HBM arena
//   K_fe_decode  warp per string     base64 -> bytes, 16 characters (12 bytes) per lane per step
//   K_fe_frame   thread per entry    MerkleTreeLeaf + CertificateChain / PrecertChainEntry framing
//   K_fe_tbs     thread per entry    precert entries: ParseTBSCertificate of the leaf's TBSCertificate
//   K_fe_issuer  warp per entry      Chain[0] bytes -> dense issuer index (hash, probe, full compare)
//   K_fe_finish  thread per entry    "failed to parse certificate in MerkleTreeLeaf" for x509 entries
//
// All of it is byte shuffling bound by HBM and the LSU, nothing here is GEMM shaped.  The decoded arena is
// what K_map then streams (explicit record lengths, ctmr_dev_batch.lens): leaves are never copied again.
#include <cub/device/device_scan.cuh>

#include "ctmr_common.cuh"

namespace ctmr {

namespace {

// ASCII -> 6-bit value, 0xFF = not in the standard alphabet ('=' included: padding is handled by position).
// One 256-byte table per CTA.  A per-lane replicated table (32 KB, conflict-free look-ups) was measured before
// the port and rejected as slower: the kernel is bound by loads in flight, and the larger table costs two
// resident CTAs per SM.
__device__ __forceinline__ void fill_b64_lut(uint8_t* lut) {
    for (uint32_t c = threadIdx.x; c < 256u; c += blockDim.x) {
        uint32_t v = 0xFFu;
        if (c >= 'A' && c <= 'Z') v = c - 'A';
        else if (c >= 'a' && c <= 'z') v = c - 'a' + 26u;
        else if (c >= '0' && c <= '9') v = c - '0' + 52u;
        else if (c == '+') v = 62u;
        else if (c == '/') v = 63u;
        lut[c] = (uint8_t)v;
    }
}

__global__ void __launch_bounds__(256) fe_sizes_kernel(FeParams p) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s > 2 * p.n) return;
    if (s == 2 * p.n) {
        p.pad_size[s] = 0;
        return;
    }
    const uint64_t e = s >> 1;
    const uint64_t off = (s & 1) ? p.extra_off[e] : p.leaf_off[e];
    const uint32_t L = (s & 1) ? p.extra_len[e] : p.leaf_len[e];
    uint32_t dec = 0;
    uint8_t bad = 0;
    if (off > p.text_bytes || L > p.text_bytes - off || (L & 3u)) {
        bad = 1;  // base64.StdEncoding wants whole, padded quanta
    } else if (L) {
        const uint32_t pad = (p.text[off + L - 1] == '=') + ((p.text[off + L - 1] == '=') & (p.text[off + L - 2] == '='));
        dec = L / 4u * 3u - pad;
    }
    p.dec_len[s] = dec;
    p.str_bad[s] = bad;
    p.pad_size[s] = ((uint64_t)dec + 15u) & ~15ull;
}

// Four characters held little-endian in `w` -> 24 decoded bits as bytes b0 | b1<<8 | b2<<16; *bad |= 0x80 bits on junk.
__device__ __forceinline__ uint32_t dec_quad(const uint8_t* lut, uint32_t w, uint32_t& bad) {
    const uint32_t v0 = lut[w & 0xffu], v1 = lut[(w >> 8) & 0xffu], v2 = lut[(w >> 16) & 0xffu], v3 = lut[w >> 24];
    bad |= v0 | v1 | v2 | v3;
    const uint32_t bits = (v0 << 18) | ((v1 & 63u) << 12) | ((v2 & 63u) << 6) | (v3 & 63u);  // b0 b1 b2, big-endian in 24 bits
    return __byte_perm(bits, 0u, 0x4012);  // -> b0 at the low byte
}

__global__ void __launch_bounds__(256) fe_decode_kernel(FeParams p) {
    __shared__ uint8_t lut[256];
    fill_b64_lut(lut);
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t s = warp0; s < 2 * p.n; s += nwarps) {
        if (p.str_bad[s]) continue;
        const uint64_t e = s >> 1;
        const uint64_t off = (s & 1) ? p.extra_off[e] : p.leaf_off[e];
        const uint32_t L = (s & 1) ? p.extra_len[e] : p.leaf_len[e];
        const uint32_t dec = p.dec_len[s];
        const uint32_t padded = (dec + 15u) & ~15u;
        const uint32_t npad = L / 4u * 3u - dec;  // '=' characters at the very end: 0, 1 or 2
        const uint8_t* src = p.text + off;
        const uint64_t a = reinterpret_cast<uint64_t>(src);
        const uint32_t* aw = reinterpret_cast<const uint32_t*>(a & ~3ull);  // the text buffer has slack at both ends
        const uint32_t sh = (uint32_t)(a & 3u) * 8u;
        uint32_t* dst = reinterpret_cast<uint32_t*>(p.decoded + p.dec_off[s]);
        uint32_t bad = 0;
        const uint32_t ngroups = (L + 15u) >> 4;
        for (uint32_t g = lane; g < ngroups; g += 32u) {
            uint32_t x[4] = {0, 0, 0, 0}, t[5];
#pragma unroll
            for (uint32_t q = 0; q < 5u; ++q) t[q] = __ldg(aw + 4u * g + q);  // five independent loads (the buffer has slack past the text)
#pragma unroll
            for (uint32_t q = 0; q < 4u; ++q) {
                const uint32_t c0 = 16u * g + 4u * q;  // first character of this quantum
                if (c0 < L) {
                    uint32_t w = __funnelshift_r(t[q], t[q + 1], sh);
                    if (c0 + 4u == L && npad) w = npad == 2u ? (w & 0x0000ffffu) | 0x41410000u : (w & 0x00ffffffu) | 0x41000000u;
                    x[q] = dec_quad(lut, w, bad);
                }
            }
            const uint32_t o[3] = {x[0] | (x[1] << 24), (x[1] >> 8) | (x[2] << 16), (x[2] >> 16) | (x[3] << 8)};
#pragma unroll
            for (uint32_t k = 0; k < 3u; ++k)
                if (12u * g + 4u * k < padded) dst[3u * g + k] = o[k];
        }
        if (__any_sync(0xffffffffu, (bad & 0x80u) != 0u) && lane == 0) p.str_bad[s] = 1;
    }
}

// big-endian fields of the TLS presentation language (RFC 5246 §4)
__device__ __forceinline__ uint32_t be24(const uint8_t* d) { return ((uint32_t)d[0] << 16) | ((uint32_t)d[1] << 8) | d[2]; }

// opaque ASN.1Cert<1..2^24-1> entries filling d[q..end) exactly; reports the first one
__device__ __forceinline__ bool walk_chain(const uint8_t* d, uint32_t q, uint32_t end, uint32_t& first_off, uint32_t& first_len) {
    first_off = first_len = 0;
    bool first = true;
    while (q < end) {
        if (q + 3u > end) return false;
        const uint32_t l = be24(d + q);
        if (l == 0u || l > end - q - 3u) return false;
        if (first) {
            first_off = q + 3u;
            first_len = l;
            first = false;
        }
        q += 3u + l;
    }
    return true;
}

__global__ void __launch_bounds__(256) fe_frame_kernel(FeParams p) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= p.n) return;
    uint32_t status = CTMR_FE_OK, etype = CTMR_ENTRY_OTHER, leaf_src = 0, leaf_rel = 0, leaf_len = 0;
    uint32_t chain_rel = 0, chain_len = 0, tbs_rel = 0, tbs_len = 0;
    uint64_t ts = 0;
    const uint8_t* li = p.decoded + p.dec_off[2 * e];
    const uint8_t* ed = p.decoded + p.dec_off[2 * e + 1];
    const uint32_t nl = p.dec_len[2 * e], ne = p.dec_len[2 * e + 1];
    if (p.str_bad[2 * e] || p.str_bad[2 * e + 1]) {
        status = CTMR_FE_BAD_BASE64;
    } else if (nl < 12u || li[1] != 0u) {  // Version(1) MerkleLeafType(1)=timestamped_entry uint64 LogEntryType(2)
        status = CTMR_FE_BAD_LEAF;
    } else {
        for (int k = 0; k < 8; ++k) ts = (ts << 8) | li[2 + k];
        const uint32_t t = ((uint32_t)li[10] << 8) | li[11];
        uint32_t q = 12;
        if (t == 0u) {  // ASN.1Cert
            etype = CTMR_ENTRY_X509;
        } else if (t == 1u) {  // PreCert: opaque issuer_key_hash[32]; TBSCertificate
            etype = CTMR_ENTRY_PRECERT;
            q += 32u;
        } else {
            status = CTMR_FE_UNKNOWN_TYPE;
        }
        if (status == CTMR_FE_OK) {
            uint32_t l = 0;
            if (q + 3u > nl || (l = be24(li + q)) == 0u || l > nl - q - 3u) {
                status = CTMR_FE_BAD_LEAF;
            } else {
                const uint32_t body = q + 3u;
                q = body + l;
                // CtExtensions extensions<0..2^16-1>, then nothing
                if (q + 2u > nl || q + 2u + (((uint32_t)li[q] << 8) | li[q + 1]) != nl) {
                    status = CTMR_FE_BAD_LEAF;
                } else if (etype == CTMR_ENTRY_X509) {
                    leaf_src = 0;
                    leaf_rel = body;
                    leaf_len = l;
                } else {
                    tbs_rel = body;
                    tbs_len = l;
                }
            }
        }
        if (status == CTMR_FE_OK) {
            uint32_t q2 = 0;
            bool ok = true;
            if (etype == CTMR_ENTRY_PRECERT) {  // PrecertChainEntry: ASN.1Cert pre_certificate; ASN.1Cert chain<0..2^24-1>
                uint32_t l = 0;
                if (ne < 3u || (l = be24(ed)) == 0u || l > ne - 3u) {
                    ok = false;
                } else {
                    leaf_src = 1;
                    leaf_rel = 3;
                    leaf_len = l;
                    q2 = 3u + l;
                }
            }
            if (ok) {
                if (q2 + 3u > ne || q2 + 3u + be24(ed + q2) != ne) ok = false;
                else ok = walk_chain(ed, q2 + 3u, ne, chain_rel, chain_len);
            }
            if (!ok) {
                status = CTMR_FE_BAD_EXTRA;
                leaf_len = 0;
            }
        }
    }
    if (status != CTMR_FE_OK) leaf_len = chain_len = tbs_len = 0;
    p.entry_status[e] = (uint8_t)status;
    p.entry_type[e] = (uint8_t)etype;
    p.timestamp[e] = ts;
    p.leaf_src[e] = (uint8_t)leaf_src;
    p.leaf_rel[e] = leaf_rel;
    p.leaf_len_out[e] = leaf_len;
    p.leaf_abs[e] = p.dec_off[2 * e + leaf_src] + leaf_rel;
    p.chain_abs[e] = p.dec_off[2 * e + 1] + chain_rel;
    p.chain_len[e] = chain_len;
    p.tbs_abs[e] = p.dec_off[2 * e] + tbs_rel;
    p.tbs_len[e] = tbs_len;
    p.issuer_idx[e] = chain_len ? CTMR_ISSUER_UNRESOLVED : CTMR_ISSUER_NONE;
}

// MerkleTreeLeaf.Precertificate() = x509.ParseTBSCertificate(tbs): trailing data is an error
__global__ void __launch_bounds__(128) fe_tbs_kernel(FeParams p) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= p.n || p.entry_status[e] != CTMR_FE_OK || p.entry_type[e] != CTMR_ENTRY_PRECERT) return;
    ParsedCert pc;
    uint32_t end = 0;
    const uint32_t len = p.tbs_len[e];
    if (parse_tbs(p.decoded + p.tbs_abs[e], 0, len, pc, end) && end == len) return;
    p.entry_status[e] = CTMR_FE_BAD_CERT;
    p.leaf_len_out[e] = 0;
    p.chain_len[e] = 0;
    p.issuer_idx[e] = CTMR_ISSUER_NONE;
}

// ---- Chain[0] -> dense issuer index --------------------------------------------------------------
// 32-bit little-endian word at byte offset x of an arbitrarily aligned byte string
__device__ __forceinline__ uint32_t ld_u32_unaligned(const uint8_t* base, uint32_t x) {
    const uint64_t a = reinterpret_cast<uint64_t>(base) + x;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~3ull);
    return __funnelshift_r(__ldg(w), __ldg(w + 1), (uint32_t)(a & 3u) * 8u);
}

__global__ void __launch_bounds__(256) fe_issuer_kernel(FeParams p, IssuerCertTable tab, uint64_t* pending, uint64_t pending_mask,
                                                        uint32_t* unknown_list, uint32_t unknown_cap, unsigned int* unknown_count) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t e = warp0; e < p.n; e += nwarps) {
        if (p.issuer_idx[e] != CTMR_ISSUER_UNRESOLVED) continue;
        const uint8_t* d = p.decoded + p.chain_abs[e];
        const uint32_t len = p.chain_len[e];
        // issuer_cert_hash (ctmr_kernels.cuh): order-independent sum over 8-byte words -> any lane split works
        const uint32_t nw = (len + 7u) >> 3;
        uint64_t acc = 0;
        for (uint32_t i = lane; i < nw; i += 32u) {
            uint32_t lo = ld_u32_unaligned(d, 8u * i), hi = 8u * i + 4u < len ? ld_u32_unaligned(d, 8u * i + 4u) : 0u;
            const uint32_t rem = len - 8u * i;  // bytes of this word that belong to the certificate
            if (rem < 4u) lo &= (1u << (8u * rem)) - 1u;
            else if (rem < 8u && rem > 4u) hi &= (1u << (8u * (rem - 4u))) - 1u;
            else if (rem == 4u) hi = 0u;
            acc += issuer_cert_word(((uint64_t)hi << 32) | lo, i);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        const uint64_t h = issuer_cert_finish(acc, len);
        uint32_t found = CTMR_ISSUER_UNRESOLVED;
        for (uint64_t slot = h & tab.mask, probes = 0; probes <= tab.mask; slot = (slot + 1) & tab.mask, ++probes) {
            const IssuerCertSlot sl = tab.slots[slot];
            if (sl.h == 0) break;
            if (sl.h != h || sl.len != len) continue;
            const uint32_t* ref = reinterpret_cast<const uint32_t*>(tab.arena + sl.arena_off);  // 16-byte aligned, zero padded
            bool diff = false;
            for (uint32_t i = lane; 4u * i < len; i += 32u) {
                uint32_t v = ld_u32_unaligned(d, 4u * i);
                const uint32_t rem = len - 4u * i;
                if (rem < 4u) v &= (1u << (8u * rem)) - 1u;
                diff |= v != __ldg(ref + i);
            }
            if (!__any_sync(0xffffffffu, diff)) {
                found = sl.idx;
                break;
            }
        }
        if (lane == 0) {
            if (found != CTMR_ISSUER_UNRESOLVED) {
                p.issuer_idx[e] = found;
            } else {  // one representative per distinct hash goes back to the host for registration
                for (uint64_t s2 = h & pending_mask, probes = 0; probes <= pending_mask; s2 = (s2 + 1) & pending_mask, ++probes) {
                    const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(pending + s2), 0ull, (unsigned long long)h);
                    if (prev == 0ull) {
                        const unsigned int k = atomicAdd(unknown_count, 1u);
                        if (k < unknown_cap) unknown_list[k] = (uint32_t)e;
                        break;
                    }
                    if (prev == h) break;
                }
            }
        }
    }
}

// x509 entries whose leaf certificate has a fatal parse error never reach the channel (ct-fetch.go:453-460)
__global__ void __launch_bounds__(256) fe_finish_kernel(FeParams p, const uint8_t* __restrict__ status) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= p.n) return;
    if (p.entry_status[e] == CTMR_FE_OK && p.entry_type[e] == CTMR_ENTRY_X509 && status[e] == CTMR_ST_PARSE_ERR)
        p.entry_status[e] = CTMR_FE_BAD_CERT;
}

unsigned grid_for_warps(uint64_t items, int sm_count) {
    const uint64_t want = (items + 7) / 8;  // 8 warps per 256-thread CTA
    const uint64_t cap = (uint64_t)sm_count * 16;
    return (unsigned)(want < cap ? (want ? want : 1) : cap);
}

}  // namespace

size_t fe_scan_temp_bytes(uint64_t n_items) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n_items);
    return bytes;
}

cudaError_t launch_fe_decode(const FeParams& p, void* scan_temp, size_t scan_temp_bytes, int sm_count, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    const uint64_t items = 2 * p.n + 1;
    fe_sizes_kernel<<<(unsigned)((items + 255) / 256), 256, 0, s>>>(p);
    cudaError_t err = cub::DeviceScan::ExclusiveSum(scan_temp, scan_temp_bytes, p.pad_size, p.dec_off, (int)items, s);
    if (err != cudaSuccess) return err;
    fe_decode_kernel<<<grid_for_warps(2 * p.n, sm_count), 256, 0, s>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_fe_frame(const FeParams& p, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    fe_frame_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, s>>>(p);
    return launch_fe_tbs(p, s);
}

cudaError_t launch_fe_tbs(const FeParams& p, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    fe_tbs_kernel<<<(unsigned)((p.n + 127) / 128), 128, 0, s>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_fe_issuer(const FeParams& p, const IssuerCertTable& tab, uint64_t* pending, uint64_t pending_mask,
                             uint32_t* unknown_list, uint32_t unknown_cap, unsigned int* unknown_count, int sm_count, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    fe_issuer_kernel<<<grid_for_warps(p.n, sm_count), 256, 0, s>>>(p, tab, pending, pending_mask, unknown_list, unknown_cap, unknown_count);
    return cudaGetLastError();
}

cudaError_t launch_fe_finish(const FeParams& p, const uint8_t* status, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    fe_finish_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, s>>>(p, status);
    return cudaGetLastError();
}

}  // namespace ctmr

// ================================================================================================
// PEM of selected certificates (SURVEY §8(f)-3): pem.EncodeToMemory(&pem.Block{Type: "CERTIFICATE",
// Bytes: cert.Raw}) as built in FilesystemDatabase.Store (storage/filesystemdatabase.go:171-175,197-198),
// i.e. "-----BEGIN CERTIFICATE-----\n", base64.StdEncoding in lines of 64 characters each ended by '\n',
// "-----END CERTIFICATE-----\n".  Only NEW certificates are stored, so only they are encoded.
// ================================================================================================
namespace ctmr {
namespace {

constexpr uint32_t kPemHead = 28, kPemTail = 26;  // the two boundary lines, newline included

__device__ __forceinline__ uint32_t pem_size(uint32_t der_len) {
    const uint32_t b64 = (der_len + 2u) / 3u * 4u;
    return kPemHead + b64 + (b64 + 63u) / 64u + kPemTail;
}

__device__ __forceinline__ uint32_t b64_char(uint32_t v) {  // 6 bits -> ASCII of the standard alphabet, branch-free
    return v + 65u + (v >= 26u ? 6u : 0u) - (v >= 52u ? 75u : 0u) - (v >= 62u ? 15u : 0u) + (v >= 63u ? 3u : 0u);
}

__global__ void __launch_bounds__(256) pem_sizes_kernel(const uint64_t* __restrict__ offsets, const uint32_t* __restrict__ lens,
                                                        const uint8_t* __restrict__ select, uint64_t n, uint64_t* __restrict__ sizes) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e > n) return;
    uint64_t sz = 0;
    if (e < n && select[e]) {
        const uint64_t len = lens ? lens[e] : offsets[e + 1] - offsets[e];
        sz = pem_size((uint32_t)len);
    }
    sizes[e] = sz;
}

__global__ void __launch_bounds__(256) pem_encode_kernel(const uint8_t* __restrict__ blob, const uint64_t* __restrict__ offsets,
                                                         const uint32_t* __restrict__ lens, const uint8_t* __restrict__ select, uint64_t n,
                                                         const uint64_t* __restrict__ pem_off, uint8_t* __restrict__ pem, uint64_t cap,
                                                         int* __restrict__ error_flag) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t e = warp0; e < n; e += nwarps) {
        if (!select[e]) continue;
        const uint64_t at = pem_off[e];
        const uint32_t L = lens ? lens[e] : (uint32_t)(offsets[e + 1] - offsets[e]);
        const uint32_t total = pem_size(L);
        if (at + total > cap) {  // caller's buffer too small: nothing of this certificate is written
            if (lane == 0) atomicExch(error_flag, CTMR_E_BATCH_TOO_LARGE);
            continue;
        }
        const uint8_t* d = blob + offsets[e];
        uint8_t* o = pem + at;
        const char* head = "-----BEGIN CERTIFICATE-----\n";
        const char* tail = "-----END CERTIFICATE-----\n";
        if (lane < kPemHead) o[lane] = (uint8_t)head[lane];
        if (lane < kPemTail) o[total - kPemTail + lane] = (uint8_t)tail[lane];
        uint8_t* body = o + kPemHead;
        const uint32_t ngroups = (L + 2u) / 3u;  // 3 bytes -> 4 characters; 16 groups per line
        for (uint32_t g = lane; g < ngroups; g += 32u) {
            const uint32_t i = 3u * g, rem = L - i;
            const uint32_t b0 = d[i], b1 = rem > 1u ? d[i + 1] : 0u, b2 = rem > 2u ? d[i + 2] : 0u;
            const uint32_t w = (b0 << 16) | (b1 << 8) | b2;
            uint8_t* q = body + 4u * g + (g >> 4);  // one '\n' behind every 16 complete groups
            q[0] = (uint8_t)b64_char(w >> 18);
            q[1] = (uint8_t)b64_char((w >> 12) & 63u);
            q[2] = rem > 1u ? (uint8_t)b64_char((w >> 6) & 63u) : (uint8_t)'=';
            q[3] = rem > 2u ? (uint8_t)b64_char(w & 63u) : (uint8_t)'=';
            if ((g & 15u) == 15u || g + 1u == ngroups) q[4] = (uint8_t)'\n';
        }
    }
}

}  // namespace

size_t pem_scan_temp_bytes(uint64_t n_items) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n_items);
    return bytes;
}

// sizes -> pem_off[0..n] (exclusive scan, pem_off[n] = total) -> text.  `sizes` is scratch of n+1 words.
cudaError_t launch_pem_encode(const uint8_t* blob, const uint64_t* offsets, const uint32_t* lens, const uint8_t* select, uint64_t n,
                              uint64_t* sizes, void* scan_temp, size_t scan_temp_bytes, uint64_t* pem_off, uint8_t* pem, uint64_t cap,
                              int* error_flag, int sm_count, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    pem_sizes_kernel<<<(unsigned)((n + 256) / 256), 256, 0, s>>>(offsets, lens, select, n, sizes);
    cudaError_t err = cub::DeviceScan::ExclusiveSum(scan_temp, scan_temp_bytes, sizes, pem_off, (int)(n + 1), s);
    if (err != cudaSuccess) return err;
    pem_encode_kernel<<<grid_for_warps(n, sm_count), 256, 0, s>>>(blob, offsets, lens, select, n, pem_off, pem, cap, error_flag);
    return cudaGetLastError();
}

}  // namespace ctmr
