// ctmr_tiles.cu -- kernels that read static-ct-api data tiles (ctmr_process_tiles, include/ctmr_frontend.h).
//
//   K_tile_split      thread per tile    TileLeaf boundaries from the length fields only; a tile that does not split
//                                        into exactly `width` TileLeafs with no trailing bytes is bad as a whole
//   K_tile_frame      thread per entry   timestamp, type, leaf / TBS spans, leaf_index check, Chain[0] fingerprint
//   (fe_tbs)                             precert entries: ParseTBSCertificate, the get-entries rule unchanged
//   K_tile_issuer     thread per entry   fingerprint -> dense issuer index (probe, full 32-byte compare)
//   K_tile_leaf_hash  thread per entry   RFC 6962 §2.1 leaf hash, when the caller asks for it
//
// The leaves stay where the upload put them: K_map reads them in place through explicit record lengths.
#include "ctmr_common.cuh"

namespace ctmr {

namespace {

__device__ __forceinline__ uint32_t rd16(const uint8_t* d) { return ((uint32_t)d[0] << 8) | d[1]; }
__device__ __forceinline__ uint32_t rd24(const uint8_t* d) { return ((uint32_t)d[0] << 16) | ((uint32_t)d[1] << 8) | d[2]; }

// One walker per tile: finding where entry j+1 starts needs entry j's lengths, so the walk is serial within a tile.
__global__ void __launch_bounds__(128) tile_split_kernel(TileParams p) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= p.n_tiles) return;
    const TileDesc td = p.tiles[t];
    const uint8_t* d = p.data + td.staged_off;
    const uint32_t L = td.len;
    uint32_t q = 0;
    bool ok = true;
    for (uint32_t j = 0; j < td.width && ok; ++j) {
        const uint32_t start = q;
        uint32_t type = 0, l = 0;
        // TimestampedEntry: uint64 timestamp, uint16 entry_type, ASN.1Cert | PreCert, CtExtensions
        if (q + 10u > L) { ok = false; break; }
        type = rd16(d + q + 8);
        q += 10u;
        if (type == 1u) q += 32u;
        else if (type != 0u) { ok = false; break; }
        if (q + 3u > L || (l = rd24(d + q)) == 0u || l > L - q - 3u) { ok = false; break; }
        q += 3u + l;
        if (q + 2u > L || (l = rd16(d + q)) > L - q - 2u) { ok = false; break; }
        q += 2u + l;
        if (type == 1u) {  // ASN.1Cert pre_certificate
            if (q + 3u > L || (l = rd24(d + q)) == 0u || l > L - q - 3u) { ok = false; break; }
            q += 3u + l;
        }
        // Fingerprint certificate_chain<0..2^16-1>
        if (q + 2u > L || ((l = rd16(d + q)) & 31u) || l > L - q - 2u) { ok = false; break; }
        q += 2u + l;
        p.entry_off[td.first + j] = td.staged_off + start;
    }
    p.tile_bad[t] = !(ok && q == L);
}

__global__ void __launch_bounds__(256) tile_frame_kernel(TileParams p) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= p.n) return;
    uint32_t lo = 0, hi = p.n_tiles;  // the tile holding entry e: last tile whose first entry is <= e
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (p.tiles[mid].first <= e) lo = mid;
        else hi = mid;
    }
    const uint32_t t = lo;
    const TileDesc td = p.tiles[t];
    uint32_t status = CTMR_FE_OK, etype = CTMR_ENTRY_OTHER, leaf_len = 0, chain_len = 0, tbs_len = 0, te = 0;
    uint64_t ts = 0, leaf_abs = 0, chain_abs = 0, tbs_abs = 0, index = 0, data_off = 0;
    if (p.tile_bad[t]) {
        status = CTMR_FE_BAD_TILE;
    } else {  // the split has checked every length below
        const uint64_t at = p.entry_off[e];
        const uint8_t* d = p.data + at;
        for (int k = 0; k < 8; ++k) ts = (ts << 8) | d[k];
        etype = rd16(d + 8);
        uint32_t q = 10u + (etype == CTMR_ENTRY_PRECERT ? 32u : 0u);
        const uint32_t body = q + 3u, l = rd24(d + q);
        q = body + l;
        const uint32_t ext = q + 2u, ext_end = ext + rd16(d + q);
        te = ext_end;
        // CtExtensions: { uint8 extension_type; opaque extension_data<0..2^16-1> } list; exactly one leaf_index (type 0)
        uint32_t n_idx = 0, idx_len = 0;
        bool list_ok = true;
        for (uint32_t r = ext; r < ext_end;) {
            if (r + 3u > ext_end) { list_ok = false; break; }
            const uint32_t el = rd16(d + r + 1);
            if (el > ext_end - r - 3u) { list_ok = false; break; }
            if (d[r] == 0u) {
                ++n_idx;
                idx_len = el;
                if (el == 5u) {
                    index = 0;
                    for (int k = 0; k < 5; ++k) index = (index << 8) | d[r + 3u + k];
                }
            }
            r += 3u + el;
        }
        if (!(list_ok && n_idx == 1u && idx_len == 5u)) index = 0;
        q = ext_end;
        uint32_t leaf_at = body;
        leaf_len = l;
        if (etype == CTMR_ENTRY_PRECERT) {
            tbs_abs = at + body;
            tbs_len = l;
            leaf_at = q + 3u;
            leaf_len = rd24(d + q);
            q = leaf_at + leaf_len;
        }
        const uint32_t c = rd16(d + q);
        chain_abs = at + q + 2u;
        chain_len = c ? 32u : 0u;
        leaf_abs = at + leaf_at;
        data_off = td.data_off + (leaf_abs - td.staged_off);
        const uint64_t want = 256ull * td.index + (e - td.first);
        if (!(list_ok && n_idx == 1u && idx_len == 5u && index == want)) {
            status = CTMR_FE_BAD_INDEX;
            leaf_len = chain_len = tbs_len = 0;
            data_off = 0;
        }
    }
    p.entry_tile[e] = t;
    p.te_len[e] = te;
    p.leaf_index[e] = index;
    p.leaf_data_off[e] = data_off;
    p.fe.entry_status[e] = (uint8_t)status;
    p.fe.entry_type[e] = (uint8_t)etype;
    p.fe.timestamp[e] = ts;
    p.fe.leaf_abs[e] = leaf_abs;
    p.fe.leaf_len_out[e] = leaf_len;
    p.fe.chain_abs[e] = chain_abs;
    p.fe.chain_len[e] = chain_len;
    p.fe.tbs_abs[e] = tbs_abs;
    p.fe.tbs_len[e] = tbs_len;
    p.fe.issuer_idx[e] = chain_len ? CTMR_ISSUER_UNRESOLVED : CTMR_ISSUER_NONE;
}

// 8 words of a 32-byte fingerprint at any alignment, bytes in order (little-endian words, as FpSlot.w holds them)
__device__ __forceinline__ void load_fp(const uint8_t* d, uint32_t (&w)[8]) {
#pragma unroll
    for (int k = 0; k < 8; ++k)
        w[k] = (uint32_t)d[4 * k] | ((uint32_t)d[4 * k + 1] << 8) | ((uint32_t)d[4 * k + 2] << 16) | ((uint32_t)d[4 * k + 3] << 24);
}

__global__ void __launch_bounds__(256) tile_issuer_kernel(TileParams p, FpTable tab) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= p.n) return;
    if (p.fe.leaf_len_out[e] == 0u) p.leaf_data_off[e] = 0;  // fe_tbs dropped the entry
    if (p.fe.issuer_idx[e] != CTMR_ISSUER_UNRESOLVED) return;
    uint32_t w[8];
    load_fp(p.data + p.fe.chain_abs[e], w);
    const uint64_t h = ((uint64_t)w[1] << 32) | w[0];
    for (uint64_t slot = h & tab.mask, probes = 0; probes <= tab.mask; slot = (slot + 1) & tab.mask, ++probes) {
        const FpSlot& sl = tab.slots[slot];
        if (!sl.used) break;
        bool same = true;
#pragma unroll
        for (int k = 0; k < 8; ++k) same &= sl.w[k] == w[k];
        if (same) {
            p.fe.issuer_idx[e] = sl.idx;
            return;
        }
    }
    atomicMin(p.first_stop, p.entry_tile[e]);  // nothing is resolved on a guess: the host stops before this tile
}

__global__ void __launch_bounds__(128) tile_leaf_hash_kernel(TileParams p) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= p.n) return;
    uint32_t out[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (p.fe.entry_status[e] != CTMR_FE_BAD_TILE) {
        // SHA-256(0x00 leaf prefix || 0x00 v1 || 0x00 timestamped_entry || TimestampedEntry)
        const uint8_t* m = p.data + p.entry_off[e];
        const uint32_t len = 3u + p.te_len[e];
        Sha256State s;
        s.init();
        const uint32_t nb = (len + 9u + 63u) / 64u;
        for (uint32_t b = 0; b < nb; ++b) {
            uint32_t w[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const uint32_t q = b * 64u + i * 4u;
                uint32_t v = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t x = q + j;
                    v = (v << 8) | (x >= 3u && x < len ? (uint32_t)m[x - 3u] : 0u);
                }
                w[i] = sha256_pad_word(v, q, len);
            }
            if (b == nb - 1u) { w[14] = 0; w[15] = len * 8u; }
            sha256_compress_rolled(s, w, 1u);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) out[i] = s.h[i];
    }
    uint8_t* o = p.leaf_hash + 32 * e;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        o[4 * i] = (uint8_t)(out[i] >> 24); o[4 * i + 1] = (uint8_t)(out[i] >> 16);
        o[4 * i + 2] = (uint8_t)(out[i] >> 8); o[4 * i + 3] = (uint8_t)out[i];
    }
}

// SHA-256 of each registered chain certificate: the fingerprint a tile names it by
__global__ void __launch_bounds__(64) fingerprint_kernel(const uint8_t* __restrict__ blob, const uint64_t* __restrict__ offsets, uint32_t n,
                                                         uint8_t* __restrict__ fps) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    uint32_t h[8];
    sha256_global(blob + offsets[k], (uint32_t)(offsets[k + 1] - offsets[k]), h);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        fps[32 * k + 4 * i] = (uint8_t)(h[i] >> 24); fps[32 * k + 4 * i + 1] = (uint8_t)(h[i] >> 16);
        fps[32 * k + 4 * i + 2] = (uint8_t)(h[i] >> 8); fps[32 * k + 4 * i + 3] = (uint8_t)h[i];
    }
}

}  // namespace

cudaError_t launch_tile_split(const TileParams& p, cudaStream_t s) {
    if (p.n_tiles == 0) return cudaSuccess;
    tile_split_kernel<<<(p.n_tiles + 127) / 128, 128, 0, s>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_tile_frame(const TileParams& p, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    tile_frame_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, s>>>(p);
    return launch_fe_tbs(p.fe, s);
}

cudaError_t launch_tile_issuer(const TileParams& p, const FpTable& tab, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    tile_issuer_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, s>>>(p, tab);
    return cudaGetLastError();
}

cudaError_t launch_tile_leaf_hash(const TileParams& p, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    tile_leaf_hash_kernel<<<(unsigned)((p.n + 127) / 128), 128, 0, s>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_fingerprints(const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint8_t* fps, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    fingerprint_kernel<<<(n + 63) / 64, 64, 0, s>>>(blob, offsets, n, fps);
    return cudaGetLastError();
}

}  // namespace ctmr
