// ctmr_merkle.cu -- the log's Merkle tree (RFC 6962 §2.1) over the entries of ctmr_process_raw_tree /
// ctmr_process_tiles_tree (include/ctmr_frontend.h).
//
//   K_raw_leaf_hash   thread per entry    SHA-256(0x00 || decoded leaf_input), read from the decoded arena
//   (tile_leaf_hash)                      tiles: the leaf hashes of ctmr_tiles.cu, unchanged
//   K_tree_missing    thread per entry    lowest log position of the chunk without a leaf (bad base64, bad tile)
//   K_tree_level      thread per parent   one level of the chunk's range: parents of the pairs inside it, the left edge
//                                         node as the first left child, the last node as the new edge node
//   K_tree_commit     one thread          the tree's new size
//   K_tree_root       one thread          the root from the edge
//
// The tree is held as its right edge (ctmr_tree): for every bit k of size, the root of the complete subtree of 2^k leaves
// ending at the highest multiple of 2^(k+1) at or below size.  Folding leaves [a, b) in: at level l the chunk covers node
// positions [a_l, b_l) = [a >> l, b >> l); pairs (2p, 2p+1) inside it make the parents [a_l >> 1, b_l >> 1); an odd a_l
// takes edge[l] as the left child of the first parent; an odd b_l leaves node b_l - 1 as the new edge[l].  Once the range
// is empty the higher rows keep what they hold.  A chunk of n leaves costs about n node hashes of two compressions each
// and one launch per level.
#include "ctmr_common.cuh"

namespace ctmr {

namespace {

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0u, 0x0123); }

// a 32-byte hash as 8 big-endian words; rows are 8-byte aligned (ctmr_tree.edge is)
__device__ __forceinline__ void load_row(const uint8_t* row, uint32_t (&w)[8]) {
    const uint2* p = reinterpret_cast<const uint2*>(row);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint2 v = p[i];
        w[2 * i] = bswap32(v.x);
        w[2 * i + 1] = bswap32(v.y);
    }
}
__device__ __forceinline__ void store_row(uint8_t* row, const uint32_t (&w)[8]) {
    uint2* p = reinterpret_cast<uint2*>(row);
#pragma unroll
    for (int i = 0; i < 4; ++i) p[i] = make_uint2(bswap32(w[2 * i]), bswap32(w[2 * i + 1]));
}

// SHA-256(0x01 || l || r): 65 bytes, two blocks; the second holds r's last byte and the padding of a 520-bit message
__device__ __forceinline__ void node_hash(const uint32_t (&l)[8], const uint32_t (&r)[8], uint32_t (&out)[8]) {
    Sha256State s;
    s.init();
    uint32_t w[16];
    w[0] = 0x01000000u | (l[0] >> 8);
#pragma unroll
    for (int j = 1; j < 8; ++j) w[j] = (l[j - 1] << 24) | (l[j] >> 8);
    w[8] = (l[7] << 24) | (r[0] >> 8);
#pragma unroll
    for (int j = 9; j < 16; ++j) w[j] = (r[j - 9] << 24) | (r[j - 8] >> 8);
    sha256_compress_rolled(s, w, 1u);
    w[0] = (r[7] << 24) | 0x00800000u;
#pragma unroll
    for (int j = 1; j < 15; ++j) w[j] = 0;
    w[15] = 65u * 8u;
    sha256_compress_rolled(s, w, 1u);
#pragma unroll
    for (int i = 0; i < 8; ++i) out[i] = s.h[i];
}

// Decoded strings sit 16-byte aligned in the arena, so the one-byte prefix is a fixed funnel shift of aligned words:
// message word i (bytes 4i .. 4i+3 of 0x00 || leaf) is leaf bytes 4i-1 .. 4i+2, the top byte of the leaf's little-endian
// word i-1 and the low three bytes of word i.
__global__ void __launch_bounds__(128) raw_leaf_hash_kernel(FeParams p, uint8_t* __restrict__ rows) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= p.n || p.str_bad[2 * e]) return;  // no leaf: the fold stops before this entry
    const uint4* src = reinterpret_cast<const uint4*>(p.decoded + p.dec_off[2 * e]);
    const uint32_t L = p.dec_len[2 * e], len = L + 1u;
    Sha256State s;
    s.init();
    const uint32_t nb = (len + 9u + 63u) / 64u;
    uint32_t carry = 0;  // the leaf's word before this block (the 0x00 prefix for block 0)
    for (uint32_t b = 0; b < nb; ++b) {
        uint32_t v[16], w[16];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            const uint4 x = 64u * b + 16u * g < L ? src[4u * b + g] : make_uint4(0, 0, 0, 0);
            v[4 * g] = x.x; v[4 * g + 1] = x.y; v[4 * g + 2] = x.z; v[4 * g + 3] = x.w;
        }
#pragma unroll
        for (int i = 0; i < 16; ++i)
            w[i] = sha256_pad_word(bswap32(__funnelshift_r(i ? v[i - 1] : carry, v[i], 24)), 64u * b + 4u * i, len);
        carry = v[15];
        if (b == nb - 1u) { w[14] = 0; w[15] = len * 8u; }
        sha256_compress_rolled(s, w, 1u);
    }
    uint32_t h[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = s.h[i];
    store_row(rows + 32 * e, h);
}

// where this chunk's fold ends: see FoldChunk
__device__ __forceinline__ uint64_t fold_end(const FoldChunk& f) {
    const uint64_t size = f.tree->t.size, lim = f.first_pos + f.cnt, miss = f.tree->missing;
    if (size < f.first_pos) return size;
    return miss < lim ? (miss > size ? miss : size) : lim;
}

__global__ void __launch_bounds__(256) tree_missing_kernel(FoldChunk f) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= f.cnt || f.flags[j * f.stride] != f.match) return;
    const uint64_t pos = f.first_pos + j;
    if (pos >= f.tree->t.size) atomicMin(&f.tree->missing, (unsigned long long)pos);
}

// src holds the level's nodes from position `base` on (level 0: the chunk's leaf rows from first_pos, higher levels: the
// previous launch's parents from a_l); dst gets the parents from a_l >> 1 on.  Only thread 0 touches edge[level]: it
// reads the old row for the first parent before it writes the new one.
__global__ void __launch_bounds__(128) tree_level_kernel(FoldChunk f, uint32_t level, const uint8_t* __restrict__ src,
                                                        uint8_t* __restrict__ dst) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t a = f.tree->t.size >> level, b = fold_end(f) >> level;
    if (a == b) return;
    const uint64_t base = level == 0 ? f.first_pos : a, pa = a >> 1, pb = b >> 1, p = pa + k;
    uint8_t* edge = f.tree->t.edge[level];
    if (p < pb) {
        uint32_t l[8], r[8], h[8];
        load_row(2 * p < a ? edge : src + 32 * (2 * p - base), l);
        load_row(src + 32 * (2 * p + 1 - base), r);
        node_hash(l, r, h);
        store_row(dst + 32 * (p - pa), h);
    }
    if (k == 0 && (b & 1)) {
        uint32_t h[8];
        load_row(src + 32 * (b - 1 - base), h);
        store_row(edge, h);
    }
}

__global__ void tree_commit_kernel(FoldChunk f) {
    f.tree->t.size = fold_end(f);
    f.tree->missing = ~0ull;
}

__global__ void tree_root_kernel(TreeDev* tree) {
    ctmr_tree& t = tree->t;
    const uint64_t size = t.size;
    uint32_t r[8];
    if (size == 0) {  // SHA-256 of the empty string
        Sha256State s;
        s.init();
        uint32_t w[16] = {0x80000000u, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        sha256_compress_rolled(s, w, 1u);
#pragma unroll
        for (int i = 0; i < 8; ++i) r[i] = s.h[i];
    } else {
        const int low = __ffsll((long long)size) - 1;
        load_row(t.edge[low], r);
        for (int k = low + 1; k < 64; ++k) {
            if (!((size >> k) & 1ull)) continue;
            uint32_t l[8], h[8];
            load_row(t.edge[k], l);
            node_hash(l, r, h);
#pragma unroll
            for (int i = 0; i < 8; ++i) r[i] = h[i];
        }
    }
    store_row(t.root, r);
    for (int k = 0; k < 64; ++k)
        if (!((size >> k) & 1ull)) memset(t.edge[k], 0, 32);
}

__host__ __forceinline__ uint64_t shr64(uint64_t x, uint32_t s) { return s >= 64u ? 0ull : x >> s; }

}  // namespace

cudaError_t launch_raw_leaf_hash(const FeParams& p, uint8_t* rows, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    raw_leaf_hash_kernel<<<(unsigned)((p.n + 127) / 128), 128, 0, s>>>(p, rows);
    return cudaGetLastError();
}

cudaError_t launch_tree_fold(const FoldChunk& f, uint8_t* const lvl[2], cudaStream_t s, uint32_t* launches) {
    *launches = 0;
    if (f.cnt == 0) return cudaSuccess;
    tree_missing_kernel<<<(unsigned)((f.cnt + 255) / 256), 256, 0, s>>>(f);
    ++*launches;
    // Levels where the chunk's own range [first_pos, first_pos + cnt) is empty are empty for the part that folds too
    const uint64_t lo = f.first_pos, hi = f.first_pos + f.cnt;
    for (uint32_t l = 0; l < 64u && shr64(lo, l) != shr64(hi, l); ++l) {
        const uint64_t parents = shr64(hi, l + 1) - shr64(lo, l + 1) + 1;
        tree_level_kernel<<<(unsigned)((parents + 127) / 128), 128, 0, s>>>(f, l, l == 0 ? f.leaves : lvl[(l - 1) & 1], lvl[l & 1]);
        ++*launches;
    }
    tree_commit_kernel<<<1, 1, 0, s>>>(f);
    ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_tree_root(TreeDev* tree, cudaStream_t s) {
    tree_root_kernel<<<1, 1, 0, s>>>(tree);
    return cudaGetLastError();
}

}  // namespace ctmr
