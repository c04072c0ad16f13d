// ctmr_merkle.cu -- the logs' Merkle trees (RFC 6962 §2.1) over the entries of ctmr_process_raw_tree /
// ctmr_process_tiles_tree (one tree) and ctmr_process_raw_trees / ctmr_process_tiles_trees (one tree per log of the
// batch) (include/ctmr_frontend.h).  The one-tree calls are the case of one tree whose order is the identity.
//
//   K_raw_leaf_hash   thread per entry    SHA-256(0x00 || decoded leaf_input), read from the decoded arena
//   (tile_leaf_hash)                      tiles: the leaf hashes of ctmr_tiles.cu, unchanged
//   K_body_fold_order warp per body       bodies (ctmr_process_raw_bodies_tree(s)): the host's per-body windows and the JSON
//                                         walk's body_base -> the chunk's order (entries skipped or after a stop unlisted)
//   K_tree_missing    thread per entry    per tree, lowest log position of the chunk without a leaf (bad base64, bad tile)
//   K_tree_level      thread per parent   one level of every tree's range: parents of the pairs inside it, the left edge
//                                         node as the first left child, the last node as the new edge node
//   K_tree_commit     thread per tree     the tree's new size
//   K_tree_root       thread per tree     the root from the edge
// On a group (ctmr_group_process_*_tree(s)) member 0 holds the trees and folds its chunk as above; members 1.. fold theirs
// into ranges (TreeRange), which member 0 appends in member order:
//   K_range_missing   thread per entry    per range, lowest log position of the chunk without a leaf
//   K_range_level     thread per parent   tree_level with the range's odd first node stored as left[l], not paired
//   K_range_commit    thread per range    the range's bounds
//   K_tree_merge      thread per tree     the members' ranges appended to the edge (member 0, after the peer copies)
//
// A tree is held as its right edge (ctmr_tree): for every bit k of size, the root of the complete subtree of 2^k leaves
// ending at the highest multiple of 2^(k+1) at or below size.  Folding leaves [a, b) in: at level l the chunk covers node
// positions [a_l, b_l) = [a >> l, b >> l); pairs (2p, 2p+1) inside it make the parents [a_l >> 1, b_l >> 1); an odd a_l
// takes edge[l] as the left child of the first parent; an odd b_l leaves node b_l - 1 as the new edge[l].  Once the range
// is empty the higher rows keep what they hold.  A chunk of n leaves costs about n node hashes of two compressions each
// and one launch per level of its widest tree range.  The host lists a chunk's entries grouped by tree (FoldChunk.order),
// so each tree reads its leaves as one run in log order; the threads of a level launch are split between the trees by
// level_base.
#include <algorithm>

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

__host__ __device__ __forceinline__ uint64_t shr64(uint64_t x, uint32_t s) { return s >= 64u ? 0ull : x >> s; }

// where a tree's fold of this chunk ends: see FoldTree
__device__ __forceinline__ uint64_t fold_end(const TreeDev* tree, const FoldTree& d) {
    const uint64_t size = tree->t.size, lim = d.first_pos + d.cnt, miss = tree->missing;
    if (size < d.first_pos) return size;
    return miss < lim ? (miss > size ? miss : size) : lim;
}

// Tree d's first thread of a level-l launch, and its first row in that launch's level buffer.  Tree d has at most
// (cnt >> (l + 1)) + 2 parents at level l, and consecutive trees' bases differ by at least that much, so the trees'
// ranges of threads and rows never overlap; the last ends below (total >> (l + 1)) + 2 * n_desc.
__device__ __forceinline__ uint64_t level_base(const FoldTree& d, uint32_t i, uint32_t level) {
    return shr64(d.off, level + 1) + 2ull * i;
}

// the last tree i with key(i) <= k; f.n_desc when there is none (binary search: key is non-decreasing in i)
template <class Key>
__device__ __forceinline__ uint32_t find_tree(const FoldChunk& f, uint64_t k, Key key) {
    if (key(0) > k) return f.n_desc;
    uint32_t lo = 0, hi = f.n_desc;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (key(mid) <= k) lo = mid;
        else hi = mid;
    }
    return lo;
}

// the leaf row of tree d's entry j (the chunk's entries in log order through f.order)
__device__ __forceinline__ const uint8_t* leaf_row(const FoldChunk& f, const FoldTree& d, uint64_t j) {
    const uint64_t at = d.off + j;
    return f.leaves + 32 * (f.order ? (uint64_t)f.order[at] : at);
}

// listed entry g: whether it has no leaf, and then its tree's index in the chunk and its log position
__device__ __forceinline__ bool no_leaf(const FoldChunk& f, uint64_t g, uint32_t* i_out, uint64_t* pos) {
    if (g >= f.total) return false;
    const uint32_t i = find_tree(f, g, [&](uint32_t x) { return (uint64_t)f.desc[x].off; });
    if (i == f.n_desc) return false;
    const FoldTree d = f.desc[i];
    if (g >= (uint64_t)d.off + d.cnt) return false;  // entries a tiles chunk cut off after its stop
    const uint64_t e = f.order ? (uint64_t)f.order[g] : g;
    if (f.flags[e * f.stride] != f.match) return false;
    *i_out = i;
    *pos = d.first_pos + (g - d.off);
    return true;
}

// one thread per listed entry: the lowest position of each tree without a leaf
__global__ void __launch_bounds__(256) tree_missing_kernel(FoldChunk f) {
    uint32_t i;
    uint64_t pos;
    if (!no_leaf(f, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, &i, &pos)) return;
    TreeDev* tree = f.trees + f.desc[i].tree;
    if (pos >= tree->t.size) atomicMin(&tree->missing, (unsigned long long)pos);
}

// One level of every tree of the chunk.  Per tree: src holds the level's nodes from position `base` on (level 0: the
// tree's leaf rows from first_pos, through the order; higher levels: the previous launch's parents from a_l, at the tree's
// rows of that launch); dst gets the parents from a_l >> 1 on, at the tree's rows of this launch.  Only the tree's first
// thread touches its edge[level]: it reads the old row for the first parent before it writes the new one.
__global__ void __launch_bounds__(128) tree_level_kernel(FoldChunk f, uint32_t level, const uint8_t* __restrict__ src,
                                                        uint8_t* __restrict__ dst) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t i = find_tree(f, k, [&](uint32_t x) { return level_base(f.desc[x], x, level); });
    if (i == f.n_desc) return;
    const FoldTree d = f.desc[i];
    TreeDev* tree = f.trees + d.tree;
    const uint64_t a = tree->t.size >> level, b = fold_end(tree, d) >> level;
    if (a == b) return;
    const uint64_t k0 = level_base(d, i, level), pa = a >> 1, pb = b >> 1, p = pa + (k - k0);
    const uint64_t in = level == 0 ? 0 : level_base(d, i, level - 1);
    auto row = [&](uint64_t pos) {  // node `pos` of this level
        return level == 0 ? leaf_row(f, d, pos - d.first_pos) : src + 32 * (in + pos - a);
    };
    uint8_t* edge = tree->t.edge[level];
    if (p < pb) {
        uint32_t l[8], r[8], h[8];
        load_row(2 * p < a ? edge : row(2 * p), l);
        load_row(row(2 * p + 1), r);
        node_hash(l, r, h);
        store_row(dst + 32 * (k0 + p - pa), h);
    }
    if (k == k0 && (b & 1)) {
        uint32_t h[8];
        load_row(row(b - 1), h);
        store_row(edge, h);
    }
}

// one thread per tree of the chunk
__global__ void tree_commit_kernel(FoldChunk f) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= f.n_desc) return;
    const FoldTree d = f.desc[i];
    TreeDev* tree = f.trees + d.tree;
    tree->t.size = fold_end(tree, d);
    tree->missing = ~0ull;
}

// one thread per tree of the call
__global__ void tree_root_kernel(TreeDev* trees, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ctmr_tree& t = trees[i].t;
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

// ---- ranges (members 1.. of a group call) and their merge on the home member -------------------------------------------
// ceil(x / 2^s)
__device__ __forceinline__ uint64_t shr64_up(uint64_t x, uint32_t s) {
    return s >= 64u ? (x != 0) : (x >> s) + ((x & ((1ull << s) - 1ull)) != 0);
}
__device__ __forceinline__ uint64_t range_begin(const FoldTree& d) { return d.first_pos + d.skip; }
// where a tree's range of this chunk ends: its first missing leaf at or above range_begin (miss), or the run's end
__device__ __forceinline__ uint64_t range_end(const FoldTree& d, unsigned long long miss) {
    const uint64_t lim = d.first_pos + d.cnt;
    return miss < lim ? miss : lim;
}

// one thread per listed entry: the lowest position of each range without a leaf
__global__ void __launch_bounds__(256) range_missing_kernel(FoldChunk f, unsigned long long* __restrict__ miss) {
    uint32_t i;
    uint64_t pos;
    if (!no_leaf(f, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, &i, &pos)) return;
    if (pos >= range_begin(f.desc[i])) atomicMin(&miss[i], (unsigned long long)pos);
}

// tree_level_kernel for ranges: level l of range i covers nodes [a, b) = [ceil(begin / 2^l), end >> l); an odd a is
// stored as left[l] instead of being paired with the edge, so the pairs start at a + 1; an odd b leaves node b - 1 as
// right[l].  The parents [(a + 1) >> 1, b >> 1) go to the range's rows of this launch.
__global__ void __launch_bounds__(128) range_level_kernel(FoldChunk f, uint32_t level, const uint8_t* __restrict__ src,
                                                         uint8_t* __restrict__ dst, TreeRange* __restrict__ out,
                                                         const unsigned long long* __restrict__ miss) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t i = find_tree(f, k, [&](uint32_t x) { return level_base(f.desc[x], x, level); });
    if (i == f.n_desc) return;
    const FoldTree d = f.desc[i];
    const uint64_t a = shr64_up(range_begin(d), level), b = range_end(d, miss[i]) >> level;
    if (a >= b) return;
    const uint64_t k0 = level_base(d, i, level), pa = (a + 1) >> 1, pb = b >> 1, p = pa + (k - k0);
    const uint64_t in = level == 0 ? 0 : level_base(d, i, level - 1);
    auto row = [&](uint64_t pos) {  // node `pos` of this level
        return level == 0 ? leaf_row(f, d, pos - d.first_pos) : src + 32 * (in + pos - a);
    };
    if (p < pb) {
        uint32_t l[8], r[8], h[8];
        load_row(row(2 * p), l);
        load_row(row(2 * p + 1), r);
        node_hash(l, r, h);
        store_row(dst + 32 * (k0 + p - pa), h);
    }
    if (k == k0) {
        uint32_t h[8];
        if (a & 1) {
            load_row(row(a), h);
            store_row(out[i].left[level], h);
        }
        if (b & 1) {
            load_row(row(b - 1), h);
            store_row(out[i].right[level], h);
        }
    }
}

// one thread per range of the chunk: its bounds and tree, and the missing-leaf word back to ~0
__global__ void range_commit_kernel(FoldChunk f, TreeRange* __restrict__ out, unsigned long long* __restrict__ miss) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= f.n_desc) return;
    const FoldTree d = f.desc[i];
    out[i].begin = range_begin(d);
    out[i].end = range_end(d, miss[i]);
    out[i].tree = d.tree;
    miss[i] = ~0ull;
}

// a complete subtree of 2^level leaves appended to the edge at position size (a multiple of 2^level): binary carry
__device__ __forceinline__ void push_node(ctmr_tree& t, uint64_t& size, const uint8_t* row, uint32_t level) {
    uint32_t h[8];
    load_row(row, h);
    uint32_t k = level;
    for (; k < 64 && ((size >> k) & 1ull); ++k) {
        uint32_t l[8], x[8];
        load_row(t.edge[k], l);
        node_hash(l, h, x);
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = x[j];
    }
    store_row(t.edge[k], h);
    size += 1ull << level;
}

// one thread per tree of the call: each member's range of the tree, in member order, appended when it starts at the
// tree's size -- left nodes by ascending level, then right nodes by descending level -- so that size ends at its end
__global__ void tree_merge_kernel(TreeDev* trees, uint32_t n, RangeSet set) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n) return;
    ctmr_tree& t = trees[d].t;
    uint64_t size = t.size;
    for (uint32_t r = 0; r < set.members; ++r) {
        const TreeRange* g = set.recv + (uint64_t)r * set.stride;
        uint32_t lo = 0, hi = set.n[r];
        while (lo < hi) {  // the member's ranges are ordered by tree
            const uint32_t mid = (lo + hi) >> 1;
            if (g[mid].tree < d) lo = mid + 1;
            else hi = mid;
        }
        if (lo == set.n[r] || g[lo].tree != d) continue;
        const TreeRange& x = g[lo];
        if (x.begin != size) continue;  // an earlier stop (or an earlier member's) ends the tree below this range
        for (uint32_t l = 0; l < 64; ++l) {
            const uint64_t a = shr64_up(x.begin, l), b = x.end >> l;
            if (a >= b) break;
            if (a & 1) push_node(t, size, x.left[l], l);
        }
        for (int l = 63; l >= 0; --l) {
            const uint64_t a = shr64_up(x.begin, (uint32_t)l), b = x.end >> l;
            if (a < b && (b & 1)) push_node(t, size, x.right[l], (uint32_t)l);
        }
    }
    t.size = size;
}

// one warp per body of the chunk: its window's entries into their slots of the order
__global__ void __launch_bounds__(128) body_fold_order_kernel(const BodyWindow* __restrict__ win, uint32_t n_bodies,
                                                             const uint32_t* __restrict__ body_base, uint32_t* __restrict__ order) {
    const uint32_t b = blockIdx.x * 4u + (threadIdx.x >> 5);
    if (b >= n_bodies) return;
    const BodyWindow w = win[b];
    const uint32_t e0 = body_base[b] + w.first;
    for (uint32_t k = threadIdx.x & 31u; k < w.cnt; k += 32u) order[w.slot + k] = e0 + k;
}

// Levels where a tree's own range [first_pos, first_pos + cnt) is empty are empty for the part that folds too: the chunk
// takes as many level launches as its widest range has levels
uint32_t fold_levels(const FoldTree* hdesc, uint32_t n) {
    uint32_t levels = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint64_t x = hdesc[i].first_pos ^ (hdesc[i].first_pos + hdesc[i].cnt);
        levels = std::max(levels, x ? 64u - (uint32_t)__builtin_clzll(x) : 0u);
    }
    return levels;
}

}  // namespace

cudaError_t launch_raw_leaf_hash(const FeParams& p, uint8_t* rows, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    raw_leaf_hash_kernel<<<(unsigned)((p.n + 127) / 128), 128, 0, s>>>(p, rows);
    return cudaGetLastError();
}

cudaError_t launch_body_fold_order(const BodyWindow* win, uint32_t n_bodies, const uint32_t* body_base, uint32_t* order, cudaStream_t s) {
    if (n_bodies == 0) return cudaSuccess;
    body_fold_order_kernel<<<(n_bodies + 3u) / 4u, 128, 0, s>>>(win, n_bodies, body_base, order);
    return cudaGetLastError();
}

cudaError_t launch_tree_fold(const FoldChunk& f, const FoldTree* hdesc, uint8_t* const lvl[2], cudaStream_t s, uint32_t* launches) {
    *launches = 0;
    if (f.n_desc == 0) return cudaSuccess;
    tree_missing_kernel<<<(unsigned)((f.total + 255) / 256), 256, 0, s>>>(f);
    ++*launches;
    const uint32_t levels = fold_levels(hdesc, f.n_desc);
    for (uint32_t l = 0; l < levels; ++l) {
        const uint64_t threads = shr64(f.total, l + 1) + 2ull * f.n_desc;
        tree_level_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(f, l, l == 0 ? f.leaves : lvl[(l - 1) & 1], lvl[l & 1]);
        ++*launches;
    }
    tree_commit_kernel<<<(f.n_desc + 127) / 128, 128, 0, s>>>(f);
    ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_tree_root(TreeDev* trees, uint32_t n, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    tree_root_kernel<<<(n + 127) / 128, 128, 0, s>>>(trees, n);
    return cudaGetLastError();
}

cudaError_t launch_range_fold(const FoldChunk& f, const FoldTree* hdesc, uint8_t* const lvl[2], TreeRange* out, unsigned long long* miss,
                              cudaStream_t s, uint32_t* launches) {
    *launches = 0;
    if (f.n_desc == 0) return cudaSuccess;
    range_missing_kernel<<<(unsigned)((f.total + 255) / 256), 256, 0, s>>>(f, miss);
    ++*launches;
    const uint32_t levels = fold_levels(hdesc, f.n_desc);
    for (uint32_t l = 0; l < levels; ++l) {
        const uint64_t threads = shr64(f.total, l + 1) + 2ull * f.n_desc;
        range_level_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(f, l, l == 0 ? f.leaves : lvl[(l - 1) & 1], lvl[l & 1], out, miss);
        ++*launches;
    }
    range_commit_kernel<<<(f.n_desc + 127) / 128, 128, 0, s>>>(f, out, miss);
    ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_tree_merge(TreeDev* trees, uint32_t n, const RangeSet& set, cudaStream_t s) {
    if (n == 0 || set.members == 0) return cudaSuccess;
    tree_merge_kernel<<<(n + 127) / 128, 128, 0, s>>>(trees, n, set);
    return cudaGetLastError();
}

}  // namespace ctmr
