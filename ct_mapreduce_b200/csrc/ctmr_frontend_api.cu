// ctmr_frontend_api.cu -- the entry points of include/ctmr_frontend.h (SURVEY.md §8(f)-2): get-entries strings -> base64
// decode -> TLS framing -> Chain[0] identification -> the path (ctmr_process_raw); static-ct-api data tiles -> split ->
// framing -> Chain[0] by fingerprint -> the path (ctmr_process_tiles, ctmr_register_chain_certs).  Each runs on one GPU, on
// a group of GPUs driven by one process (ctmr_group_*), on one GPU with the log's Merkle tree folded in
// (ctmr_process_*_tree), and as a collective call of one process per GPU (a ctx attached with ctmr_peer_attach).
//
// One driver serves them all (process_members, over the members of the call: one ctx, or the members of a group).  A call
// is cut into ROUNDS of one CHUNK per member (entry and character budgets of the front end's buffers).  Per round:
//   upload   each chunk's characters and string spans (pages) or tile bytes (tiles), on a copy stream, into one of two
//            upload stages -- round k+1's uploads overlap round k's kernels and the host round trips of its issuer
//            identification;
//   front    pages: fe_decode / fe_frame / fe_tbs / fe_issuer, the decoded leaves stay in the arena; tiles: tile_split /
//            tile_frame / fe_tbs / tile_issuer, the leaves stay in the stage.  The chunk becomes a device-resident batch
//            (ctmr_dev_batch with explicit lengths);
//   path     K_map ... K_pairs over that batch in place -- ctmr_process_device on one GPU; on a group one round of the key
//            exchange (run_round, ctmr_api.cu, with each member's chunk as its slice and its stream for everything):
//            every member maps its chunk, hands foreign keys to their owners over NVLink, the owners reduce, the bits
//            are pulled back;
//   back     x509 leaf failures, PEM of the new certificates, outputs to the host.
// On one GPU a chunk is as large as the budgets allow.  On a group a round takes one chunk per member, cut from ONE
// contiguous window of the batch, so that entry i keeps global index next_index + i and the result equals the
// single-GPU run on the same input.  The two formats (Pages, Tiles) supply only what differs between them.
#include <thread>

#include "ctmr_ctx.cuh"

namespace {

// One member's chunk of a round: units [lo, hi) of the caller's batch (entries of pages, or tiles) and their entries
// [e0, e1) (the same range for pages), from its upload to its back half.
struct Chunk {
    uint64_t lo = 0, hi = 0;
    uint64_t e0 = 0, e1 = 0;
    uint64_t bytes = 0;           // uploaded: the characters of pages, the tile bytes of tiles
    int stage = 0;                // upload stage it sits in
    TileParams p{};               // the front end's kernel parameters; pages use p.fe only
    ctmr_dev_batch db{};
    ctmr_dev_out dout{};
    bool stopped = false;         // tiles: holds the first tile with an unknown Chain[0] fingerprint; [lo, hi) cut before it
    std::vector<std::array<uint8_t, 32>> missing;  // that tile's unknown fingerprints, sorted
    // tree calls (tree_group): the trees of the chunk's entries, in tree order; whether their order was uploaded into the
    // stage (it is not when it is the identity); how many entries it lists
    std::vector<FoldTree> fold;
    bool ordered = false;
    uint64_t listed = 0;

    // keeps the first `units` units, which hold `entries` entries
    void cut(uint64_t units, uint64_t entries) {
        hi = lo + units;
        e1 = e0 + entries;
        p.n_tiles = (uint32_t)units;
        p.n = p.fe.n = db.n = entries;
    }
};

// the front end's buffers on a member, and its counters of this call
int fe_prepare(ctmr_ctx* c) {
    CU(c, cudaSetDevice(c->device));
    const int rc = frontend_ensure(c);
    if (rc) return rc;
    c->fe->fe_ms = c->fe->path_ms = 0.f;
    c->fe->launches = 0;
    return CTMR_OK;
}

// ---- the logs' Merkle trees (ctmr_process_*_tree, ctmr_process_*_trees) ------------------------------------------------
// The trees of a tree call: the one-tree forms pass one tree and no log (every entry is the tree's); the routed forms
// pass n trees and the tree of every entry (pages), tile (tiles) or body (bodies), CTMR_NO_TREE for none.  Bodies also
// pass the log position of every body's first entry (the start of its get-entries request).
struct TreeArgs {
    ctmr_tree* trees = nullptr;
    uint32_t n = 0;
    const uint32_t* log = nullptr;
    bool routed = false;
    const uint64_t* start = nullptr;
};

// the arguments of a routed call before the format's own rules: `units` entries or tiles, and their trees
int tree_route_args(ctmr_ctx* c, const TreeArgs* t, uint64_t units) {
    if (t->n > CTMR_MAX_TREES) return fail(c, CTMR_E_INVALID, "trees: more than CTMR_MAX_TREES trees");
    if (t->n && !t->trees) return fail(c, CTMR_E_INVALID, "trees: null trees");
    if (units && !t->log) return fail(c, CTMR_E_INVALID, "trees: null log ids");
    for (uint64_t u = 0; u < units; ++u)
        if (t->log[u] >= t->n && t->log[u] != CTMR_NO_TREE) return fail(c, CTMR_E_INVALID, "trees: a log id names no tree");
    return CTMR_OK;
}

// the tree state for n trees, built whole (a smaller one is released first); `ranges`: with the range buffers of a
// group's member 1..; `recv_members`: with member 0's room for that many members' ranges
int tree_ensure(ctmr_ctx* c, uint32_t n, bool ranges, uint32_t recv_members) {
    FrontEnd* f = c->fe.get();
    if (f->tree && f->tree->cap_trees >= n && (!ranges || f->tree->range_miss) && f->tree->recv_members >= recv_members) return CTMR_OK;
    f->tree.reset();
    std::unique_ptr<TreeState> tr(new (std::nothrow) TreeState());
    if (!tr) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    const uint64_t E = f->cap_entries;
    const uint32_t cap = (uint32_t)pow2_at_least(std::max<uint32_t>(n, 1));
    CU(c, alloc(tr->dev, cap));
    CU(c, alloc(tr->host, cap));
    CU(c, alloc(tr->desc, cap));
    CU(c, alloc(tr->h_desc, cap));
    for (int k = 0; k < 2; ++k) {
        CU(c, alloc(tr->order[k], E));
        CU(c, alloc(tr->h_order[k], E));
    }
    CU(c, alloc(tr->leaf, E * 32));
    for (DevBuf<uint8_t>& lvl : tr->lvl) CU(c, alloc(lvl, (E / 2 + 2ull * cap) * 32));
    if (ranges) {
        for (DevBuf<TreeRange>& r : tr->range) CU(c, alloc(r, cap));
        CU(c, alloc(tr->range_miss, cap));
    }
    if (recv_members) {
        CU(c, alloc(tr->recv, (uint64_t)recv_members * cap));
        CU(c, create(tr->merge0, cudaEventDefault));
        CU(c, create(tr->merge1, cudaEventDefault));
    }
    tr->recv_members = recv_members;
    tr->cap_trees = cap;
    f->tree = std::move(tr);
    return CTMR_OK;
}

// The caller's trees to the device of member 0 (c) for the whole call, with room for the ranges of `others` more
// members; next[d]: log position of tree d's first entry in the call
int tree_begin(ctmr_ctx* c, const TreeArgs* t, const std::vector<uint64_t>& next, uint32_t others) {
    int rc = tree_ensure(c, t->n, false, others);
    if (rc) return rc;
    TreeState* tr = c->fe->tree.get();
    tr->start.resize(t->n);
    for (uint32_t d = 0; d < t->n; ++d) {
        std::memcpy(&tr->host[d].t, &t->trees[d], sizeof(ctmr_tree));
        tr->host[d].missing = ~0ull;
        tr->start[d] = t->trees[d].size;
    }
    CU(c, cudaMemcpyAsync(tr->dev, tr->host, t->n * sizeof(TreeDev), cudaMemcpyHostToDevice, c->stream));
    tr->n_trees = t->n;
    tr->log = t->log;
    tr->next = next;
    tr->count.assign(t->n, 0);
    tr->active = true;
    tr->ranges = false;
    tr->merge_timed = false;
    return CTMR_OK;
}

// a group's member 1.. (c) of a call of n trees: range buffers, and the missing-leaf words at ~0
int tree_begin_ranges(ctmr_ctx* c, uint32_t n) {
    int rc = tree_ensure(c, n, true, 0);
    if (rc) return rc;
    TreeState* tr = c->fe->tree.get();
    CU(c, cudaMemsetAsync(tr->range_miss, 0xFF, tr->cap_trees * sizeof(unsigned long long), c->stream));
    tr->ranges = true;
    return CTMR_OK;
}

// Groups the entries of units [ch.lo, ch.hi) by tree (unit u holds width(u) entries) into ch.fold, each tree's entries
// taking its next log positions from the call's tree state `home` (member 0's: every member's upload reads and advances
// it, in member order), and uploads their order into the stage of c's chunk on the copy stream unless it is the identity
// (one tree and no entry of none).
template <class Width>
int tree_group(ctmr_ctx* c, TreeState* home, Chunk& ch, Width width) {
    ch.fold.clear();
    ch.ordered = false;
    ch.listed = 0;
    if (!home || !home->active) return CTMR_OK;
    std::vector<uint32_t>& cnt = home->count;
    std::fill(cnt.begin(), cnt.end(), 0u);
    uint64_t none = 0;
    for (uint64_t u = ch.lo; u < ch.hi; ++u) {
        const uint32_t l = home->log ? home->log[u] : 0;
        if (l == CTMR_NO_TREE) none += width(u);
        else cnt[l] += width(u);
    }
    uint32_t off = 0;
    for (uint32_t d = 0; d < home->n_trees; ++d) {
        if (!cnt[d]) continue;
        const uint64_t first = home->next[d], skip = home->start[d] > first ? home->start[d] - first : 0;  // <= 256
        ch.fold.push_back(FoldTree{first, d, off, cnt[d], (uint32_t)skip});
        home->next[d] += cnt[d];
        off += cnt[d];
    }
    ch.listed = off;
    ch.ordered = none || ch.fold.size() > 1;
    if (!ch.ordered || !off) return CTMR_OK;
    for (const FoldTree& t : ch.fold) cnt[t.tree] = t.off;  // from here on: each tree's next slot in the order
    TreeState* tr = c->fe->tree.get();
    uint32_t* h = tr->h_order[ch.stage];
    uint32_t e = 0;
    for (uint64_t u = ch.lo; u < ch.hi; ++u) {
        const uint32_t l = home->log ? home->log[u] : 0, w = width(u);
        if (l != CTMR_NO_TREE)
            for (uint32_t k = 0; k < w; ++k) h[cnt[l]++] = e + k;
        e += w;
    }
    CU(c, cudaMemcpyAsync(tr->order[ch.stage], h, off * 4ull, cudaMemcpyHostToDevice, c->fe->copy_stream));
    return CTMR_OK;
}

// a chunk cut to units [ch.lo, ch.hi) (tiles, at a stop) folds only their entries: each tree keeps the head of its run.
// The members' front halves run on threads of their own, so the counts are not home->count.
template <class Width>
void tree_cut(const TreeState* home, Chunk& ch, Width width) {
    if (ch.fold.empty()) return;
    std::vector<uint32_t> cnt(home->n_trees, 0u);
    for (uint64_t u = ch.lo; u < ch.hi; ++u) {
        const uint32_t l = home->log ? home->log[u] : 0;
        if (l != CTMR_NO_TREE) cnt[l] += width(u);
    }
    std::vector<FoldTree> kept;
    for (FoldTree t : ch.fold)
        if ((t.cnt = cnt[t.tree]) != 0) kept.push_back(t);
    ch.fold.swap(kept);
}

// folds a chunk's leaves into its trees (see FoldChunk), or on a group's member 1.. into its ranges of the chunk's stage
int tree_fold(ctmr_ctx* c, const Chunk& ch, const uint8_t* leaves, const uint8_t* flags, uint32_t stride, uint32_t match) {
    if (ch.fold.empty()) return CTMR_OK;
    TreeState* tr = c->fe->tree.get();
    const uint32_t n = (uint32_t)ch.fold.size();
    std::memcpy(tr->h_desc, ch.fold.data(), n * sizeof(FoldTree));
    CU(c, cudaMemcpyAsync(tr->desc, tr->h_desc, n * sizeof(FoldTree), cudaMemcpyHostToDevice, c->stream));
    const FoldChunk fc{tr->ranges ? nullptr : tr->dev.get(), tr->desc, n, stride, ch.ordered ? tr->order[ch.stage].get() : nullptr,
                       ch.listed, leaves, flags, match};
    uint8_t* const lvl[2] = {tr->lvl[0], tr->lvl[1]};
    uint32_t launches = 0;
    if (tr->ranges) CU(c, launch_range_fold(fc, ch.fold.data(), lvl, tr->range[ch.stage], tr->range_miss, c->stream, &launches));
    else CU(c, launch_tree_fold(fc, ch.fold.data(), lvl, c->stream, &launches));
    c->fe->launches += launches;
    return CTMR_OK;
}

// the last merge's time into member 0's fe_ms, once member 0's stream has passed it
int tree_merge_time(ctmr_ctx* c) {
    TreeState* tr = c->fe->tree.get();
    if (!tr->merge_timed) return CTMR_OK;
    float ms = 0.f;
    CU(c, cudaEventElapsedTime(&ms, tr->merge0, tr->merge1));
    c->fe->fe_ms += ms;
    tr->merge_timed = false;
    return CTMR_OK;
}

// A group's round: the ranges of members 1..upto-1 (members after a stop are left out) appended to the trees on member
// 0, on its stream, in one launch.  Issued after the round's back halves, so before member 0's next front half, which
// folds the next entries of each tree.  Each copy reads the member's ranges of this round's stage.  The member's range
// fold of the next round writes the other stage's, and the one after that is issued only once the next round's back
// half on member 0 has synchronized member 0's stream, which is past this copy.
int tree_merge(ctmr_ctx** m, uint32_t upto, const Chunk* cur, ctmr_ctx** failed) {
    ctmr_ctx* h = m[0];
    *failed = h;
    TreeState* tr = h->fe->tree.get();
    if (upto < 2 || tr->n_trees == 0) return CTMR_OK;
    CU(h, cudaSetDevice(h->device));
    int rc = tree_merge_time(h);  // the previous round's: member 0's stream was synchronized since
    if (rc) return rc;
    RangeSet set{tr->recv, tr->cap_trees, upto - 1, {}};
    for (uint32_t r = 1; r < upto; ++r) CU(h, cudaStreamWaitEvent(h->stream, m[r]->fe->ev1, 0));  // after the range fold
    CU(h, cudaEventRecord(tr->merge0, h->stream));
    for (uint32_t r = 1; r < upto; ++r) {
        const uint32_t n = set.n[r - 1] = (uint32_t)cur[r].fold.size();
        if (n)
            CU(h, cudaMemcpyPeerAsync(tr->recv + (uint64_t)(r - 1) * tr->cap_trees, h->device, m[r]->fe->tree->range[cur[r].stage],
                                      m[r]->device, n * sizeof(TreeRange), h->stream));
    }
    CU(h, launch_tree_merge(tr->dev, tr->n_trees, set, h->stream));
    CU(h, cudaEventRecord(tr->merge1, h->stream));
    ++h->fe->launches;
    tr->merge_timed = true;
    return CTMR_OK;
}

// the roots, and the trees back to the caller
int tree_end(ctmr_ctx* c, const TreeArgs* t) {
    TreeState* tr = c->fe->tree.get();
    CU(c, launch_tree_root(tr->dev, t->n, c->stream));
    CU(c, cudaMemcpyAsync(tr->host, tr->dev, t->n * sizeof(TreeDev), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    const int rc = tree_merge_time(c);
    if (rc) return rc;
    for (uint32_t d = 0; d < t->n; ++d) std::memcpy(&t->trees[d], &tr->host[d].t, sizeof(ctmr_tree));
    return CTMR_OK;
}

// ================================================================================================================
// get-entries pages: the units of a chunk are entries.  The stage is free again once the chunk is decoded.
// ================================================================================================================
struct Pages {
    static constexpr const char* kTooLarge = "a single entry exceeds the front end's character budget";
    static constexpr bool kStageHoldsLeaves = false;
    const ctmr_raw_batch* b;
    ctmr_raw_out* out;
    uint64_t done;  // entries that take their indices: all n whenever there is a batch, also when the call fails once a
                    // chunk has reached the path
    bool meta = false;  // the call computes string identities (process_members)

    std::vector<uint64_t> tree_pos;  // tree calls: log position of each tree's first entry
    TreeState* tree_state = nullptr;  // tree calls: the call's tree state, member 0's (process_members)

    Pages(const ctmr_raw_batch* b_, ctmr_raw_out* out_) : b(b_), out(out_), done(b_ ? b_->n : 0) {}
    int check(ctmr_ctx* c, const TreeArgs* tree);
    uint64_t units() const { return b->n; }
    uint64_t q_max(const ctmr_ctx* c) const { return c->fe->cap_entries; }
    int prepare(ctmr_ctx* c) const { return fe_prepare(c); }
    int fit(ctmr_ctx* c, uint64_t lo, uint64_t max_entries, uint64_t* hi_out) const;
    int upload(ctmr_ctx* c, Chunk& ch) const;
    int front(ctmr_ctx* c, Chunk& ch) const;
    int copy_back(ctmr_ctx* c, const Chunk& ch) const;
    void completed(uint64_t) const {}
    int stop(ctmr_ctx*, const Chunk&) const { return CTMR_OK; }  // a page chunk never stops
    void place(ctmr_ctx**, Chunk*, uint32_t) const {}  // entry positions are known at upload
    int fold(ctmr_ctx*, const Chunk&) const { return CTMR_OK; }  // folded in the front half
    uint64_t entries() const { return done; }
};

// tree: ctmr_process_raw_tree's rule as well; a routed call's rules fail before any index is taken
int Pages::check(ctmr_ctx* c, const TreeArgs* tree) {
    if (!b || !out || (tree && !tree->routed && !tree->trees)) return fail(c, CTMR_E_INVALID, "bad argument");
    if (b->n && (!b->text || !b->leaf_input_off || !b->leaf_input_len || !b->extra_data_off || !b->extra_data_len))
        return fail(c, CTMR_E_INVALID, "null batch buffers");
    int rc = check_pem(c, &out->path);
    if (rc) return rc;
    if (!tree) return CTMR_OK;
    if (!tree->routed) {
        if (b->n > ~0ull - tree->trees[0].size) return fail(c, CTMR_E_INVALID, "tree size + entries wraps around 2^64");
        tree_pos.assign(1, tree->trees[0].size);
        return CTMR_OK;
    }
    rc = tree_route_args(c, tree, b->n);
    std::vector<uint64_t> cnt(tree->n, 0);
    for (uint64_t i = 0; rc == CTMR_OK && i < b->n; ++i)
        if (tree->log[i] != CTMR_NO_TREE) ++cnt[tree->log[i]];
    for (uint32_t d = 0; rc == CTMR_OK && d < tree->n; ++d)
        if (cnt[d] > ~0ull - tree->trees[d].size) rc = fail(c, CTMR_E_INVALID, "trees: a tree's size + its entries wraps around 2^64");
    if (rc) {
        done = 0;
        return rc;
    }
    tree_pos.resize(tree->n);
    for (uint32_t d = 0; d < tree->n; ++d) tree_pos[d] = tree->trees[d].size;
    return CTMR_OK;
}

// How many entries starting at `lo` fit one chunk (at most max_entries): entry budget and half the character budget
// (the other half belongs to the stage being uploaded next).  Also validates the spans.
int Pages::fit(ctmr_ctx* c, uint64_t lo, uint64_t max_entries, uint64_t* hi_out) const {
    FrontEnd* f = c->fe.get();
    uint64_t hi = lo, chars = 0;
    while (hi < b->n && hi - lo < max_entries && hi - lo < f->cap_entries) {
        const uint64_t l1 = b->leaf_input_off[hi] + b->leaf_input_len[hi], x1 = b->extra_data_off[hi] + b->extra_data_len[hi];
        if (l1 > b->text_bytes || x1 > b->text_bytes) return fail(c, CTMR_E_INVALID, "string span outside the text buffer");
        const uint64_t add = (uint64_t)b->leaf_input_len[hi] + b->extra_data_len[hi];
        if (chars + add > f->cap_text / 2) break;
        chars += add;
        ++hi;
    }
    *hi_out = hi;
    return CTMR_OK;
}

// Characters and spans of entries [lo, hi) into upload stage ch.stage, asynchronously on the copy stream.
int Pages::upload(ctmr_ctx* c, Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    FeStage& st = f->stage[ch.stage];
    const uint64_t lo = ch.lo, cnt = ch.hi - ch.lo;
    ch.e0 = ch.lo;
    ch.e1 = ch.hi;
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaStreamWaitEvent(f->copy_stream, st.consumed, 0));  // the decode that last read this stage has run
    if (!cnt) {
        ch.bytes = 0;
        CU(c, cudaEventRecord(st.uploaded, f->copy_stream));
        return CTMR_OK;
    }
    const int rc = tree_group(c, tree_state, ch, [](uint64_t) { return 1u; });
    if (rc) return rc;
    uint64_t chars = 0, min_off = ~0ull, max_end = 0;
    for (uint64_t i = lo; i < ch.hi; ++i) {
        const uint64_t l0 = b->leaf_input_off[i], l1 = l0 + b->leaf_input_len[i];
        const uint64_t x0 = b->extra_data_off[i], x1 = x0 + b->extra_data_len[i];
        chars += (uint64_t)b->leaf_input_len[i] + b->extra_data_len[i];
        min_off = std::min(min_off, std::min(l0, x0));
        max_end = std::max(max_end, std::max(l1, x1));
    }
    std::memcpy(st.h_leaf_len, b->leaf_input_len + lo, cnt * 4);
    std::memcpy(st.h_extra_len, b->extra_data_len + lo, cnt * 4);
    if (max_end - min_off <= f->cap_text) {  // strings in place inside the response bodies: one copy
        ch.bytes = max_end - min_off;
        for (uint64_t i = 0; i < cnt; ++i) {
            st.h_leaf_off[i] = b->leaf_input_off[lo + i] - min_off;
            st.h_extra_off[i] = b->extra_data_off[lo + i] - min_off;
        }
        CU(c, cudaMemcpyAsync(st.text + 16, b->text + min_off, ch.bytes, cudaMemcpyHostToDevice, f->copy_stream));
    } else {  // scattered: pack on the host first
        st.pack.resize(chars);
        uint64_t w = 0;
        for (uint64_t i = 0; i < cnt; ++i) {
            st.h_leaf_off[i] = w;
            std::memcpy(st.pack.data() + w, b->text + b->leaf_input_off[lo + i], b->leaf_input_len[lo + i]);
            w += b->leaf_input_len[lo + i];
            st.h_extra_off[i] = w;
            std::memcpy(st.pack.data() + w, b->text + b->extra_data_off[lo + i], b->extra_data_len[lo + i]);
            w += b->extra_data_len[lo + i];
        }
        ch.bytes = w;
        CU(c, cudaMemcpyAsync(st.text + 16, st.pack.data(), ch.bytes, cudaMemcpyHostToDevice, f->copy_stream));
    }
    CU(c, cudaMemcpyAsync(st.leaf_off, st.h_leaf_off, cnt * 8, cudaMemcpyHostToDevice, f->copy_stream));
    CU(c, cudaMemcpyAsync(st.extra_off, st.h_extra_off, cnt * 8, cudaMemcpyHostToDevice, f->copy_stream));
    CU(c, cudaMemcpyAsync(st.leaf_len, st.h_leaf_len, cnt * 4, cudaMemcpyHostToDevice, f->copy_stream));
    CU(c, cudaMemcpyAsync(st.extra_len, st.h_extra_len, cnt * 4, cudaMemcpyHostToDevice, f->copy_stream));
    CU(c, cudaEventRecord(st.uploaded, f->copy_stream));
    return CTMR_OK;
}

// decode + frame + Chain[0] -> dense index of the cnt entries whose string spans are in stage ch.stage (text_bytes of
// characters from the stage's text); leaves ch.db / ch.dout describing the device-resident batch.  Issued after f->ev0.
int spans_front(ctmr_ctx* c, Chunk& ch, uint64_t text_bytes, uint64_t cnt, int64_t now_unix_ns, const ctmr_out* po, bool meta) {
    FrontEnd* f = c->fe.get();
    cudaStream_t s = c->stream;
    FeStage& st = f->stage[ch.stage];
    FeParams& p = ch.p.fe;
    p = FeParams{};
    p.text = st.text + 16;
    p.text_bytes = text_bytes;
    p.leaf_off = st.leaf_off; p.leaf_len = st.leaf_len; p.extra_off = st.extra_off; p.extra_len = st.extra_len;
    p.n = cnt;
    p.pad_size = f->pad_size; p.dec_off = f->dec_off; p.dec_len = f->dec_len; p.str_bad = f->str_bad; p.decoded = f->decoded;
    p.entry_status = f->entry_status; p.entry_type = f->entry_type; p.timestamp = f->timestamp; p.leaf_src = f->leaf_src;
    p.leaf_rel = f->leaf_rel; p.leaf_len_out = f->leaf_len_out; p.leaf_abs = f->leaf_abs; p.chain_abs = f->chain_abs;
    p.chain_len = f->chain_len; p.tbs_abs = f->tbs_abs; p.tbs_len = f->tbs_len; p.issuer_idx = f->issuer_idx;
    ch.db = ctmr_dev_batch{};
    ch.dout = ctmr_dev_out{};
    if (cnt) {
        CU(c, launch_fe_decode(p, f->scan_temp, f->scan_temp_bytes, c->sm_count, s));
        CU(c, cudaEventRecord(st.consumed, s));  // text and spans are dead once decoded: the stage may be refilled
        CU(c, launch_fe_frame(p, s));
        f->launches += 5;  // sizes, scan (cub: one kernel visible to us), decode, frame, tbs
        // ---- Chain[0] -> dense index; certificates never seen before go through ctmr_register_issuers once (the registry
        // is the group's: whichever member meets an issuer first, every member gets the same index)
        for (int round = 0;; ++round) {
            if (round > 64) return fail(c, CTMR_E_CUDA, "front end: issuer identification does not converge");
            IssuerCertTable tab{f->slots_dev, f->slot_mask, f->arena};
            CU(c, cudaMemsetAsync(f->pending, 0, (f->pending_mask + 1) * 8, s));
            CU(c, cudaMemsetAsync(f->unknown_count, 0, 4, s));
            CU(c, launch_fe_issuer(p, tab, f->pending, f->pending_mask, f->unknown_list, f->unknown_cap, f->unknown_count, c->sm_count, s));
            ++f->launches;
            unsigned int n_unknown = 0;
            CU(c, cudaMemcpyAsync(&n_unknown, f->unknown_count, 4, cudaMemcpyDeviceToHost, s));
            CU(c, cudaStreamSynchronize(s));
            if (n_unknown == 0) break;
            if (n_unknown > f->unknown_cap) n_unknown = f->unknown_cap;  // the rest shows up again next round
            std::vector<uint32_t> list(n_unknown);
            CU(c, cudaMemcpyAsync(list.data(), f->unknown_list, n_unknown * 4ull, cudaMemcpyDeviceToHost, s));
            CU(c, cudaStreamSynchronize(s));
            std::vector<uint8_t> blob;
            std::vector<uint64_t> offs(1, 0);
            for (uint32_t e : list) {
                uint64_t at = 0;
                uint32_t len = 0;
                CU(c, cudaMemcpyAsync(&at, f->chain_abs + e, 8, cudaMemcpyDeviceToHost, s));
                CU(c, cudaMemcpyAsync(&len, f->chain_len + e, 4, cudaMemcpyDeviceToHost, s));
                CU(c, cudaStreamSynchronize(s));
                const size_t w = blob.size();
                blob.resize(w + len);
                CU(c, cudaMemcpyAsync(blob.data() + w, f->decoded + at, len, cudaMemcpyDeviceToHost, s));
                CU(c, cudaStreamSynchronize(s));
                offs.push_back(blob.size());
            }
            std::vector<uint32_t> dense(n_unknown);
            const uint64_t before = f->slots_used;
            int rc = ctmr_register_issuers(c, blob.data(), offs.data(), n_unknown, dense.data());
            if (rc) return rc;
            if (f->slots_used == before) return fail(c, CTMR_E_CUDA, "front end: unresolved Chain[0] is already registered");
        }
        if (!ch.fold.empty()) {  // the leaves of this chunk into its trees, while the arena still holds them
            CU(c, launch_raw_leaf_hash(p, f->tree->leaf, s));
            ++f->launches;
            const int rc = tree_fold(c, ch, f->tree->leaf, f->str_bad, 2, 1);
            if (rc) return rc;
        }
    } else {
        CU(c, cudaEventRecord(st.consumed, s));
    }
    CU(c, cudaEventRecord(f->ev1, s));
    // ---- the path's input: the decoded arena, leaves where the decoder put them
    ctmr_dev_batch& db = ch.db;
    db.blob = f->decoded;
    if (cnt) {
        CU(c, cudaMemcpyAsync(&db.blob_bytes, f->dec_off + 2 * cnt, 8, cudaMemcpyDeviceToHost, s));
        CU(c, cudaStreamSynchronize(s));
    }
    db.offsets = f->leaf_abs;
    db.lens = f->leaf_len_out;
    db.n = cnt;
    db.issuer_idx = f->issuer_idx;
    db.now_unix_ns = now_unix_ns;
    ch.dout = f->out.dev_out(po->sha256 != nullptr, meta);
    return CTMR_OK;
}

int Pages::front(ctmr_ctx* c, Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaStreamWaitEvent(c->stream, f->stage[ch.stage].uploaded, 0));
    CU(c, cudaEventRecord(f->ev0, c->stream));
    return spans_front(c, ch, ch.bytes, ch.hi - ch.lo, b->now_unix_ns, &out->path, meta);
}

// the ctmr_raw_out outputs of a chunk's entries [e0, e1) after the path's, on c's stream (not waited for)
int raw_copy_back(ctmr_ctx* c, const Chunk& ch, const ctmr_raw_out* out) {
    FrontEnd* f = c->fe.get();
    cudaStream_t s = c->stream;
    const uint64_t lo = ch.e0, cnt = ch.e1 - ch.e0;
    if (cnt) {
        CU(c, d2h_rows(out->entry_status, f->entry_status, lo, cnt, s));
        CU(c, d2h_rows(out->entry_type, f->entry_type, lo, cnt, s));
        CU(c, d2h_rows(out->timestamp_ms, f->timestamp, lo, cnt, s));
        CU(c, d2h_rows(out->issuer, f->issuer_idx, lo, cnt, s));
        CU(c, d2h_rows(out->leaf_src, f->leaf_src, lo, cnt, s));
        CU(c, d2h_rows(out->leaf_off, f->leaf_rel, lo, cnt, s));
        CU(c, d2h_rows(out->leaf_len, f->leaf_len_out, lo, cnt, s));
    }
    return CTMR_OK;
}

// the front end's own outputs of a chunk, after the path's; waits for the chunk
int Pages::copy_back(ctmr_ctx* c, const Chunk& ch) const {
    const int rc = raw_copy_back(c, ch, out);
    if (rc) return rc;
    CU(c, cudaStreamSynchronize(c->stream));
    return CTMR_OK;
}

// ================================================================================================================
// static-ct-api data tiles: the units of a chunk are tiles.  The uploaded tile bytes ARE the path's input: K_map reads
// the leaves where the upload put them, so the stage stays busy until the chunk's PEM has been encoded.
// ================================================================================================================
struct Tiles {
    static constexpr const char* kTooLarge = "a single tile exceeds the front end's staging budget";
    static constexpr bool kStageHoldsLeaves = true;
    const ctmr_tile_batch* b;
    ctmr_tile_out* out;
    uint64_t done = 0;         // entries that take their indices: none when the arguments fail, those before a stop, else all
    bool meta = false;         // the call computes string identities (process_members)
    std::vector<uint64_t> ent;  // entries before each tile: ent[t] = sum of widths of tiles [0, t)
    std::vector<uint64_t> tree_pos;  // tree calls: log position of each tree's first entry (its first tile's)
    TreeState* tree_state = nullptr;  // tree calls: the call's tree state, member 0's (process_members)

    Tiles(const ctmr_tile_batch* b_, ctmr_tile_out* out_) : b(b_), out(out_) {}
    int check(ctmr_ctx* c, const TreeArgs* tree);
    uint64_t units() const { return b->n_tiles; }
    uint64_t q_max(const ctmr_ctx*) const { return ~0ull; }  // fit keeps a chunk inside the entry budget
    int prepare(ctmr_ctx* c) const;
    int fit(ctmr_ctx* c, uint64_t lo, uint64_t max_tiles, uint64_t* hi_out) const;
    int upload(ctmr_ctx* c, Chunk& ch) const;
    int front(ctmr_ctx* c, Chunk& ch) const;
    int copy_back(ctmr_ctx* c, const Chunk& ch) const;
    void completed(uint64_t tiles) const { out->tiles_done = tiles; }
    int stop(ctmr_ctx* c, const Chunk& ch) const;
    void place(ctmr_ctx**, Chunk*, uint32_t) const {}
    int fold(ctmr_ctx*, const Chunk&) const { return CTMR_OK; }  // folded in the front half
    uint64_t entries() const { return done; }
};

// ctmr_process_tiles_tree's rules for the tiles of one log (the batch's tiles of log `log`; every tile without a log),
// checked before any work like the widths and spans.  *first_pos: the log position of its first tile.
int tree_tile_args(ctmr_ctx* c, const ctmr_tile_batch* b, const uint32_t* tile_log, uint32_t log, const ctmr_tree* tree,
                   uint64_t* first_pos) {
    uint64_t first = ~0ull, prev = ~0ull, n = 0;
    for (uint64_t t = 0; t < b->n_tiles; ++t) {
        if (tile_log && tile_log[t] != log) continue;
        if (prev != ~0ull) {
            if (b->tile_index[t] != b->tile_index[prev] + 1) return fail(c, CTMR_E_INVALID, "tree: tiles are not consecutive");
            if (b->tile_width[prev] != 256) return fail(c, CTMR_E_INVALID, "tree: a partial tile that is not the last");
        } else {
            first = t;
        }
        prev = t;
        n += b->tile_width[t];
    }
    *first_pos = 0;
    if (first == ~0ull) return CTMR_OK;
    if (b->tile_index[first] > (~0ull - n) >> 8) return fail(c, CTMR_E_INVALID, "tree: the batch's last leaf index does not fit 64 bits");
    *first_pos = 256 * b->tile_index[first];
    if (tree->size < *first_pos || tree->size > *first_pos + b->tile_width[first])
        return fail(c, CTMR_E_INVALID, "tree: size is not inside the batch's first tile");
    return CTMR_OK;
}

// validates widths and spans (and with a tree its rules), fills ent
int Tiles::check(ctmr_ctx* c, const TreeArgs* tree) {
    if (!b || !out || (tree && !tree->routed && !tree->trees)) return fail(c, CTMR_E_INVALID, "bad argument");
    if (b->n_tiles && (!b->data || !b->tile_off || !b->tile_len || !b->tile_index || !b->tile_width))
        return fail(c, CTMR_E_INVALID, "null batch buffers");
    int rc = check_pem(c, &out->path);
    if (rc) return rc;
    if (out->missing_cap && !out->missing_fp) return fail(c, CTMR_E_INVALID, "missing_cap without missing_fp");
    ent.assign(b->n_tiles + 1, 0);
    for (uint64_t t = 0; t < b->n_tiles; ++t) {
        if (b->tile_width[t] < 1 || b->tile_width[t] > 256) return fail(c, CTMR_E_INVALID, "tile width outside 1..256");
        if (b->tile_off[t] > b->data_bytes || b->tile_len[t] > b->data_bytes - b->tile_off[t])
            return fail(c, CTMR_E_INVALID, "tile outside the data buffer");
        ent[t + 1] = ent[t] + b->tile_width[t];
    }
    if (tree) {
        const uint32_t* log = tree->routed ? tree->log : nullptr;
        if (tree->routed) {
            rc = tree_route_args(c, tree, b->n_tiles);
            if (rc) return rc;
        }
        tree_pos.assign(tree->n, 0);
        for (uint32_t d = 0; d < tree->n; ++d) {
            rc = tree_tile_args(c, b, log, d, &tree->trees[d], &tree_pos[d]);
            if (rc) return rc;
        }
    }
    done = ent[b->n_tiles];
    out->tiles_done = 0;
    out->n_missing = 0;
    return CTMR_OK;
}

int Tiles::prepare(ctmr_ctx* c) const {
    int rc = fe_prepare(c);
    if (rc == CTMR_OK) rc = tiles_ensure(c);
    if (rc) return rc;
    c->fe->tl->split_ms = 0.f;
    return CTMR_OK;
}

// How many tiles starting at `lo` fit one chunk (at most max_tiles): the entry budget and half the byte budget
int Tiles::fit(ctmr_ctx* c, uint64_t lo, uint64_t max_tiles, uint64_t* hi_out) const {
    FrontEnd* f = c->fe.get();
    uint64_t hi = lo, bytes = 0;
    while (hi < b->n_tiles && hi - lo < max_tiles && ent[hi + 1] - ent[lo] <= f->cap_entries && bytes + b->tile_len[hi] <= f->cap_text / 2) {
        bytes += b->tile_len[hi];
        ++hi;
    }
    *hi_out = hi;
    return CTMR_OK;
}

// tiles [lo, hi) into upload stage ch.stage, asynchronously on the copy stream
int Tiles::upload(ctmr_ctx* c, Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    TileState* tl = f->tl.get();
    FeStage& st = f->stage[ch.stage];
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaStreamWaitEvent(f->copy_stream, st.consumed, 0));  // the chunk that last used this stage is done with it
    ch.e0 = ent[ch.lo];
    ch.e1 = ent[ch.hi];
    const uint64_t cnt = ch.hi - ch.lo;
    TileDesc* h = tl->h_tiles[ch.stage];
    uint64_t bytes = 0, min_off = ~0ull, max_end = 0;
    for (uint64_t t = ch.lo; t < ch.hi; ++t) {
        bytes += b->tile_len[t];
        min_off = std::min(min_off, b->tile_off[t]);
        max_end = std::max(max_end, b->tile_off[t] + b->tile_len[t]);
    }
    const bool one_copy = cnt && max_end - min_off <= f->cap_text;  // tiles back to back in the caller's buffer
    uint64_t w = 0;
    if (!one_copy) st.pack.resize(bytes);
    for (uint64_t i = 0; i < cnt; ++i) {
        const uint64_t t = ch.lo + i;
        TileDesc& d = h[i];
        d.data_off = b->tile_off[t];
        d.index = b->tile_index[t];
        d.len = b->tile_len[t];
        d.first = (uint32_t)(ent[t] - ch.e0);
        d.width = b->tile_width[t];
        d.pad = 0;
        if (one_copy) {
            d.staged_off = b->tile_off[t] - min_off;
        } else {
            d.staged_off = w;
            std::memcpy(st.pack.data() + w, b->data + b->tile_off[t], d.len);
            w += d.len;
        }
    }
    ch.bytes = one_copy ? max_end - min_off : w;
    if (ch.bytes)
        CU(c, cudaMemcpyAsync(st.text + 16, one_copy ? b->data + min_off : st.pack.data(), ch.bytes, cudaMemcpyHostToDevice, f->copy_stream));
    if (cnt) CU(c, cudaMemcpyAsync(tl->tiles[ch.stage], h, cnt * sizeof(TileDesc), cudaMemcpyHostToDevice, f->copy_stream));
    const int rc = tree_group(c, tree_state, ch, [this](uint64_t t) { return (uint32_t)b->tile_width[t]; });
    if (rc) return rc;
    CU(c, cudaEventRecord(st.uploaded, f->copy_stream));
    return CTMR_OK;
}

// split + frame + fingerprint -> dense index of an uploaded chunk.  A chunk holding a tile with an unknown Chain[0]
// fingerprint is cut before that tile (ch.stopped, ch.missing).  Leaves ch.db / ch.dout describing the device-resident batch.
int Tiles::front(ctmr_ctx* c, Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    TileState* tl = f->tl.get();
    cudaStream_t s = c->stream;
    CU(c, cudaSetDevice(c->device));
    FeStage& st = f->stage[ch.stage];
    CU(c, cudaStreamWaitEvent(s, st.uploaded, 0));
    TileParams& p = ch.p;
    p = TileParams{};
    p.data = st.text + 16;
    p.tiles = tl->tiles[ch.stage];
    p.n_tiles = (uint32_t)(ch.hi - ch.lo);
    p.n = ch.e1 - ch.e0;
    p.tile_bad = tl->tile_bad; p.entry_off = tl->entry_off; p.entry_tile = tl->entry_tile; p.te_len = tl->te_len;
    p.leaf_index = tl->leaf_index; p.leaf_data_off = tl->leaf_data_off; p.first_stop = tl->first_stop; p.leaf_hash = tl->leaf_hash;
    FeParams& q = p.fe;
    q.n = p.n;
    q.decoded = st.text + 16;
    q.entry_status = f->entry_status; q.entry_type = f->entry_type; q.timestamp = f->timestamp; q.leaf_len_out = f->leaf_len_out;
    q.leaf_abs = f->leaf_abs; q.chain_abs = f->chain_abs; q.chain_len = f->chain_len; q.tbs_abs = f->tbs_abs; q.tbs_len = f->tbs_len;
    q.issuer_idx = f->issuer_idx;
    ch.db = ctmr_dev_batch{};
    ch.dout = ctmr_dev_out{};
    ch.stopped = false;
    ch.missing.clear();
    CU(c, cudaEventRecord(f->ev0, s));
    if (p.n) {
        unsigned int stop = ~0u;
        CU(c, cudaMemsetAsync(tl->first_stop, 0xFF, 4, s));
        CU(c, cudaEventRecord(tl->ev_split0, s));
        CU(c, launch_tile_split(p, s));
        CU(c, cudaEventRecord(tl->ev_split1, s));
        CU(c, launch_tile_frame(p, s));
        CU(c, launch_tile_issuer(p, FpTable{tl->fp_dev, tl->fp_mask}, s));
        f->launches += 4;  // split, frame, tbs, issuer
        if (out->leaf_hash || !ch.fold.empty()) {
            CU(c, launch_tile_leaf_hash(p, s));
            ++f->launches;
        }
        CU(c, cudaMemcpyAsync(&stop, tl->first_stop, 4, cudaMemcpyDeviceToHost, s));
        CU(c, cudaStreamSynchronize(s));
        float split = 0.f;
        CU(c, cudaEventElapsedTime(&split, tl->ev_split0, tl->ev_split1));
        tl->split_ms += split;
        if (stop != ~0u) {  // nothing is resolved on a guess: tiles from `stop` on wait for the host to register their issuers
            const TileDesc& td = tl->h_tiles[ch.stage][stop];
            std::vector<uint32_t> idx(td.width);
            std::vector<uint64_t> at(td.width);
            CU(c, cudaMemcpyAsync(idx.data(), f->issuer_idx + td.first, td.width * 4ull, cudaMemcpyDeviceToHost, s));
            CU(c, cudaMemcpyAsync(at.data(), f->chain_abs + td.first, td.width * 8ull, cudaMemcpyDeviceToHost, s));
            CU(c, cudaStreamSynchronize(s));
            for (uint32_t j = 0; j < td.width; ++j) {
                if (idx[j] != CTMR_ISSUER_UNRESOLVED) continue;
                std::array<uint8_t, 32> fp;
                std::memcpy(fp.data(), b->data + td.data_off + (at[j] - td.staged_off), 32);  // the host's own copy of the tile
                ch.missing.push_back(fp);
            }
            std::sort(ch.missing.begin(), ch.missing.end());
            ch.missing.erase(std::unique(ch.missing.begin(), ch.missing.end()), ch.missing.end());
            ch.stopped = true;
            ch.cut(stop, td.first);
            tree_cut(tree_state, ch, [this](uint64_t t) { return (uint32_t)b->tile_width[t]; });
        }
        {  // the completed tiles' leaves into their trees; a bad tile has none
            const int rc = tree_fold(c, ch, tl->leaf_hash, f->entry_status, 1, CTMR_FE_BAD_TILE);
            if (rc) return rc;
        }
    }
    CU(c, cudaEventRecord(f->ev1, s));
    ctmr_dev_batch& db = ch.db;
    db.blob = p.data;
    db.blob_bytes = ch.bytes;
    db.offsets = f->leaf_abs;
    db.lens = f->leaf_len_out;
    db.n = p.n;
    db.issuer_idx = f->issuer_idx;
    db.now_unix_ns = b->now_unix_ns;
    ch.dout = f->out.dev_out(out->path.sha256 != nullptr, meta);
    return CTMR_OK;
}

// the front end's own outputs of a chunk, after the path's; waits for the chunk
int Tiles::copy_back(ctmr_ctx* c, const Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    TileState* tl = f->tl.get();
    cudaStream_t s = c->stream;
    const uint64_t lo = ch.e0, cnt = ch.e1 - ch.e0, nt = ch.hi - ch.lo;
    std::vector<uint8_t> bad(nt);
    if (cnt) {
        CU(c, d2h_rows(out->entry_status, f->entry_status, lo, cnt, s));
        CU(c, d2h_rows(out->entry_type, f->entry_type, lo, cnt, s));
        CU(c, d2h_rows(out->timestamp_ms, f->timestamp, lo, cnt, s));
        CU(c, d2h_rows(out->issuer, f->issuer_idx, lo, cnt, s));
        CU(c, d2h_rows(out->leaf_index, tl->leaf_index, lo, cnt, s));
        CU(c, d2h_rows(out->leaf_off, tl->leaf_data_off, lo, cnt, s));
        CU(c, d2h_rows(out->leaf_len, f->leaf_len_out, lo, cnt, s));
        CU(c, d2h_rows(out->leaf_hash, tl->leaf_hash, lo, cnt, s, 32));
        if (out->tile_status) CU(c, cudaMemcpyAsync(bad.data(), tl->tile_bad, nt, cudaMemcpyDeviceToHost, s));
    }
    CU(c, cudaStreamSynchronize(s));
    if (out->tile_status)
        for (uint64_t i = 0; i < nt; ++i) out->tile_status[ch.lo + i] = bad[i] ? CTMR_FE_BAD_TILE : CTMR_FE_OK;
    return CTMR_OK;
}

// the stop: the unknown fingerprints, and the call's result code
int Tiles::stop(ctmr_ctx* c, const Chunk& ch) const {
    out->n_missing = (uint32_t)std::min<size_t>(ch.missing.size(), out->missing_cap);
    for (uint32_t i = 0; i < out->n_missing; ++i) std::memcpy(out->missing_fp + 32ull * i, ch.missing[i].data(), 32);
    return fail(c, CTMR_E_UNKNOWN_ISSUER, "tile " + std::to_string(ch.hi) + " names a Chain[0] fingerprint that is not registered "
                                          "(ctmr_register_chain_certs, then call again from tiles_done)");
}

// ================================================================================================================
// whole get-entries bodies: the units of a chunk are bodies.  The JSON kernels (ctmr_json.cu) leave the entries' spans in
// the stage as Pages::upload puts them, escaped strings unescaped into the stage's spare half, and the rest is Pages'.
// A chunk's entries are counted on the device, so their positions are given out after the front halves (place).
//
// The tree forms (ctmr_process_raw_bodies_tree(s)): the entries of body b are log positions start[b], start[b] + 1, ...
// of its log, known only once the front half has counted them, and a log may answer short, so that the bodies of a
// pipelining client leave gaps or overlap.  The front half hashes the leaves and reads back each body's status and count
// with the chunk's entry count; place walks the round's bodies in member order against each tree's end (the call's tree
// state: member 0's `next`, and `stopped`) and leaves per body a window of the entries that fold; fold expands the
// windows into the chunk's order on the device (body_fold_order) and folds, on each member's stream.
// ================================================================================================================
struct Bodies {
    static constexpr const char* kTooLarge = "a single body exceeds the front end's staging budget";
    static constexpr bool kStageHoldsLeaves = false;
    const ctmr_body_batch* b;
    ctmr_body_out* bo;
    ctmr_raw_out* out;  // &bo->raw
    uint64_t done = 0;    // entries that take their indices after a failure: the sum of body_max
    uint64_t placed = 0;  // entries found so far (positions given out)
    bool meta = false;
    std::vector<uint64_t> tree_pos;  // tree calls: each tree's size at the start of the call, its first end
    TreeState* tree_state = nullptr;  // tree calls: the call's tree state, member 0's (process_members)
    const uint32_t* log = nullptr;    // tree calls: the log of each body (NULL: every body is tree 0's)
    const uint64_t* start = nullptr;  // tree calls: the log position of each body's first entry
    std::vector<uint8_t> stopped;     // tree calls: the trees whose fold has stopped for this call

    Bodies(const ctmr_body_batch* b_, ctmr_body_out* bo_) : b(b_), bo(bo_), out(bo_ ? &bo_->raw : nullptr) {}
    int check(ctmr_ctx* c, const TreeArgs* tree);
    uint64_t units() const { return b->n_bodies; }
    uint64_t q_max(const ctmr_ctx*) const { return ~0ull; }  // fit keeps a chunk inside the budgets
    int prepare(ctmr_ctx* c) const;
    int fit(ctmr_ctx* c, uint64_t lo, uint64_t max_bodies, uint64_t* hi_out) const;
    int upload(ctmr_ctx* c, Chunk& ch) const;
    int front(ctmr_ctx* c, Chunk& ch) const;
    int copy_back(ctmr_ctx* c, const Chunk& ch) const;
    void completed(uint64_t) const { bo->n_entries = placed; }
    int stop(ctmr_ctx*, const Chunk&) const { return CTMR_OK; }
    void place(ctmr_ctx** m, Chunk* cur, uint32_t W);
    int fold(ctmr_ctx* c, const Chunk& ch) const;
    uint64_t entries() const { return placed; }
    bool folds() const { return tree_state && tree_state->active; }
};

// the tree rules of a tree call, per log in batch order: starts that never decrease, a first body that starts at or
// below the tree's size, and starts whose requested entries do not wrap around 2^64
int body_tree_args(ctmr_ctx* c, const ctmr_body_batch* b, const TreeArgs* tree) {
    const uint64_t nb = b->n_bodies;
    if (tree->routed) {
        const int rc = tree_route_args(c, tree, nb);
        if (rc) return rc;
    }
    if (nb && !tree->start) return fail(c, CTMR_E_INVALID, "trees: null body starts");
    std::vector<uint64_t> prev(tree->n, 0);
    std::vector<uint8_t> seen(tree->n, 0);
    for (uint64_t i = 0; i < nb; ++i) {
        const uint32_t l = tree->routed ? tree->log[i] : 0;
        if (l == CTMR_NO_TREE) continue;
        const uint64_t s = tree->start[i];
        if (s > ~0ull - b->body_max[i]) return fail(c, CTMR_E_INVALID, "trees: a body's start + its requested entries wraps around 2^64");
        if (!seen[l] && s > tree->trees[l].size) return fail(c, CTMR_E_INVALID, "trees: a log's first body starts after its tree's size");
        if (seen[l] && s < prev[l]) return fail(c, CTMR_E_INVALID, "trees: a log's body starts decrease");
        seen[l] = 1;
        prev[l] = s;
    }
    return CTMR_OK;
}

int Bodies::check(ctmr_ctx* c, const TreeArgs* tree) {
    if (!b || !bo || (tree && !tree->routed && !tree->trees)) return fail(c, CTMR_E_INVALID, "bad argument");
    if (b->n_bodies && (!b->text || !b->body_off || !b->body_len || !b->body_max)) return fail(c, CTMR_E_INVALID, "null batch buffers");
    int rc = check_pem(c, &out->path);
    if (rc) return rc;
    uint64_t requested = 0;
    for (uint64_t i = 0; i < b->n_bodies; ++i) {
        if (b->body_off[i] > b->text_bytes || b->body_len[i] > b->text_bytes - b->body_off[i])
            return fail(c, CTMR_E_INVALID, "body outside the text buffer");
        requested += b->body_max[i];
    }
    if (tree) {
        rc = body_tree_args(c, b, tree);
        if (rc) return rc;
        log = tree->routed ? tree->log : nullptr;
        start = tree->start;
        tree_pos.resize(tree->n);
        for (uint32_t d = 0; d < tree->n; ++d) tree_pos[d] = tree->trees[d].size;
        stopped.assign(tree->n, 0);
    }
    done = requested;  // only a batch that passed every check takes indices
    bo->n_entries = 0;
    return CTMR_OK;
}

// the budgets, before any work: a body must fit a chunk on its own
int Bodies::prepare(ctmr_ctx* c) const {
    int rc = fe_prepare(c);
    if (rc == CTMR_OK) rc = bodies_ensure(c);
    if (rc == CTMR_OK && !tree_pos.empty()) rc = bodies_fold_ensure(c);
    if (rc) return rc;
    c->fe->bd->json_ms = 0.f;
    for (uint64_t i = 0; i < b->n_bodies; ++i)
        if (b->body_len[i] > c->fe->cap_text / 2 || b->body_max[i] > c->fe->cap_entries) return fail(c, CTMR_E_BATCH_TOO_LARGE, kTooLarge);
    return CTMR_OK;
}

// How many bodies starting at `lo` fit one chunk (at most max_bodies): half the character budget (the other half takes
// the unescaped strings), and at most cap_entries bodies and requested entries
int Bodies::fit(ctmr_ctx* c, uint64_t lo, uint64_t max_bodies, uint64_t* hi_out) const {
    FrontEnd* f = c->fe.get();
    uint64_t hi = lo, bytes = 0, slots = 0;
    while (hi < b->n_bodies && hi - lo < max_bodies && hi - lo < f->cap_entries && bytes + b->body_len[hi] <= f->cap_text / 2 &&
           slots + b->body_max[hi] <= f->cap_entries) {
        bytes += b->body_len[hi];
        slots += b->body_max[hi];
        ++hi;
    }
    *hi_out = hi;
    return CTMR_OK;
}

// bodies [lo, hi) into upload stage ch.stage, asynchronously on the copy stream: one copy when they lie in order, apart
// and close together in the caller's text, packed back to back otherwise
int Bodies::upload(ctmr_ctx* c, Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    BodyState* bd = f->bd.get();
    FeStage& st = f->stage[ch.stage];
    CU(c, cudaSetDevice(c->device));
    CU(c, cudaStreamWaitEvent(f->copy_stream, st.consumed, 0));
    ch.e0 = ch.e1 = 0;
    const uint64_t cnt = ch.hi - ch.lo;
    bool in_order = true;
    uint64_t bytes = 0, min_off = ~0ull, max_end = 0;
    for (uint64_t i = ch.lo; i < ch.hi; ++i) {
        if (i > ch.lo && b->body_off[i] < b->body_off[i - 1] + b->body_len[i - 1]) in_order = false;
        bytes += b->body_len[i];
        min_off = std::min(min_off, b->body_off[i]);
        max_end = std::max(max_end, b->body_off[i] + b->body_len[i]);
    }
    const bool one_copy = cnt && in_order && max_end - min_off <= f->cap_text / 2;
    BodyDesc* h = bd->h_desc[ch.stage];
    uint64_t w = 0;
    uint32_t slot = 0;
    if (!one_copy) st.pack.resize(bytes);
    for (uint64_t i = 0; i < cnt; ++i) {
        const uint64_t k = ch.lo + i;
        BodyDesc& d = h[i];
        d.text_off = b->body_off[k];
        d.len = b->body_len[k];
        d.max = b->body_max[k];
        d.slot0 = slot;
        d.pad = 0;
        slot += d.max;
        if (one_copy) {
            d.staged_off = b->body_off[k] - min_off;
        } else {
            d.staged_off = w;
            std::memcpy(st.pack.data() + w, b->text + b->body_off[k], d.len);
            w += d.len;
        }
    }
    ch.bytes = one_copy ? max_end - min_off : w;
    if (ch.bytes)
        CU(c, cudaMemcpyAsync(st.text + 16, one_copy ? b->text + min_off : st.pack.data(), ch.bytes, cudaMemcpyHostToDevice, f->copy_stream));
    if (cnt) CU(c, cudaMemcpyAsync(bd->desc[ch.stage], h, cnt * sizeof(BodyDesc), cudaMemcpyHostToDevice, f->copy_stream));
    CU(c, cudaEventRecord(st.uploaded, f->copy_stream));
    return CTMR_OK;
}

// JSON kernels, one read-back of the entry count (a sync of its own: fe_decode's grid depends on it; a tree call reads
// each body's status and count with it), then what Pages runs on its spans; a tree call then hashes the leaves, which
// fold once place has given out their positions
int Bodies::front(ctmr_ctx* c, Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    BodyState* bd = f->bd.get();
    cudaStream_t s = c->stream;
    CU(c, cudaSetDevice(c->device));
    FeStage& st = f->stage[ch.stage];
    CU(c, cudaStreamWaitEvent(s, st.uploaded, 0));
    CU(c, cudaEventRecord(f->ev0, s));
    const uint64_t nb = ch.hi - ch.lo;
    uint64_t sparse = 0;
    for (uint64_t i = 0; i < nb; ++i) sparse += bd->h_desc[ch.stage][i].max;
    BodyParams p{};
    p.text = st.text + 16;
    p.spare = f->cap_text / 2;
    p.bodies = bd->desc[ch.stage];
    p.n_bodies = (uint32_t)nb;
    p.starts = bd->starts; p.trans = bd->trans; p.carry = bd->carry; p.masks = bd->masks; p.stack = bd->stack;
    p.body_status = bd->body_status; p.body_count = bd->body_count; p.body_base = bd->body_base;
    for (int k = 0; k < 2; ++k) {
        p.s_off[k] = bd->s_off[k]; p.s_len[k] = bd->s_len[k]; p.abs_off[k] = bd->abs_off[k]; p.raw_len[k] = bd->raw_len[k];
    }
    p.off[0] = st.leaf_off; p.len[0] = st.leaf_len; p.off[1] = st.extra_off; p.len[1] = st.extra_len;
    p.s_esc = bd->s_esc; p.esc = bd->esc;
    uint32_t count = 0;
    CU(c, cudaEventRecord(bd->ev_json0, s));
    uint32_t launches = 0;
    CU(c, launch_json_bodies(p, ch.bytes, sparse, bd->temp, bd->temp_bytes, s, &launches));
    CU(c, cudaEventRecord(bd->ev_json1, s));
    f->launches += launches;
    if (nb) CU(c, cudaMemcpyAsync(&count, bd->body_base + nb, 4, cudaMemcpyDeviceToHost, s));
    const bool tree = folds();
    if (nb && tree) {
        CU(c, cudaMemcpyAsync(bd->fold->h_status, bd->body_status, nb, cudaMemcpyDeviceToHost, s));
        CU(c, cudaMemcpyAsync(bd->fold->h_count, bd->body_count, nb * 4, cudaMemcpyDeviceToHost, s));
    }
    CU(c, cudaStreamSynchronize(s));
    float ms = 0.f;
    CU(c, cudaEventElapsedTime(&ms, bd->ev_json0, bd->ev_json1));
    bd->json_ms += ms;
    if (count > sparse) return fail(c, CTMR_E_CUDA, "bodies: more entries found than requested");
    const int rc = spans_front(c, ch, f->cap_text, count, b->now_unix_ns, &out->path, meta);
    if (rc || !tree || !count) return rc;
    CU(c, launch_raw_leaf_hash(ch.p.fe, f->tree->leaf, s));
    ++f->launches;
    CU(c, cudaEventRecord(f->ev1, s));
    return CTMR_OK;
}

// A tree call's round, after its front halves: the bodies of members 0..W-1 in member order against each tree's end
// (home->next) and stop.  Per body a window (BodyWindow) of the entries that fold; per member's chunk its trees
// (ch.fold), and whether its order must be built (it is the identity when one tree takes every entry of the chunk).
void Bodies::place(ctmr_ctx** m, Chunk* cur, uint32_t W) {  // positions: dense, in member order
    for (uint32_t r = 0; r < W; ++r) {
        cur[r].e0 = placed;
        placed += cur[r].db.n;
        cur[r].e1 = placed;
    }
    if (!folds()) return;
    TreeState* home = tree_state;
    std::vector<uint32_t>& cnt = home->count;
    std::vector<uint64_t> first;
    for (uint32_t r = 0; r < W; ++r) {
        Chunk& ch = cur[r];
        ch.fold.clear();
        ch.ordered = false;
        ch.listed = 0;
        const uint64_t nb = ch.hi - ch.lo;
        if (!nb) continue;
        BodyFoldState* bf = m[r]->fe->bd->fold.get();
        std::fill(cnt.begin(), cnt.end(), 0u);
        first = home->next;
        for (uint64_t i = 0; i < nb; ++i) {
            const uint64_t u = ch.lo + i;
            const uint32_t l = log ? log[u] : 0;
            BodyWindow& w = bf->h_win[i];
            w = BodyWindow{0, 0, 0};
            if (l == CTMR_NO_TREE || stopped[l]) continue;
            const uint64_t end = home->next[l];
            if (bf->h_status[i] != CTMR_BODY_OK || start[u] > end) {  // positions unknown, or a gap: the fold stops at end
                stopped[l] = 1;
                continue;
            }
            const uint32_t n = bf->h_count[i];
            const uint32_t skip = (uint32_t)std::min<uint64_t>(n, end - start[u]);  // already in the tree
            w.first = skip;
            w.cnt = n - skip;
            cnt[l] += w.cnt;
            home->next[l] = std::max(end, start[u] + n);
        }
        uint32_t off = 0;
        for (uint32_t d = 0; d < home->n_trees; ++d) {
            if (!cnt[d]) continue;
            ch.fold.push_back(FoldTree{first[d], d, off, cnt[d], 0});
            const uint32_t c_d = cnt[d];
            cnt[d] = off;  // from here on: the tree's next slot in the order
            off += c_d;
        }
        ch.listed = off;
        ch.ordered = off && !(ch.fold.size() == 1 && off == ch.db.n);
        if (!ch.ordered) continue;
        for (uint64_t i = 0; i < nb; ++i) {
            BodyWindow& w = bf->h_win[i];
            if (!w.cnt) continue;
            const uint32_t l = log ? log[ch.lo + i] : 0;
            w.slot = cnt[l];
            cnt[l] += w.cnt;
        }
    }
}

// a member's chunk into its trees (member 0) or ranges (members 1..), on its stream: the order from the windows unless
// it is the identity, then the fold of the pages form
int Bodies::fold(ctmr_ctx* c, const Chunk& ch) const {
    if (ch.fold.empty()) return CTMR_OK;
    FrontEnd* f = c->fe.get();
    CU(c, cudaSetDevice(c->device));
    if (ch.ordered) {
        BodyFoldState* bf = f->bd->fold.get();
        const uint64_t nb = ch.hi - ch.lo;
        CU(c, cudaMemcpyAsync(bf->win, bf->h_win, nb * sizeof(BodyWindow), cudaMemcpyHostToDevice, c->stream));
        CU(c, launch_body_fold_order(bf->win, (uint32_t)nb, f->bd->body_base, f->tree->order[ch.stage], c->stream));
        ++f->launches;
    }
    const int rc = tree_fold(c, ch, f->tree->leaf, f->str_bad, 2, 1);
    if (rc) return rc;
    CU(c, cudaEventRecord(f->ev1, c->stream));  // the fold is front-end time, as in the pages form
    return CTMR_OK;
}

int Bodies::copy_back(ctmr_ctx* c, const Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    BodyState* bd = f->bd.get();
    cudaStream_t s = c->stream;
    int rc = raw_copy_back(c, ch, out);
    if (rc) return rc;
    const uint64_t lo = ch.e0, cnt = ch.e1 - ch.e0, nb = ch.hi - ch.lo;
    if (cnt) {
        CU(c, d2h_rows(bo->leaf_input_off, bd->abs_off[0], lo, cnt, s));
        CU(c, d2h_rows(bo->leaf_input_len, bd->raw_len[0], lo, cnt, s));
        CU(c, d2h_rows(bo->extra_data_off, bd->abs_off[1], lo, cnt, s));
        CU(c, d2h_rows(bo->extra_data_len, bd->raw_len[1], lo, cnt, s));
        CU(c, d2h_rows(bo->escaped, bd->esc, lo, cnt, s));
    }
    std::vector<uint8_t> status(nb);
    std::vector<uint32_t> count(nb), base(nb);
    if (nb) {
        CU(c, cudaMemcpyAsync(status.data(), bd->body_status, nb, cudaMemcpyDeviceToHost, s));
        CU(c, cudaMemcpyAsync(count.data(), bd->body_count, nb * 4, cudaMemcpyDeviceToHost, s));
        CU(c, cudaMemcpyAsync(base.data(), bd->body_base, nb * 4, cudaMemcpyDeviceToHost, s));
    }
    CU(c, cudaStreamSynchronize(s));
    for (uint64_t i = 0; i < nb; ++i) {
        if (bo->body_status) bo->body_status[ch.lo + i] = status[i];
        if (bo->body_entries) bo->body_entries[ch.lo + i] = count[i];
        if (bo->body_first) bo->body_first[ch.lo + i] = ch.e0 + base[i];
    }
    return CTMR_OK;
}

// ================================================================================================================
// the driver
// ================================================================================================================

// fn(r) for every member: in member order, or with `threads` on one thread each (the halves of a chunk wait on the host:
// issuer round trips, D2H), in order if threads cannot be had.  Returns the error of the first member in member order
// that failed, and names it in *failed.  No exception leaves this function (C ABI).
template <class F>
int for_each_member(ctmr_ctx** m, uint32_t W, bool threads, ctmr_ctx** failed, F fn) {
    std::vector<int> rcs(W, CTMR_OK);
    std::vector<std::thread> th;
    uint32_t started = 0;
    if (threads) {
        try {
            for (; started < W; ++started) th.emplace_back([&rcs, &fn, r = started] { rcs[r] = fn(r); });
        } catch (...) {
        }
        for (std::thread& t : th) t.join();
    }
    for (uint32_t r = started; r < W; ++r)
        if ((rcs[r] = fn(r)) != CTMR_OK) break;
    for (uint32_t r = 0; r < W; ++r)
        if (rcs[r]) {
            *failed = m[r];
            return rcs[r];
        }
    return CTMR_OK;
}

// Cuts the round that starts at unit `pos` and issues its uploads into stage `stage`.  One member takes the greedy chunk
// fit returns (an empty chunk at the end of the batch: a rank of a collective call runs its last rounds empty).  A group
// takes one chunk per member from ONE contiguous window (split_window), a chunk fitting when fit keeps all of it.
template <class Format>
int plan_round(ctmr_ctx** m, uint32_t W, const Format& fm, uint64_t pos, int stage, std::vector<Chunk>& ch, ctmr_ctx** failed) {
    const uint64_t total = fm.units();
    *failed = m[0];
    uint64_t q = 0;
    if (W == 1) {
        uint64_t hi = pos;
        if (pos < total) {
            const int rc = fm.fit(m[0], pos, ~0ull, &hi);
            if (rc) return rc;
            if (hi == pos) return fail(m[0], CTMR_E_BATCH_TOO_LARGE, Format::kTooLarge);
        }
        q = hi - pos;
    } else {
        const auto fits = [&](uint32_t r, uint64_t lo, uint64_t want, bool* ok) {
            uint64_t hi = 0;
            const int rc = fm.fit(m[r], lo, want - lo, &hi);
            if (rc) *failed = m[r];
            *ok = hi == want;
            return rc;
        };
        const uint64_t q0 = std::max<uint64_t>(1, std::min<uint64_t>(fm.q_max(m[0]), (total - pos + W - 1) / W));
        const int rc = split_window(total, pos, W, q0, fits, &q);
        if (rc) return rc;
        if (q == 0) return fail(m[0], CTMR_E_BATCH_TOO_LARGE, Format::kTooLarge);
    }
    ch.assign(W, Chunk{});
    for (uint32_t r = 0; r < W; ++r) {
        ch[r].lo = std::min(total, pos + r * q);
        ch[r].hi = std::min(total, pos + (r + 1) * q);
        ch[r].stage = stage;
        *failed = m[r];
        const int rc = fm.upload(m[r], ch[r]);
        if (rc) return rc;
    }
    return CTMR_OK;
}

// A member's device-resident chunk as its part of round `parity` (run_round).  Everything runs on the member's stream,
// so there is no chain: the back half waits for each round before the next is issued.
int fe_member(ctmr_ctx* c, const ctmr_dev_batch& db, const ctmr_dev_out& dout, int parity, RoundMember& x) {
    CU(c, cudaSetDevice(c->device));
    int rc = ensure_scratch(c, std::max<uint64_t>(db.n, 1));
    if (rc == CTMR_OK) rc = ensure_order(c, db.n);
    if (rc) return rc;
    x = RoundMember{};
    x.c = c;
    x.db = db;
    x.dout = dout;
    x.dout.keys = c->keys_scratch;
    x.slot_of = c->slot_scratch; x.pair_slot = c->pair_scratch; x.order = c->order_scratch; x.len_hist = c->len_hist;
    x.meta_slots = c->meta_scratch;
    x.map_stream = x.reduce_stream = c->stream;
    x.mapped = c->fe->out.mapped; x.reduced = c->fe->out.reduced; x.meta_done = c->fe->out.meta_done;
    // The members of an in-process group meet through their events; peer_barrier does nothing for them.  The ranks of a
    // collective call (one process per GPU) meet at these barriers, which the host pipeline's rounds use too: both
    // calls are synchronous, so while a front-end call runs no stage stream of any rank has a barrier queued, and
    // every rank passes each channel's epochs in the same order.
    x.ch_map = CH_STAGE_MAP + parity;
    x.ch_resolve = CH_STAGE_RESOLVE + parity;
    x.ch_meta = CH_STAGE_META + parity;
    return CTMR_OK;
}

// ---- one process per GPU (ctmr_peer_*): every front-end call on an attached ctx is collective -------------------------
// The ranks first agree, through the mailbox, on the number of rounds R, on whether the call computes string identities
// and on whether every rank's checks passed.  Then every rank runs R rounds of the key exchange over its own chunks (an
// empty chunk when it has none left, has stopped or has failed), and a last mailbox exchange tells every rank how many
// ranks stopped at an unknown Chain[0] fingerprint: they resume with another collective call.

// What the ranks of a collective call agreed on.
struct PeerCall {
    bool on = false;
    uint64_t E = 0;       // entries per rank and round in the index rule: the largest chunk any rank may cut
    uint64_t rounds = 0;  // R: the most chunks any rank has, at least 1
    uint64_t span = 0;    // R * world * E: the indices the call takes once agreed
};

// The agreement's payload (peer_word): the rank's chunk count, its E and whether it wants string identities.
constexpr uint64_t kAgreeMeta = 1ull << 62;
constexpr int kAgreeEShift = 40;  // E <= kStageEntries < 2^22 in bits 40..61, the chunk count below 2^40
static_assert(kStageEntries < (1ull << 22), "agreement word layout");

// the chunks of the whole batch, cut by fit before the agreement exactly as the upload loop cuts them
template <class Format>
int count_chunks(ctmr_ctx* c, const Format& fm, uint64_t* chunks) {
    for (uint64_t pos = 0, hi = 0; pos < fm.units(); pos = hi, ++*chunks) {
        const int rc = fm.fit(c, pos, ~0ull, &hi);
        if (rc) return rc;
        if (hi == pos) return fail(c, CTMR_E_BATCH_TOO_LARGE, Format::kTooLarge);
    }
    return CTMR_OK;
}

// The path over round k's chunks.  One ctx: ctmr_process_device on the ctx's stream, which overlaps the map and the
// reduce of a large chunk.  A group, or a rank of a collective call: one round of the key exchange, each member's chunk
// as its slice.
int run_path(ctmr_ctx** m, uint32_t W, uint64_t k, Chunk* cur, bool meta, const PeerCall& pc, ctmr_ctx** failed) {
    if (W == 1 && !pc.on) {
        *failed = m[0];
        return cur[0].db.n ? process_device(m[0], &cur[0].db, &cur[0].dout, m[0]->stream, false) : CTMR_OK;
    }
    const int parity = (int)(k % kParities);
    RoundMember rm[kMaxWorld];
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        const int rc = fe_member(m[r], cur[r].db, cur[r].dout, parity, rm[r]);
        if (rc) return rc;
    }
    return run_round(rm, W, parity, pc.on ? pc.E : m[0]->fe->cap_entries, meta, failed);
}

// after the path: x509 leaf failures, PEM, outputs to the host; waits for the chunk
template <class Format>
int back(ctmr_ctx* c, const Format& fm, const Chunk& ch, uint64_t* pem_base) {
    FrontEnd* f = c->fe.get();
    cudaStream_t s = c->stream;
    CU(c, cudaSetDevice(c->device));
    const uint64_t cnt = ch.e1 - ch.e0;
    const ctmr_out* po = &fm.out->path;
    if (cnt) {
        CU(c, launch_fe_finish(ch.p.fe, f->out.status, s));
        ++f->launches;
    }
    CU(c, cudaEventRecord(f->ev2, s));
    if (cnt && po->pem) {  // the new certificates' PEM, encoded from the DER in HBM
        const int rc = pem_chunk(c, f->pem, ch.p.fe.decoded, f->leaf_abs, f->leaf_len_out, f->out.was_unknown, cnt, po, ch.e0, pem_base, s);
        if (rc) return rc;
    }
    if (Format::kStageHoldsLeaves) CU(c, cudaEventRecord(f->stage[ch.stage].consumed, s));  // the leaves' last read is done
    if (cnt) {
        const int rc = copy_out(c, ch.dout, cnt, po, ch.e0, s);
        if (rc) return rc;
    }
    const int rc = fm.copy_back(c, ch);
    if (rc) return rc;
    float a = 0.f, d = 0.f;
    CU(c, cudaEventElapsedTime(&a, f->ev0, f->ev1));
    CU(c, cudaEventElapsedTime(&d, f->ev1, f->ev2));
    f->fe_ms += a;
    f->path_ms += d;
    return CTMR_OK;
}

// One front-end call on the members m[0..W): one ctx (W == 1), or the members of a group; on a ctx attached to peers
// (pc.on) this rank's part of a collective call.  The batch's entries take the global indices from *next_index on;
// tree: fold the entries into the trees too, written back when the call succeeds or stops (on a group member 0 holds
// the trees and folds its chunks into them; the others fold theirs into ranges, merged into the trees after each
// round's back halves, tree_merge).  A stop
// (tiles) ends the call after the round that meets it; on a collective call the rank runs its remaining rounds empty,
// and so does a rank whose front or back half fails.  On error *failed names the member that failed.
template <class Format>
int process_members(ctmr_ctx** m, uint32_t W, uint64_t* next_index, Format& fm, const TreeArgs* targs, PeerCall& pc,
                    ctmr_ctx** failed) {
    *failed = m[0];
    pc.on = W == 1 && peer_call(m[0]);
    if (pc.on) m[0]->fe_peer_stopped = 0;
    int rc = fm.check(m[0], targs);
    if (rc && !pc.on) return rc;
    // The entries take their indices once a chunk reaches the path; a call that fails before has changed no table.
    const uint64_t takes = fm.done;
    fm.done = 0;
    const uint64_t total = rc ? 0 : fm.units();
    const TreeArgs* tree = targs && targs->n ? targs : nullptr;  // a routed call of no tree folds nothing
    if (total == 0 && !tree && !pc.on) return CTMR_OK;
    const ctmr_out* po = rc ? nullptr : &fm.out->path;
    // everything the call builds on first use, before its first kernel, and on a collective call its chunks
    uint64_t chunks = 0;
    const auto setup = [&]() -> int {
        for (uint32_t r = 0; r < W; ++r) {
            *failed = m[r];
            int rc = fm.prepare(m[r]);
            const uint64_t E = rc ? 0 : m[r]->fe->cap_entries;
            if (rc == CTMR_OK && po->pem) rc = pem_ensure(m[r], m[r]->fe->pem, E, m[r]->fe->cap_decoded);
            if (rc == CTMR_OK && pc.on) rc = ensure_scratch(m[r], E);  // the rounds' scratch (fe_member)
            if (rc == CTMR_OK && pc.on) rc = ensure_order(m[r], E);
            if (rc == CTMR_OK && W == 1 && !pc.on) rc = ensure_device_path(m[r], E);  // ctmr_process_device
            if (rc == CTMR_OK && tree && r > 0) rc = tree_begin_ranges(m[r], tree->n);
            if (rc) return rc;
        }
        *failed = m[0];
        if (tree) {
            const int rc = tree_begin(m[0], tree, fm.tree_pos, W - 1);
            if (rc) return rc;
            fm.tree_state = m[0]->fe->tree.get();
        }
        return pc.on ? count_chunks(m[0], fm, &chunks) : CTMR_OK;
    };
    if (rc == CTMR_OK) rc = setup();
    const uint64_t world = m[0]->st.peer.world, rank = m[0]->st.peer.rank;
    if (pc.on) {  // every check of every rank is done and no table has changed: the ranks go on together, or all return
        // E <= the key-exchange region X: alloc_exchange sizes X to at least the stage size, the front end's entry budget
        const uint64_t mine = rc ? 0 : chunks | m[0]->fe->cap_entries << kAgreeEShift | (want_meta(po) ? kAgreeMeta : 0);
        uint64_t row[kMaxWorld] = {};
        rc = peer_agree(m[0], rc, mine, row, "", "collective call failed before any work");
        if (rc) return rc;
        bool meta = false;
        for (uint32_t r = 0; r < world; ++r) {
            pc.rounds = std::max<uint64_t>(pc.rounds, row[r] & ((1ull << kAgreeEShift) - 1));
            pc.E = std::max<uint64_t>(pc.E, (row[r] >> kAgreeEShift) & ((1ull << 22) - 1));
            meta |= (row[r] & kAgreeMeta) != 0;
        }
        pc.rounds = std::max<uint64_t>(pc.rounds, 1);  // at least one round: its barriers fence the next call's post
        pc.span = pc.rounds * world * pc.E;
        fm.meta = meta;
    } else {
        if (rc) return rc;
        fm.meta = want_meta(po);
        if (tree && total == 0) return tree_end(m[0], tree);
    }
    uint64_t pem_base = 0;
    std::vector<Chunk> ch[2];  // round k's chunks in ch[k & 1], uploaded into stage k & 1
    rc = plan_round(m, W, fm, 0, 0, ch[0], failed);
    if (rc) return rc;
    Chunk* cur = nullptr;
    Chunk held;          // the chunk that holds the stop
    uint32_t stop = W;   // the member whose chunk holds the stop
    int local = CTMR_OK;  // a collective call: this rank's error after the agreement, returned at the end of the call
    std::string local_err;
    const auto fail_locally = [&](int code) {
        local = code;
        local_err = m[0]->err;
    };
    for (uint64_t k = 0;; ++k) {
        cur = ch[k & 1].data();
        const uint64_t end = cur[W - 1].hi;
        const bool idle = stop < W || local;  // a rank that stopped or failed runs its remaining rounds empty
        const bool last = pc.on ? k + 1 >= pc.rounds : end >= total;
        if (!last) {  // the next round's uploads overlap this round's kernels and host round trips
            rc = plan_round(m, W, fm, idle ? total : end, (k + 1) & 1, ch[(k + 1) & 1], failed);
            if (rc) return rc;
        }
        if (idle) cur[0].cut(0, 0);
        // The front halves wait on the host (issuer identification round trips, the arena size): one thread per member,
        // so that the members' waits overlap instead of adding up.  Each thread touches its own ctx only; the issuer
        // registry they all resolve against is device memory reached with atomics.
        rc = for_each_member(m, W, W > 1, failed, [&](uint32_t r) { return fm.front(m[r], cur[r]); });
        const bool front_failed = rc != CTMR_OK;
        if (front_failed) {
            if (!pc.on) return rc;
            fail_locally(rc);
            cur[0].cut(0, 0);
            cur[0].stopped = false;
            cur[0].dout = m[0]->fe->out.dev_out(po->sha256 != nullptr, fm.meta);
        }
        fm.place(m, cur, W);
        if (tree) {  // bodies: the round's leaves into the trees, now that place has given out their log positions
            rc = for_each_member(m, W, false, failed, [&](uint32_t r) { return fm.fold(m[r], cur[r]); });
            if (rc) return rc;
        }
        for (uint32_t r = 0; r < W; ++r) {
            if (stop < W) {
                cur[r].cut(0, 0);  // after a stop in an earlier member: its entries must not touch the tables
            } else if (cur[r].stopped) {
                stop = r;
                held = cur[r];
            }
            cur[r].db.first_index = *next_index + (pc.on ? (k * world + rank) * pc.E : cur[r].e0);
        }
        fm.done = takes;
        rc = run_path(m, W, k, cur, fm.meta, pc, failed);
        if (rc) return rc;
        if (!front_failed) {
            // in entry order when there is PEM (the texts are appended in that order); otherwise each member writes its
            // own ranges of the outputs, and on a group the members' copies and waits overlap
            rc = for_each_member(m, W, W > 1 && !po->pem, failed, [&](uint32_t r) { return back(m[r], fm, cur[r], &pem_base); });
            if (rc && !pc.on) return rc;
            if (rc) fail_locally(rc);
            else if (!idle) fm.completed(stop < W ? held.hi : end);
        }
        if (tree && W > 1) {  // the other members' ranges into the trees, up to the member that stopped
            rc = tree_merge(m, stop < W ? stop + 1 : W, cur, failed);
            if (rc) return rc;
        }
        if (last || (!pc.on && stop < W)) break;
    }
    if (stop < W) fm.done = held.e1;
    if (po->pem) po->pem_off[fm.entries()] = pem_base;
    for (uint32_t r = 0; r < W && !local; ++r) {  // a table that filled up during the completed chunks is this call's error
        *failed = m[r];
        rc = ctmr_check_device(m[r], nullptr);
        if (rc && !pc.on) return rc;
        if (rc) fail_locally(rc);
    }
    *failed = m[0];
    if (tree && !local) {  // at a stop the completed tiles are in the tree: the resumed call continues from there
        rc = tree_end(m[0], tree);
        if (rc && !pc.on) return rc;
        if (rc) fail_locally(rc);
    }
    if (pc.on) {  // every rank learns how many ranks stopped: a resume loop calls again while any did
        uint64_t row[kMaxWorld] = {};
        rc = peer_mailbox(m[0], stop < W ? 1 : 0, row);
        if (rc) return rc;
        for (uint32_t r = 0; r < world; ++r) m[0]->fe_peer_stopped += row[r] != 0;
        rc = ctmr_check_device(m[0], nullptr);  // a barrier that timed out; the count above is then unreliable
        if (rc && !local) return rc;
        if (local) {
            m[0]->err = local_err;
            return local;
        }
    }
    if (stop == W) return CTMR_OK;
    *failed = m[stop];
    return fm.stop(m[stop], held);
}

// an upload of the NEXT chunk may still be reading the caller's text and an output copy may still be writing the caller's
// arrays: neither may outlive a failed call
void drain_frontend(ctmr_ctx* c) {
    if (!c || !c->fe) return;
    const cudaStream_t s[] = {c->fe->copy_stream, c->stream};
    drain_streams(c, s, 2);
}

// Every front-end entry point: the call on members m[0..W), then, also after a failure, the entries that took their
// indices are used up (a retry must not reuse them: its entries then read as known), the tree is the caller's again,
// and a failure drains every member and becomes the last error of the group g (if any).
template <class Format>
int front_end_call(ctmr_ctx** m, uint32_t W, uint64_t* next_index, Format fm, const TreeArgs* tree, ctmr_group* g) {
    ctmr_ctx* failed = nullptr;
    PeerCall pc;  // a collective call takes pc.span indices once the ranks agreed, whatever happens after
    int rc = note_call_start(m, W, *next_index);  // on each member's stream, which runs the path
    if (rc == CTMR_OK) rc = process_members(m, W, next_index, fm, tree, pc, &failed);
    *next_index += pc.on ? pc.span : rc == CTMR_OK ? fm.entries() : fm.done;
    for (uint32_t r = 0; r < W; ++r) {
        if (m[r]->fe && m[r]->fe->tree) {
            m[r]->fe->tree->active = false;
            m[r]->fe->tree->log = nullptr;
        }
        if (rc != CTMR_OK) drain_frontend(m[r]);
    }
    return rc != CTMR_OK ? group_fail(g, failed, rc) : rc;
}

// Fingerprints of chain certificates on the GPU, then: a fingerprint table slot for each new one (capacity first, so a
// certificate the table cannot take is never registered), the registry (ctmr_register_issuers), the slots written.
int register_chain_certs(ctmr_ctx* c, const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint32_t* dense_out, uint8_t* fp_out) {
    if (n && (!blob || !offsets || !dense_out)) return fail(c, CTMR_E_INVALID, "bad argument");
    CU(c, cudaSetDevice(c->device));
    int rc = frontend_ensure(c);
    if (rc == CTMR_OK) rc = tiles_ensure(c);
    if (rc || n == 0) return rc;
    TileState* tl = c->fe->tl.get();
    for (uint32_t k = 0; k < n; ++k)
        if (offsets[k + 1] < offsets[k]) return fail(c, CTMR_E_INVALID, "chain certificate offsets not monotonic");
    const uint64_t base = offsets[0], bytes = offsets[n] - base;
    std::vector<uint64_t> rel(n + 1);
    for (uint32_t k = 0; k <= n; ++k) rel[k] = offsets[k] - base;
    std::vector<uint8_t> fps(32ull * n);
    DevBuf<uint8_t> d_blob, d_fp;
    DevBuf<uint64_t> d_off;
    CU(c, alloc(d_blob, bytes + 64));
    CU(c, alloc(d_off, n + 1));
    CU(c, alloc(d_fp, 32ull * n));
    CU(c, cudaMemcpyAsync(d_blob, blob + base, bytes, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(d_off, rel.data(), (n + 1) * 8ull, cudaMemcpyHostToDevice, c->stream));
    CU(c, launch_fingerprints(d_blob, d_off, n, d_fp, c->stream));
    CU(c, cudaMemcpyAsync(fps.data(), d_fp, 32ull * n, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (fp_out) std::memcpy(fp_out, fps.data(), fps.size());
    std::vector<uint32_t> fresh;  // first position of each fingerprint the table does not hold yet
    std::unordered_map<std::string, uint32_t> seen;
    for (uint32_t k = 0; k < n; ++k) {
        std::string key(reinterpret_cast<const char*>(fps.data() + 32ull * k), 32);
        if (!tl->fp_memo.count(key) && seen.emplace(key, k).second) fresh.push_back(k);
    }
    if (fresh.empty()) {
        for (uint32_t k = 0; k < n; ++k) dense_out[k] = tl->fp_memo[std::string(reinterpret_cast<const char*>(fps.data() + 32ull * k), 32)];
        return CTMR_OK;
    }
    if (tl->fp_used + fresh.size() > 2ull * c->st.max_issuers)
        return fail(c, CTMR_E_TOO_MANY_ISSUERS, "more chain certificate fingerprints than the table holds (raise config.max_issuers)");
    std::vector<uint8_t> packed;
    std::vector<uint64_t> poff(1, 0);
    for (uint32_t k : fresh) {
        packed.insert(packed.end(), blob + offsets[k], blob + offsets[k + 1]);
        poff.push_back(packed.size());
    }
    std::vector<uint32_t> dense(fresh.size());
    rc = ctmr_register_issuers(c, packed.data(), poff.data(), (uint32_t)fresh.size(), dense.data());
    if (rc) return rc;
    for (size_t i = 0; i < fresh.size(); ++i) {
        FpSlot sl{};
        std::memcpy(sl.w, fps.data() + 32ull * fresh[i], 32);
        sl.idx = dense[i];
        sl.used = 1;
        uint64_t slot = ((((uint64_t)sl.w[1]) << 32) | sl.w[0]) & tl->fp_mask;
        while (tl->fp_host[slot].used) slot = (slot + 1) & tl->fp_mask;
        tl->fp_host[slot] = sl;
        ++tl->fp_used;
        tl->fp_memo.emplace(std::string(reinterpret_cast<const char*>(sl.w), 32), sl.idx);
        CU(c, cudaMemcpyAsync(tl->fp_dev + slot, &tl->fp_host[slot], sizeof sl, cudaMemcpyHostToDevice, c->stream));
    }
    CU(c, cudaStreamSynchronize(c->stream));
    for (uint32_t k = 0; k < n; ++k) dense_out[k] = tl->fp_memo[std::string(reinterpret_cast<const char*>(fps.data() + 32ull * k), 32)];
    return CTMR_OK;
}

}  // namespace

extern "C" {

int ctmr_process_raw(ctmr_ctx* c, const ctmr_raw_batch* b, ctmr_raw_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode == PEER_GROUP) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_process_raw");
    return front_end_call(&c, 1, &c->next_index, Pages(b, out), nullptr, nullptr);
}

int ctmr_group_process_raw(ctmr_group* g, const ctmr_raw_batch* b, ctmr_raw_out* out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Pages(b, out), nullptr, g);
}

int ctmr_process_tiles(ctmr_ctx* c, const ctmr_tile_batch* b, ctmr_tile_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode == PEER_GROUP) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_process_tiles");
    return front_end_call(&c, 1, &c->next_index, Tiles(b, out), nullptr, nullptr);
}

int ctmr_group_process_tiles(ctmr_group* g, const ctmr_tile_batch* b, ctmr_tile_out* out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Tiles(b, out), nullptr, g);
}

int ctmr_process_raw_bodies(ctmr_ctx* c, const ctmr_body_batch* b, ctmr_body_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode == PEER_GROUP) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_process_raw_bodies");
    return front_end_call(&c, 1, &c->next_index, Bodies(b, out), nullptr, nullptr);
}

int ctmr_group_process_raw_bodies(ctmr_group* g, const ctmr_body_batch* b, ctmr_body_out* out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Bodies(b, out), nullptr, g);
}

int ctmr_bodies_profile_last(ctmr_ctx* c, float* json_ms) {
    if (!c || !c->fe || !c->fe->bd) return fail(c, CTMR_E_INVALID, "no ctmr_process_raw_bodies call to report");
    if (json_ms) *json_ms = c->fe->bd->json_ms;
    return CTMR_OK;
}

int ctmr_process_raw_tree(ctmr_ctx* c, const ctmr_raw_batch* b, ctmr_raw_out* out, ctmr_tree* tree) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode == PEER_GROUP) return fail(c, CTMR_E_INVALID, "member of a group: the tree forms take one ctx");
    const TreeArgs t{tree, 1, nullptr, false};
    return front_end_call(&c, 1, &c->next_index, Pages(b, out), &t, nullptr);
}

int ctmr_process_tiles_tree(ctmr_ctx* c, const ctmr_tile_batch* b, ctmr_tile_out* out, ctmr_tree* tree) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode == PEER_GROUP) return fail(c, CTMR_E_INVALID, "member of a group: the tree forms take one ctx");
    const TreeArgs t{tree, 1, nullptr, false};
    return front_end_call(&c, 1, &c->next_index, Tiles(b, out), &t, nullptr);
}

int ctmr_process_raw_trees(ctmr_ctx* c, const ctmr_raw_batch* b, ctmr_raw_out* out, const uint32_t* entry_log, ctmr_tree* trees,
                           uint32_t n_trees) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode == PEER_GROUP) return fail(c, CTMR_E_INVALID, "member of a group: the tree forms take one ctx");
    const TreeArgs t{trees, n_trees, entry_log, true};
    return front_end_call(&c, 1, &c->next_index, Pages(b, out), &t, nullptr);
}

int ctmr_process_tiles_trees(ctmr_ctx* c, const ctmr_tile_batch* b, ctmr_tile_out* out, const uint32_t* tile_log, ctmr_tree* trees,
                             uint32_t n_trees) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode == PEER_GROUP) return fail(c, CTMR_E_INVALID, "member of a group: the tree forms take one ctx");
    const TreeArgs t{trees, n_trees, tile_log, true};
    return front_end_call(&c, 1, &c->next_index, Tiles(b, out), &t, nullptr);
}

int ctmr_group_process_raw_tree(ctmr_group* g, const ctmr_raw_batch* b, ctmr_raw_out* out, ctmr_tree* tree) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const TreeArgs t{tree, 1, nullptr, false};
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Pages(b, out), &t, g);
}

int ctmr_group_process_tiles_tree(ctmr_group* g, const ctmr_tile_batch* b, ctmr_tile_out* out, ctmr_tree* tree) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const TreeArgs t{tree, 1, nullptr, false};
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Tiles(b, out), &t, g);
}

int ctmr_group_process_raw_trees(ctmr_group* g, const ctmr_raw_batch* b, ctmr_raw_out* out, const uint32_t* entry_log, ctmr_tree* trees,
                                 uint32_t n_trees) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const TreeArgs t{trees, n_trees, entry_log, true};
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Pages(b, out), &t, g);
}

int ctmr_group_process_tiles_trees(ctmr_group* g, const ctmr_tile_batch* b, ctmr_tile_out* out, const uint32_t* tile_log,
                                   ctmr_tree* trees, uint32_t n_trees) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const TreeArgs t{trees, n_trees, tile_log, true};
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Tiles(b, out), &t, g);
}

int ctmr_process_raw_bodies_tree(ctmr_ctx* c, const ctmr_body_batch* b, ctmr_body_out* out, const uint64_t* body_start, ctmr_tree* tree) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode == PEER_GROUP) return fail(c, CTMR_E_INVALID, "member of a group: the tree forms take one ctx");
    const TreeArgs t{tree, 1, nullptr, false, body_start};
    return front_end_call(&c, 1, &c->next_index, Bodies(b, out), &t, nullptr);
}

int ctmr_process_raw_bodies_trees(ctmr_ctx* c, const ctmr_body_batch* b, ctmr_body_out* out, const uint32_t* body_log,
                                  const uint64_t* body_start, ctmr_tree* trees, uint32_t n_trees) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode == PEER_GROUP) return fail(c, CTMR_E_INVALID, "member of a group: the tree forms take one ctx");
    const TreeArgs t{trees, n_trees, body_log, true, body_start};
    return front_end_call(&c, 1, &c->next_index, Bodies(b, out), &t, nullptr);
}

int ctmr_group_process_raw_bodies_tree(ctmr_group* g, const ctmr_body_batch* b, ctmr_body_out* out, const uint64_t* body_start,
                                       ctmr_tree* tree) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const TreeArgs t{tree, 1, nullptr, false, body_start};
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Bodies(b, out), &t, g);
}

int ctmr_group_process_raw_bodies_trees(ctmr_group* g, const ctmr_body_batch* b, ctmr_body_out* out, const uint32_t* body_log,
                                        const uint64_t* body_start, ctmr_tree* trees, uint32_t n_trees) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    const TreeArgs t{trees, n_trees, body_log, true, body_start};
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Bodies(b, out), &t, g);
}

int ctmr_next_index(ctmr_ctx* c, uint64_t* next_index) {
    if (!c) return CTMR_E_INVALID;
    if (!next_index || c->group) return fail(c, CTMR_E_INVALID, "bad argument (a member of a group has no index of its own)");
    *next_index = c->next_index;
    return CTMR_OK;
}

int ctmr_peer_frontend_stopped(ctmr_ctx* c, uint32_t* ranks) {
    if (!c) return CTMR_E_INVALID;
    if (!ranks || !peer_call(c)) return fail(c, CTMR_E_INVALID, "not a ctx attached to peers (ctmr_peer_attach)");
    *ranks = c->fe_peer_stopped;
    return CTMR_OK;
}

int ctmr_tiles_profile_last(ctmr_ctx* c, float* split_ms) {
    if (!c || !c->fe || !c->fe->tl) return fail(c, CTMR_E_INVALID, "no ctmr_process_tiles call to report");
    if (split_ms) *split_ms = c->fe->tl->split_ms;
    return CTMR_OK;
}

int ctmr_register_chain_certs(ctmr_ctx* c, const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint32_t* dense_out, uint8_t* fp_out) {
    if (!c) return CTMR_E_INVALID;
    return register_chain_certs(c, blob, offsets, n, dense_out, fp_out);
}

int ctmr_group_register_chain_certs(ctmr_group* g, const uint8_t* blob, const uint64_t* offsets, uint32_t n, uint32_t* dense_out,
                                    uint8_t* fp_out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    for (ctmr_ctx* c : g->m) {  // every member's table, from the one registry: the same dense indices everywhere
        const int rc = register_chain_certs(c, blob, offsets, n, dense_out, fp_out);
        if (rc) {
            g->err = c->err;
            return rc;
        }
    }
    return CTMR_OK;
}

}  // extern "C"

namespace ctmr_host {

int tiles_ensure(ctmr_ctx* c) {
    FrontEnd* f = c->fe.get();
    if (f->tl) return CTMR_OK;
    std::unique_ptr<TileState> tl(new (std::nothrow) TileState());
    if (!tl) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    const uint64_t E = f->cap_entries;
    tl->fp_mask = pow2_at_least(4ull * c->st.max_issuers) - 1;
    tl->fp_host.assign(tl->fp_mask + 1, FpSlot{});
    for (int k = 0; k < 2; ++k) {
        CU(c, alloc(tl->tiles[k], E));
        CU(c, alloc(tl->h_tiles[k], E));
    }
    CU(c, alloc(tl->tile_bad, E));
    CU(c, alloc(tl->entry_off, E));
    CU(c, alloc(tl->leaf_index, E));
    CU(c, alloc(tl->leaf_data_off, E));
    CU(c, alloc(tl->entry_tile, E));
    CU(c, alloc(tl->te_len, E));
    CU(c, alloc(tl->first_stop, 4));
    CU(c, alloc(tl->leaf_hash, E * 32));
    CU(c, alloc(tl->fp_dev, tl->fp_mask + 1));
    CU(c, create(tl->ev_split0, cudaEventDefault));
    CU(c, create(tl->ev_split1, cudaEventDefault));
    CU(c, cudaMemsetAsync(tl->fp_dev, 0, (tl->fp_mask + 1) * sizeof(FpSlot), c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    f->tl = std::move(tl);
    return CTMR_OK;
}

int bodies_ensure(ctmr_ctx* c) {
    FrontEnd* f = c->fe.get();
    if (f->bd) return CTMR_OK;
    std::unique_ptr<BodyState> bd(new (std::nothrow) BodyState());
    if (!bd) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    const uint64_t E = f->cap_entries, blocks = (f->cap_text / 2 + 63) / 64 + 1;
    for (int k = 0; k < 2; ++k) {
        CU(c, alloc(bd->desc[k], E));
        CU(c, alloc(bd->h_desc[k], E));
        CU(c, alloc(bd->s_off[k], E));
        CU(c, alloc(bd->s_len[k], E));
        CU(c, alloc(bd->abs_off[k], E));
        CU(c, alloc(bd->raw_len[k], E));
    }
    CU(c, alloc(bd->starts, blocks + 1));
    CU(c, alloc(bd->trans, blocks));
    CU(c, alloc(bd->carry, blocks));
    CU(c, alloc(bd->masks, blocks));
    CU(c, alloc(bd->stack, blocks * 2 + 2));  // a bit per staged byte
    CU(c, alloc(bd->body_status, E));
    CU(c, alloc(bd->body_count, E + 1));
    CU(c, alloc(bd->body_base, E + 1));
    CU(c, alloc(bd->s_esc, E));
    CU(c, alloc(bd->esc, E));
    bd->temp_bytes = json_scan_temp_bytes(blocks, E);
    CU(c, alloc(bd->temp, bd->temp_bytes ? bd->temp_bytes : 16));
    CU(c, create(bd->ev_json0, cudaEventDefault));
    CU(c, create(bd->ev_json1, cudaEventDefault));
    f->bd = std::move(bd);
    return CTMR_OK;
}

int bodies_fold_ensure(ctmr_ctx* c) {
    BodyState* bd = c->fe->bd.get();
    if (bd->fold) return CTMR_OK;
    std::unique_ptr<BodyFoldState> bf(new (std::nothrow) BodyFoldState());
    if (!bf) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    const uint64_t E = c->fe->cap_entries;
    CU(c, alloc(bf->h_status, E));
    CU(c, alloc(bf->h_count, E));
    CU(c, alloc(bf->h_win, E));
    CU(c, alloc(bf->win, E));
    bd->fold = std::move(bf);
    return CTMR_OK;
}

int tiles_clear_fingerprints(ctmr_ctx* c) {
    TileState* tl = c->fe ? c->fe->tl.get() : nullptr;
    if (!tl) return CTMR_OK;
    std::fill(tl->fp_host.begin(), tl->fp_host.end(), FpSlot{});
    tl->fp_used = 0;
    tl->fp_memo.clear();
    CU(c, cudaMemsetAsync(tl->fp_dev, 0, (tl->fp_mask + 1) * sizeof(FpSlot), c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return CTMR_OK;
}

}  // namespace ctmr_host
