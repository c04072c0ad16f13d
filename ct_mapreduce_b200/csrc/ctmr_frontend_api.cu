// ctmr_frontend_api.cu -- the entry points of include/ctmr_frontend.h (SURVEY.md §8(f)-2): get-entries strings -> base64
// decode -> TLS framing -> Chain[0] identification -> the path (ctmr_process_raw); static-ct-api data tiles -> split ->
// framing -> Chain[0] by fingerprint -> the path (ctmr_process_tiles, ctmr_register_chain_certs).  Each runs on one GPU, on
// a group of GPUs driven by one process (ctmr_group_*), and on one GPU with the log's Merkle tree folded in
// (ctmr_process_*_tree).
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

    // keeps the first `units` units, which hold `entries` entries
    void cut(uint64_t units, uint64_t entries) {
        hi = lo + units;
        e1 = e0 + entries;
        p.n_tiles = (uint32_t)units;
        p.n = p.fe.n = db.n = entries;
    }
};

bool want_meta(const ctmr_out* o) { return o->first_issuer_dn || o->first_crldp || o->issuer_name_off || o->crldp_off; }

int check_pem(ctmr_ctx* c, const ctmr_out* o) {
    if ((o->pem != nullptr) != (o->pem_off != nullptr)) return fail(c, CTMR_E_INVALID, "pem and pem_off go together");
    return CTMR_OK;
}

// where the path writes a chunk's results: the front end's per-chunk buffers (sha256 and string identities when asked for)
ctmr_dev_out chunk_path_out(FrontEnd* f, const ctmr_out* po) {
    const uint64_t E = f->cap_entries;
    ctmr_dev_out dout{};
    dout.status = f->status;
    dout.sha256 = po->sha256 ? f->sha.get() : nullptr;
    dout.exp_hour = f->exp_hour;
    dout.serial_off = f->serial_off;
    dout.serial_len = f->serial_len;
    dout.was_unknown = f->was_unknown;
    dout.first_issuer_hour = f->first;
    if (want_meta(po)) {
        dout.issuer_name_off = f->spans;
        dout.issuer_name_len = f->spans + E;
        dout.crldp_off = f->spans + 2 * E;
        dout.crldp_len = f->spans + 3 * E;
        dout.first_issuer_dn = f->first_meta;
        dout.first_crldp = f->first_meta + E;
    }
    return dout;
}

// the front end's buffers on a member, and its counters of this call
int fe_prepare(ctmr_ctx* c) {
    CU(c, cudaSetDevice(c->device));
    const int rc = frontend_ensure(c);
    if (rc) return rc;
    c->fe->fe_ms = c->fe->path_ms = 0.f;
    c->fe->launches = 0;
    return CTMR_OK;
}

// D2H of a chunk's device rows [0, cnt) of `per` bytes each to rows [lo, lo + cnt) of the caller's `dst`, if it asked for them
#define CHUNK_D2H(dst, src, per) \
    if (dst) CU(c, cudaMemcpyAsync(reinterpret_cast<uint8_t*>(dst) + lo * (per), (src), cnt * (per), cudaMemcpyDeviceToHost, s))

// ---- the log's Merkle tree (ctmr_process_raw_tree, ctmr_process_tiles_tree) ----------------------------------------------
int tree_ensure(ctmr_ctx* c) {
    FrontEnd* f = c->fe.get();
    if (f->tree) return CTMR_OK;
    std::unique_ptr<TreeState> tr(new (std::nothrow) TreeState());
    if (!tr) return fail(c, CTMR_E_NOMEM, "host allocation failed");
    const uint64_t E = f->cap_entries;
    CU(c, alloc(tr->dev, 1));
    CU(c, alloc(tr->host, 1));
    CU(c, alloc(tr->leaf, E * 32));
    for (DevBuf<uint8_t>& lvl : tr->lvl) CU(c, alloc(lvl, (E / 2 + 2) * 32));
    f->tree = std::move(tr);
    return CTMR_OK;
}

// the caller's tree to the device for the whole call; the call's entries start at log position `base`
int tree_begin(ctmr_ctx* c, const ctmr_tree* tree, uint64_t base) {
    int rc = tree_ensure(c);
    if (rc) return rc;
    TreeState* tr = c->fe->tree.get();
    std::memcpy(&tr->host->t, tree, sizeof(ctmr_tree));
    tr->host->missing = ~0ull;
    CU(c, cudaMemcpyAsync(tr->dev, tr->host, sizeof(TreeDev), cudaMemcpyHostToDevice, c->stream));
    tr->base = base;
    tr->active = true;
    return CTMR_OK;
}

// folds entries [0, cnt) of a chunk, log positions first_pos.., into the tree (see FoldChunk)
int tree_fold(ctmr_ctx* c, const uint8_t* leaves, const uint8_t* flags, uint32_t stride, uint32_t match, uint64_t first_pos, uint64_t cnt) {
    TreeState* tr = c->fe->tree.get();
    const FoldChunk fc{tr->dev, leaves, flags, stride, match, first_pos, cnt};
    uint8_t* const lvl[2] = {tr->lvl[0], tr->lvl[1]};
    uint32_t launches = 0;
    CU(c, launch_tree_fold(fc, lvl, c->stream, &launches));
    c->fe->launches += launches;
    return CTMR_OK;
}

// the root, and the tree back to the caller
int tree_end(ctmr_ctx* c, ctmr_tree* tree) {
    TreeState* tr = c->fe->tree.get();
    CU(c, launch_tree_root(tr->dev, c->stream));
    CU(c, cudaMemcpyAsync(tr->host, tr->dev, sizeof(TreeDev), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    std::memcpy(tree, &tr->host->t, sizeof(ctmr_tree));
    return CTMR_OK;
}

bool tree_active(const FrontEnd* f) { return f->tree && f->tree->active; }

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

    Pages(const ctmr_raw_batch* b_, ctmr_raw_out* out_) : b(b_), out(out_), done(b_ ? b_->n : 0) {}
    int check(ctmr_ctx* c, const ctmr_tree* tree) const;
    uint64_t units() const { return b->n; }
    uint64_t q_max(const ctmr_ctx* c) const { return c->fe->cap_entries; }
    uint64_t tree_base(const ctmr_tree* tree) const { return tree->size; }
    int prepare(ctmr_ctx* c) const { return fe_prepare(c); }
    int fit(ctmr_ctx* c, uint64_t lo, uint64_t max_entries, uint64_t* hi_out) const;
    int upload(ctmr_ctx* c, Chunk& ch) const;
    int front(ctmr_ctx* c, Chunk& ch) const;
    int copy_back(ctmr_ctx* c, const Chunk& ch) const;
    void completed(uint64_t) const {}
    int stop(ctmr_ctx*, const Chunk&) const { return CTMR_OK; }  // a page chunk never stops
};

// tree: ctmr_process_raw_tree's rule as well
int Pages::check(ctmr_ctx* c, const ctmr_tree* tree) const {
    if (!b || !out) return fail(c, CTMR_E_INVALID, "bad argument");
    if (b->n && (!b->text || !b->leaf_input_off || !b->leaf_input_len || !b->extra_data_off || !b->extra_data_len))
        return fail(c, CTMR_E_INVALID, "null batch buffers");
    const int rc = check_pem(c, &out->path);
    if (rc) return rc;
    if (tree && b->n > ~0ull - tree->size) return fail(c, CTMR_E_INVALID, "tree size + entries wraps around 2^64");
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

// decode + frame + Chain[0] -> dense index of an uploaded chunk; leaves ch.db / ch.dout describing the device-resident batch
int Pages::front(ctmr_ctx* c, Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    cudaStream_t s = c->stream;
    CU(c, cudaSetDevice(c->device));
    FeStage& st = f->stage[ch.stage];
    const uint64_t cnt = ch.hi - ch.lo;
    CU(c, cudaStreamWaitEvent(s, st.uploaded, 0));
    FeParams& p = ch.p.fe;
    p = FeParams{};
    p.text = st.text + 16;
    p.text_bytes = ch.bytes;
    p.leaf_off = st.leaf_off; p.leaf_len = st.leaf_len; p.extra_off = st.extra_off; p.extra_len = st.extra_len;
    p.n = cnt;
    p.pad_size = f->pad_size; p.dec_off = f->dec_off; p.dec_len = f->dec_len; p.str_bad = f->str_bad; p.decoded = f->decoded;
    p.entry_status = f->entry_status; p.entry_type = f->entry_type; p.timestamp = f->timestamp; p.leaf_src = f->leaf_src;
    p.leaf_rel = f->leaf_rel; p.leaf_len_out = f->leaf_len_out; p.leaf_abs = f->leaf_abs; p.chain_abs = f->chain_abs;
    p.chain_len = f->chain_len; p.tbs_abs = f->tbs_abs; p.tbs_len = f->tbs_len; p.issuer_idx = f->issuer_idx;
    ch.db = ctmr_dev_batch{};
    ch.dout = ctmr_dev_out{};
    CU(c, cudaEventRecord(f->ev0, s));
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
        if (tree_active(f)) {  // the leaves of this chunk into the tree, while the arena still holds them
            CU(c, launch_raw_leaf_hash(p, f->tree->leaf, s));
            ++f->launches;
            const int rc = tree_fold(c, f->tree->leaf, f->str_bad, 2, 1, f->tree->base + ch.lo, cnt);
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
    db.now_unix_ns = b->now_unix_ns;
    ch.dout = chunk_path_out(f, &out->path);
    return CTMR_OK;
}

// the front end's own outputs of a chunk, after the path's; waits for the chunk
int Pages::copy_back(ctmr_ctx* c, const Chunk& ch) const {
    FrontEnd* f = c->fe.get();
    cudaStream_t s = c->stream;
    const uint64_t lo = ch.e0, cnt = ch.e1 - ch.e0;
    if (cnt) {
        CHUNK_D2H(out->entry_status, f->entry_status, 1);
        CHUNK_D2H(out->entry_type, f->entry_type, 1);
        CHUNK_D2H(out->timestamp_ms, f->timestamp, 8);
        CHUNK_D2H(out->issuer, f->issuer_idx, 4);
        CHUNK_D2H(out->leaf_src, f->leaf_src, 1);
        CHUNK_D2H(out->leaf_off, f->leaf_rel, 4);
        CHUNK_D2H(out->leaf_len, f->leaf_len_out, 4);
    }
    CU(c, cudaStreamSynchronize(s));
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
    std::vector<uint64_t> ent;  // entries before each tile: ent[t] = sum of widths of tiles [0, t)

    Tiles(const ctmr_tile_batch* b_, ctmr_tile_out* out_) : b(b_), out(out_) {}
    int check(ctmr_ctx* c, const ctmr_tree* tree);
    uint64_t units() const { return b->n_tiles; }
    uint64_t q_max(const ctmr_ctx*) const { return ~0ull; }  // fit keeps a chunk inside the entry budget
    uint64_t tree_base(const ctmr_tree*) const { return b->n_tiles ? 256 * b->tile_index[0] : 0; }
    int prepare(ctmr_ctx* c) const;
    int fit(ctmr_ctx* c, uint64_t lo, uint64_t max_tiles, uint64_t* hi_out) const;
    int upload(ctmr_ctx* c, Chunk& ch) const;
    int front(ctmr_ctx* c, Chunk& ch) const;
    int copy_back(ctmr_ctx* c, const Chunk& ch) const;
    void completed(uint64_t tiles) const { out->tiles_done = tiles; }
    int stop(ctmr_ctx* c, const Chunk& ch) const;
};

// ctmr_process_tiles_tree's rules for the tiles of one log, checked before any work like the widths and spans
int tree_tile_args(ctmr_ctx* c, const ctmr_tile_batch* b, const ctmr_tree* tree, uint64_t n) {
    if (b->n_tiles == 0) return CTMR_OK;
    if (b->tile_index[0] > (~0ull - n) >> 8) return fail(c, CTMR_E_INVALID, "tree: the batch's last leaf index does not fit 64 bits");
    for (uint64_t t = 0; t + 1 < b->n_tiles; ++t) {
        if (b->tile_index[t + 1] != b->tile_index[t] + 1) return fail(c, CTMR_E_INVALID, "tree: tiles are not consecutive");
        if (b->tile_width[t] != 256) return fail(c, CTMR_E_INVALID, "tree: a partial tile that is not the last");
    }
    const uint64_t first = 256 * b->tile_index[0];
    if (tree->size < first || tree->size > first + b->tile_width[0])
        return fail(c, CTMR_E_INVALID, "tree: size is not inside the batch's first tile");
    return CTMR_OK;
}

// validates widths and spans (and with a tree its rules), fills ent
int Tiles::check(ctmr_ctx* c, const ctmr_tree* tree) {
    if (!b || !out) return fail(c, CTMR_E_INVALID, "bad argument");
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
        rc = tree_tile_args(c, b, tree, ent[b->n_tiles]);
        if (rc) return rc;
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
        if (out->leaf_hash || tree_active(f)) {
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
        }
        if (p.n && tree_active(f)) {  // the completed tiles' leaves into the tree; a bad tile has none
            const int rc = tree_fold(c, tl->leaf_hash, f->entry_status, 1, CTMR_FE_BAD_TILE, f->tree->base + ch.e0, p.n);
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
    ch.dout = chunk_path_out(f, &out->path);
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
        CHUNK_D2H(out->entry_status, f->entry_status, 1);
        CHUNK_D2H(out->entry_type, f->entry_type, 1);
        CHUNK_D2H(out->timestamp_ms, f->timestamp, 8);
        CHUNK_D2H(out->issuer, f->issuer_idx, 4);
        CHUNK_D2H(out->leaf_index, tl->leaf_index, 8);
        CHUNK_D2H(out->leaf_off, tl->leaf_data_off, 8);
        CHUNK_D2H(out->leaf_len, f->leaf_len_out, 4);
        CHUNK_D2H(out->leaf_hash, tl->leaf_hash, 32);
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

#undef CHUNK_D2H

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
// fit returns.  A group takes one chunk per member from ONE contiguous window, q units each, q halved until every
// member's chunk fits.
template <class Format>
int plan_round(ctmr_ctx** m, uint32_t W, const Format& fm, uint64_t pos, int stage, std::vector<Chunk>& ch, ctmr_ctx** failed) {
    const uint64_t total = fm.units();
    *failed = m[0];
    uint64_t q = 0;
    if (W == 1) {
        uint64_t hi = 0;
        const int rc = fm.fit(m[0], pos, ~0ull, &hi);
        if (rc) return rc;
        if (hi == pos) return fail(m[0], CTMR_E_BATCH_TOO_LARGE, Format::kTooLarge);
        q = hi - pos;
    } else {
        q = std::max<uint64_t>(1, std::min<uint64_t>(fm.q_max(m[0]), (total - pos + W - 1) / W));
        for (;;) {
            bool fits = true;
            for (uint32_t r = 0; r < W && fits; ++r) {
                const uint64_t lo = std::min(total, pos + r * q), want = std::min(total, pos + (r + 1) * q);
                uint64_t hi = 0;
                const int rc = fm.fit(m[r], lo, want - lo, &hi);
                if (rc) {
                    *failed = m[r];
                    return rc;
                }
                fits = hi == want;
            }
            if (fits) break;
            if (q == 1) return fail(m[0], CTMR_E_BATCH_TOO_LARGE, Format::kTooLarge);
            q = (q + 1) / 2;
        }
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
    x.mapped = c->fe->mapped; x.reduced = c->fe->reduced; x.meta_done = c->fe->meta_done;
    // the members of an in-process group meet through their events; peer_barrier does nothing for them
    x.ch_map = CH_STAGE_MAP + parity;
    x.ch_resolve = CH_STAGE_RESOLVE + parity;
    x.ch_meta = CH_STAGE_META + parity;
    return CTMR_OK;
}

// The path over round k's chunks.  One member: ctmr_process_device on the ctx's stream, which overlaps the map and the
// reduce of a large chunk.  A group: one round of the key exchange, each member's chunk as its slice.
int run_path(ctmr_ctx** m, uint32_t W, int k, Chunk* cur, bool meta, ctmr_ctx** failed) {
    if (W == 1) {
        *failed = m[0];
        return cur[0].db.n ? ctmr_process_device(m[0], &cur[0].db, &cur[0].dout, m[0]->stream) : CTMR_OK;
    }
    const int parity = k % (int)kParities;
    RoundMember rm[kMaxWorld];
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        const int rc = fe_member(m[r], cur[r].db, cur[r].dout, parity, rm[r]);
        if (rc) return rc;
    }
    return run_round(rm, W, parity, m[0]->fe->cap_entries, meta, failed);
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
        CU(c, launch_fe_finish(ch.p.fe, f->status, s));
        ++f->launches;
    }
    CU(c, cudaEventRecord(f->ev2, s));
    if (cnt && po->pem) {  // the new certificates' PEM, encoded from the DER in HBM
        const int rc = pem_chunk(c, f->pem, ch.p.fe.decoded, f->leaf_abs, f->leaf_len_out, f->was_unknown, cnt, po, ch.e0, pem_base, s);
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

// One front-end call on the members m[0..W): one ctx (W == 1), or the members of a group.  The batch's entries take the
// global indices from *next_index on; tree (one member only): fold the entries into it too, written back when the call
// succeeds or stops.  A stop (tiles) ends the call after the round that meets it.  On error *failed names the member
// that failed.
template <class Format>
int process_members(ctmr_ctx** m, uint32_t W, uint64_t* next_index, Format& fm, ctmr_tree* tree, ctmr_ctx** failed) {
    *failed = m[0];
    int rc = fm.check(m[0], tree);
    if (rc) return rc;
    // The entries take their indices once a chunk reaches the path; a call that fails before has changed no table.
    const uint64_t takes = fm.done;
    fm.done = 0;
    const uint64_t total = fm.units();
    if (total == 0 && !tree) return CTMR_OK;
    const ctmr_out* po = &fm.out->path;
    // everything the call builds on first use, before its first kernel
    for (uint32_t r = 0; r < W; ++r) {
        *failed = m[r];
        rc = fm.prepare(m[r]);
        if (rc == CTMR_OK && po->pem) rc = pem_ensure(m[r], m[r]->fe->pem, m[r]->fe->cap_entries, m[r]->fe->cap_decoded);
        if (rc == CTMR_OK && W == 1) rc = ensure_device_path(m[r], m[r]->fe->cap_entries);  // ctmr_process_device
        if (rc) return rc;
    }
    *failed = m[0];
    if (tree) {
        rc = tree_begin(m[0], tree, fm.tree_base(tree));
        if (rc) return rc;
        if (total == 0) return tree_end(m[0], tree);
    }
    uint64_t pem_base = 0;
    std::vector<Chunk> ch[2];  // round k's chunks in ch[k & 1], uploaded into stage k & 1
    rc = plan_round(m, W, fm, 0, 0, ch[0], failed);
    if (rc) return rc;
    Chunk* cur = nullptr;
    uint32_t stop = W;  // the member whose chunk holds the stop
    for (int k = 0;; ++k) {
        cur = ch[k & 1].data();
        const uint64_t end = cur[W - 1].hi;
        if (end < total) {  // the next round's uploads overlap this round's kernels and host round trips
            rc = plan_round(m, W, fm, end, (k + 1) & 1, ch[(k + 1) & 1], failed);
            if (rc) return rc;
        }
        // The front halves wait on the host (issuer identification round trips, the arena size): one thread per member,
        // so that the members' waits overlap instead of adding up.  Each thread touches its own ctx only; the issuer
        // registry they all resolve against is device memory reached with atomics.
        rc = for_each_member(m, W, W > 1, failed, [&](uint32_t r) { return fm.front(m[r], cur[r]); });
        if (rc) return rc;
        for (uint32_t r = 0; r < W; ++r) {
            if (stop < W) cur[r].cut(0, 0);  // after a stop in an earlier member: its entries must not touch the tables
            else if (cur[r].stopped) stop = r;
            cur[r].db.first_index = *next_index + cur[r].e0;
        }
        fm.done = takes;
        rc = run_path(m, W, k, cur, want_meta(po), failed);
        if (rc) return rc;
        // in entry order when there is PEM (the texts are appended in that order); otherwise each member writes its own
        // ranges of the outputs, and on a group the members' copies and waits overlap
        rc = for_each_member(m, W, W > 1 && !po->pem, failed, [&](uint32_t r) { return back(m[r], fm, cur[r], &pem_base); });
        if (rc) return rc;
        fm.completed(stop < W ? cur[stop].hi : end);
        if (stop < W || end >= total) break;
    }
    if (stop < W) fm.done = cur[stop].e1;
    if (po->pem) po->pem_off[fm.done] = pem_base;
    for (uint32_t r = 0; r < W; ++r) {  // a table that filled up during the completed chunks is this call's error
        *failed = m[r];
        rc = ctmr_check_device(m[r], nullptr);
        if (rc) return rc;
    }
    *failed = m[0];
    if (tree) {  // at a stop the completed tiles are in the tree: the resumed call continues from there
        rc = tree_end(m[0], tree);
        if (rc) return rc;
    }
    if (stop == W) return CTMR_OK;
    *failed = m[stop];
    return fm.stop(m[stop], cur[stop]);
}

// an upload of the NEXT chunk may still be reading the caller's text and an output copy may still be writing the caller's
// arrays: neither may outlive a failed call
void drain_frontend(ctmr_ctx* c) {
    if (!c || !c->fe) return;
    const std::string keep = c->err;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->fe->copy_stream);
    cudaStreamSynchronize(c->stream);
    c->err = keep;
}

// Every front-end entry point: the call on members m[0..W), then, also after a failure, the entries that took their
// indices are used up (a retry must not reuse them: its entries then read as known), the tree is the caller's again,
// and a failure drains every member and becomes the last error of the group g (if any).
template <class Format>
int front_end_call(ctmr_ctx** m, uint32_t W, uint64_t* next_index, Format fm, ctmr_tree* tree, ctmr_group* g) {
    ctmr_ctx* failed = nullptr;
    const int rc = process_members(m, W, next_index, fm, tree, &failed);
    *next_index += fm.done;
    for (uint32_t r = 0; r < W; ++r) {
        if (m[r]->fe && m[r]->fe->tree) m[r]->fe->tree->active = false;
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
    if (c->group || c->peer_mode != PEER_NONE) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_process_raw");
    return front_end_call(&c, 1, &c->next_index, Pages(b, out), nullptr, nullptr);
}

int ctmr_group_process_raw(ctmr_group* g, const ctmr_raw_batch* b, ctmr_raw_out* out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Pages(b, out), nullptr, g);
}

int ctmr_process_tiles(ctmr_ctx* c, const ctmr_tile_batch* b, ctmr_tile_out* out) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode != PEER_NONE) return fail(c, CTMR_E_INVALID, "member of a group: use ctmr_group_process_tiles");
    return front_end_call(&c, 1, &c->next_index, Tiles(b, out), nullptr, nullptr);
}

int ctmr_group_process_tiles(ctmr_group* g, const ctmr_tile_batch* b, ctmr_tile_out* out) {
    if (!g || g->m.empty()) return CTMR_E_INVALID;
    return front_end_call(g->m.data(), (uint32_t)g->m.size(), &g->next_index, Tiles(b, out), nullptr, g);
}

int ctmr_process_raw_tree(ctmr_ctx* c, const ctmr_raw_batch* b, ctmr_raw_out* out, ctmr_tree* tree) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode != PEER_NONE) return fail(c, CTMR_E_INVALID, "member of a group: the tree forms take one ctx");
    if (!tree) return fail(c, CTMR_E_INVALID, "bad argument");
    return front_end_call(&c, 1, &c->next_index, Pages(b, out), tree, nullptr);
}

int ctmr_process_tiles_tree(ctmr_ctx* c, const ctmr_tile_batch* b, ctmr_tile_out* out, ctmr_tree* tree) {
    if (!c) return CTMR_E_INVALID;
    if (c->group || c->peer_mode != PEER_NONE) return fail(c, CTMR_E_INVALID, "member of a group: the tree forms take one ctx");
    if (!tree) return fail(c, CTMR_E_INVALID, "bad argument");
    return front_end_call(&c, 1, &c->next_index, Tiles(b, out), tree, nullptr);
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
