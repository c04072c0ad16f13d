// kmap_split.cu -- experiments build of K_map for tools/kmap_split.py: the streaming kernel of ctmr_map.cu compiled
// under one of its timing policies (CTMR_KMAP_SKIP_WALK / CTMR_KMAP_SKIP_HASH on the command line), plus one entry
// point that runs the map half of a bench step with it.  Never part of libctmr.so.
#include <algorithm>
#include <cstring>

#include "../ct_mapreduce_b200/csrc/ctmr_map.cu"

struct kmap_split_args {
    const uint8_t* blob;
    uint64_t blob_bytes;
    const uint64_t* offsets;  // [n + 1]
    const uint32_t* issuer_idx;
    uint64_t n;
    uint8_t* status;
    uint8_t* sha256;
    int64_t* exp_hour;
    ctmr_key* keys;
    uint32_t* slot_of;
    uint32_t* order;
    unsigned int* len_hist;  // [rounds][256]
    ctmr::KnownSlot* table;
    uint64_t table_slots;  // power of two
    unsigned long long* status_counts;
    int* error_flag;
    int64_t now_sec;
    uint32_t rounds;
    uint32_t per_round;
    int32_t sm_count;
};

#define KS(x)                          \
    do {                               \
        cudaError_t e_ = (x);          \
        if (e_ != cudaSuccess) return (int)e_; \
    } while (0)

// `steps` steps, each the way ctmr_process_device issues its map half: the table emptied, then `rounds` K_map launches
// on two alternating streams, each behind its own length ordering.  *ms = mean time of the launches of a step (the
// table reset is outside the timed span, as it is outside K_map's span in the library).
extern "C" int kmap_split_run(const kmap_split_args* a, int steps, float* ms) {
    cudaStream_t user, sa[2];
    cudaEvent_t fork, join[2], t0, t1;
    KS(cudaStreamCreateWithFlags(&user, cudaStreamNonBlocking));
    for (auto& s : sa) KS(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    KS(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
    for (auto& e : join) KS(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    KS(cudaEventCreate(&t0));
    KS(cudaEventCreate(&t1));
    double total = 0;
    for (int it = 0; it < steps; ++it) {
        KS(cudaMemsetAsync(a->table, 0, a->table_slots * sizeof(ctmr::KnownSlot), user));
        KS(cudaEventRecord(t0, user));
        KS(cudaEventRecord(fork, user));
        for (auto& s : sa) KS(cudaStreamWaitEvent(s, fork, 0));
        for (uint32_t k = 0; k < a->rounds; ++k) {
            const uint64_t lo = std::min<uint64_t>(a->n, (uint64_t)a->per_round * k), hi = std::min<uint64_t>(a->n, (uint64_t)a->per_round * (k + 1));
            if (hi == lo) continue;
            ctmr::MapParams p;
            std::memset(&p, 0, sizeof p);
            p.blob = a->blob;
            p.blob_bytes = a->blob_bytes;
            p.offsets = a->offsets + lo;
            p.n = hi - lo;
            p.issuer_idx = a->issuer_idx + lo;
            p.first_index = lo;
            p.now_sec = a->now_sec;
            p.one = 1;
            p.status = a->status + lo;
            p.sha256 = a->sha256 + 32 * lo;
            p.exp_hour = a->exp_hour + lo;
            p.keys = a->keys + lo;
            p.status_counts = a->status_counts;
            p.filter.log_expired = 1;
            p.route.world = 1;
            p.table = a->table;
            p.table_mask = a->table_slots - 1;
            p.error_flag = a->error_flag;
            p.slot_of = a->slot_of + lo;
            p.order = a->order + lo;
            KS(ctmr::launch_len_order(p.offsets, nullptr, p.n, p.blob_bytes, a->len_hist + 256 * k, a->order + lo, a->sm_count, sa[k & 1]));
            KS(ctmr::launch_map(p, a->sm_count, sa[k & 1]));
        }
        for (int i = 0; i < 2; ++i) {
            KS(cudaEventRecord(join[i], sa[i]));
            KS(cudaStreamWaitEvent(user, join[i], 0));
        }
        KS(cudaEventRecord(t1, user));
        KS(cudaStreamSynchronize(user));
        float one = 0;
        KS(cudaEventElapsedTime(&one, t0, t1));
        total += one;
    }
    *ms = (float)(total / (steps > 0 ? steps : 1));
    KS(cudaEventDestroy(fork));
    for (auto& e : join) KS(cudaEventDestroy(e));
    KS(cudaEventDestroy(t0));
    KS(cudaEventDestroy(t1));
    KS(cudaStreamDestroy(user));
    for (auto& s : sa) KS(cudaStreamDestroy(s));
    return 0;
}
