// ring_schedule.cu -- K_map's copy schedule (ring_chunk_copy / ring_step, ctmr_common.cuh) run on the host.
//
// A simulated lane ring records, for every byte, which source byte the last copy put there.  Copies land the moment
// they are issued -- the earliest an asynchronous copy can land, so a copy that overwrites bytes the walker or the hash
// still needs is caught every time instead of once in a while.  At every step the walker's bytes (from kWalkNeed
// before the chunk to its end) and the hash's 17-word reads (ring offsets as map_stream_kernel computes them) must
// hold the record's own bytes, for every misalignment m and every record length up to `max_len`.
//   ring_schedule <max_len>     prints "ok <records checked>" or the first failure, exit code 1
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../ct_mapreduce_b200/csrc/ctmr_common.cuh"
#include "../../ct_mapreduce_b200/csrc/ctmr_stream.cuh"

using ctmr::StreamCfg;

static bool check_record(uint32_t m, uint32_t L) {
    constexpr uint32_t CHUNK = StreamCfg::kChunk, RING = StreamCfg::kRing;
    std::vector<int64_t> ring(StreamCfg::kLaneBytes, -1);  // source byte offset held by each ring byte
    const uint32_t yend = L ? (m + L + 15u) >> 4 : 0u;
    const uint32_t ndata = (L + CHUNK - 1) / CHUNK;
    const uint32_t nb = (L >> 6) + 1u + ((L & 63u) >= 56u ? 1u : 0u);
    uint32_t nch = (nb + StreamCfg::kBlocksPerChunk - 1) / StreamCfg::kBlocksPerChunk;
    nch = nch > ndata ? nch : ndata;
    bool ok = true;
    auto fail = [&](const char* what, uint32_t c, uint32_t x) {
        if (ok) std::printf("FAIL m=%u L=%u step %u: %s reads record byte %u from a ring byte that does not hold it\n", m, L, c, what, x);
        ok = false;
    };
    auto copy = [&](uint32_t y0, uint32_t y1) {  // the kernel's addressing: one contiguous run, ring granule 0 mirrored
        if (y0 > y1) { std::printf("FAIL m=%u L=%u: copy range [%u, %u)\n", m, L, y0, y1); ok = false; return; }
        const uint32_t dst = (16u * y0) & (RING - 1u);
        if (y0 < y1 && dst == 0u)
            for (uint32_t b = 0; b < 16u; ++b) ring[RING + b] = 16 * (int64_t)y0 + b;
        for (uint32_t j = 0; j < 16u * (y1 - y0); ++j) {
            if (dst + j >= RING) { std::printf("FAIL m=%u L=%u: copy [%u, %u) crosses the ring's end\n", m, L, y0, y1); ok = false; return; }
            ring[dst + j] = 16 * (int64_t)y0 + j;
        }
    };
    const ctmr::RingCopy r0 = ctmr::ring_chunk_copy(0u, m, yend);
    copy(r0.y0, r0.y1);
    for (uint32_t c = 0; c < nch && ok; ++c) {
        auto walk = [&] {  // the walker resumes at most kWalkNeed bytes before the chunk and reads up to its end
            if (c >= ndata) return;
            const uint32_t lo = c * CHUNK > ctmr::kWalkNeed ? c * CHUNK - ctmr::kWalkNeed : 0u;
            const uint32_t hi = (c + 1u) * CHUNK < L ? (c + 1u) * CHUNK : L;
            for (uint32_t x = lo; x < hi; ++x)
                if (ring[(x + m) & (RING - 1u)] != (int64_t)(x + m)) fail("the walker", c, x);
        };
        auto hash = [&] {  // 17 words from ring offset ((c & 1) * CHUNK + m + 64 * bb) & ~3; bytes past L are padding
            for (uint32_t bb = 0; bb < (uint32_t)StreamCfg::kBlocksPerChunk; ++bb) {
                const uint32_t b = c * StreamCfg::kBlocksPerChunk + bb;
                if (b >= nb) break;
                const uint32_t w0 = ((c & 1u) * CHUNK + m + 64u * bb) & ~3u;
                if (w0 + 68u > (uint32_t)StreamCfg::kLaneBytes) { fail("the hash (past the mirror)", c, 64u * b); return; }
                for (uint32_t i = 0; i < 64u && 64u * b + i < L; ++i) {
                    const uint32_t x = 64u * b + i;
                    if (ring[w0 + (m & 3u) + i] != (int64_t)(x + m)) fail("the hash", c, x);
                }
            }
        };
        ctmr::ring_step(c, m, yend, walk, copy, hash);
    }
    return ok;
}

int main(int argc, char** argv) {
    const uint32_t max_len = argc > 1 ? (uint32_t)std::atoi(argv[1]) : 1200u;
    uint32_t n = 0;
    for (uint32_t m = 0; m < 16u; ++m)
        for (uint32_t L = 1; L <= max_len; ++L, ++n)
            if (!check_record(m, L)) return 1;
    std::printf("ok %u\n", n);
    return 0;
}
