// peer_word.cpp -- the mailbox word of a collective call's agreements (peer_word and its readers, ctmr_kernels.cuh) run
// on the host.  Prints "ok <checks>", or the first failed check and exit code 1.
#include <cstdio>
#include <cstdlib>

#include "../../ct_mapreduce_b200/csrc/ctmr_kernels.cuh"

using namespace ctmr;

static unsigned checks = 0;
#define CHECK(c)                                                                                     \
    do {                                                                                             \
        ++checks;                                                                                    \
        if (!(c)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); std::exit(1); }        \
    } while (0)

int main() {
    const int codes[] = {CTMR_E_INVALID,         CTMR_E_CUDA,         CTMR_E_NOMEM,          CTMR_E_TABLE_FULL,
                         CTMR_E_TOO_MANY_ISSUERS, CTMR_E_NO_DEVICE,    CTMR_E_BATCH_TOO_LARGE, CTMR_E_PAIR_TABLE_FULL,
                         CTMR_E_META_TABLE_FULL, CTMR_E_PEER_TIMEOUT, CTMR_E_PEER,          CTMR_E_UNKNOWN_ISSUER,
                         CTMR_E_PEER_FAILED};
    // payloads: the edges, every single bit below 63, and the front end's largest packing (chunks < 2^40 in bits 0..39,
    // E < 2^22 in bits 40..61, string identities in bit 62), which sets bits 0..62
    const uint64_t fe_max = ((1ull << 40) - 1) | ((1ull << 22) - 1) << 40 | 1ull << 62;
    CHECK(fe_max == kPeerWordFailed - 1);
    uint64_t payloads[64 + 5] = {0, 1, 0x5555555555555555ull, 0x2aaaaaaaaaaaaaaaull, fe_max};
    int np = 5;
    for (int b = 0; b < 63; ++b) payloads[np++] = 1ull << b;

    for (int k = 0; k < np; ++k) {  // a payload survives untouched and never reads as a failure
        const uint64_t w = peer_word(CTMR_OK, payloads[k]);
        CHECK(w == payloads[k]);
        CHECK(!peer_word_failed(w));
    }
    for (int rc : codes) {  // every error code: a failed word, whatever payload came with it, that gives the code back
        for (int k = 0; k < np; ++k) {
            const uint64_t w = peer_word(rc, payloads[k]);
            CHECK(w == (kPeerWordFailed | (uint32_t)(-rc)));
            CHECK(peer_word_failed(w));
            CHECK(peer_word_code(w) == rc);
        }
    }

    // the row verdict: the lowest rank of the world whose word failed, the world when none did
    uint64_t row[kMaxWorld] = {};
    for (uint32_t world = 1; world <= kMaxWorld; ++world) {
        for (uint32_t r = 0; r < kMaxWorld; ++r) row[r] = peer_word(CTMR_OK, fe_max - r);
        CHECK(peer_row_failed(row, world) == world);
        if (world < kMaxWorld) {  // a failed word past the world is not read
            row[world] = peer_word(CTMR_E_NOMEM, 0);
            CHECK(peer_row_failed(row, world) == world);
        }
        for (uint32_t f = 0; f < world; ++f) {
            for (uint32_t r = 0; r < kMaxWorld; ++r) row[r] = peer_word(CTMR_OK, r);
            row[f] = peer_word(CTMR_E_TABLE_FULL, 0);
            for (uint32_t g = f + 1; g < world; ++g) row[g] = peer_word(CTMR_E_PEER_TIMEOUT, 0);
            CHECK(peer_row_failed(row, world) == f);
            CHECK(peer_word_code(row[peer_row_failed(row, world)]) == CTMR_E_TABLE_FULL);
        }
    }
    std::printf("ok %u\n", checks);
    return 0;
}
