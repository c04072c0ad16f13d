// pair_hash.cu -- the library's own pair_hash (ctmr_common.cuh, __host__ __device__) run on the host.
//
// Reads lines of 11 unsigned 32-bit words (an (issuer, serial) pair as ctmr_crl.cu's pair_words lays it out) from stdin
// and prints one hash per line, so that the numpy restatement (tests/crl_pair_model.py) can be held against the
// compiled function.
#include <cstdio>

#include "../../ct_mapreduce_b200/csrc/ctmr_common.cuh"

int main() {
    uint32_t w[11];
    for (;;) {
        for (int i = 0; i < 11; ++i)
            if (std::scanf("%u", &w[i]) != 1) return 0;
        std::printf("%u\n", ctmr::pair_hash(w));
    }
}
