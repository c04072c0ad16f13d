// key_owner.cu -- the library's own key_owner (ctmr_device.cuh, __host__ __device__) run on the host.
//
// Reads "exp_hour issuer world" triples from stdin (exp_hour signed 32-bit, issuer unsigned 32-bit, world 1..8) and
// prints one owner per line, so that the Python restatement can be held against the compiled function.
#include <cstdio>

#include "../../ct_mapreduce_b200/csrc/ctmr_common.cuh"

int main() {
    long long hour = 0;
    unsigned long long issuer = 0;
    unsigned world = 0;
    while (std::scanf("%lld %llu %u", &hour, &issuer, &world) == 3)
        std::printf("%u\n", ctmr::key_owner((int32_t)hour, (uint32_t)issuer, world));
    return 0;
}
