// table_epoch.cu -- the tables' epoch encodings (ctmr_common.cuh, __host__ __device__) checked on the host: a slot is
// live only at its own epoch, zeroed memory is empty at every epoch, the hash filter ignores epoch and state, the epoch
// wraps to a clear, and a slot stamped with any epoch comes back to the same canonical bytes.  Prints "ok <checks>".
#include <cstdio>
#include <cstring>

#include "../../ct_mapreduce_b200/csrc/ctmr_common.cuh"

using namespace ctmr;

static unsigned long checks = 0, failures = 0;
#define CHECK(c)                                                                  \
    do {                                                                          \
        ++checks;                                                                 \
        if (!(c)) {                                                               \
            ++failures;                                                           \
            std::printf("FAIL line %d: %s\n", __LINE__, #c);                      \
        }                                                                         \
    } while (0)

template <class S>
static bool same_bytes(const S& a, const S& b) { return std::memcmp(&a, &b, sizeof(S)) == 0; }

int main() {
    const uint32_t epochs[] = {1u, 2u, 3u, 0x7FFFu, 0x8000u, kEpochMax - 1u, kEpochMax};
    uint64_t rng = 0x243F6A8885A308D3ull;
    for (uint32_t e : epochs) {
        CHECK(slot_state(0ull, e) == 0u);  // zeroed memory is empty at every epoch
        for (int k = 0; k < 200; ++k) {
            rng = mix64(rng + 0x9E3779B97F4A7C15ull);
            const uint64_t h = rng;
            for (uint32_t st : {kSlotPending, kSlotReady}) {
                const uint64_t w = slot_word(e, st, h);
                CHECK(slot_state(w, e) == st);
                for (uint32_t o : epochs)
                    if (o != e) CHECK(slot_state(w, o) == 0u);  // a slot of another epoch is empty
                CHECK(tag_hash_eq(w, h));
                CHECK(tag_hash_eq(w, slot_word(e == 1u ? 2u : 1u, kSlotReady, h)));
                CHECK(!tag_hash_eq(w, h ^ 4ull) && !tag_hash_eq(w, h ^ (1ull << 47)));
                CHECK(tag_hash_eq(w, h ^ (1ull << 48)) && tag_hash_eq(w, h ^ 3ull));  // bits the tag does not hold
                CHECK(slot_state(slot_word(e, st), e) == st && (slot_word(e, st) & kTagHashBits) == 0ull);
            }
        }
    }
    CHECK(next_epoch(1u) == 2u && next_epoch(kEpochMax - 1u) == kEpochMax && next_epoch(kEpochMax) == 0u);

    // ranks agreeing on one epoch at attach: a slot live at `from` is live at `to` with its hash bits, nothing else moves
    for (int k = 0; k < 200; ++k) {
        rng = mix64(rng + 7ull);
        const uint64_t h = rng;
        const uint32_t from = 1u + (uint32_t)(rng >> 60), to = from + 1u + (uint32_t)((rng >> 40) & 0xFFu);
        const uint64_t live = slot_word(from, kSlotReady, h);
        CHECK(restamp_word(live, from, to) == slot_word(to, kSlotReady, h));
        CHECK(restamp_word(slot_word(from, kSlotReady), from, to) == slot_word(to, kSlotReady));
        CHECK(restamp_word(0ull, from, to) == 0ull);
        const uint64_t stale = slot_word(from - 1u, kSlotReady, h);
        CHECK(restamp_word(stale, from, to) == stale && slot_state(restamp_word(stale, from, to), to) == 0u);
    }

    for (int k = 0; k < 500; ++k) {
        KnownSlot ks{};
        for (int i = 0; i < 12; ++i) {
            rng = mix64(rng + 1ull);
            ks.body[i] = (uint32_t)rng;
        }
        ks.inv_first = ~(uint64_t)k;
        ks.tag = (key_hash(ks.body) & ~3ull) | 2ull;  // the canonical (pre-epoch) encoding of a ready key
        CHECK(canonical_tag(ks.body) == ks.tag);
        PairSlot ps{0x100000000ull * (k + 1) + 7ull, ~(uint64_t)k, (uint64_t)k, 0ull};
        MetaSlot ms{mix64(k) | 1ull, mix64(k + 99) | 1ull, ~(uint64_t)k, 0ull};
        for (uint32_t e : epochs) {
            KnownSlot a = ks;
            PairSlot b = ps;
            MetaSlot c = ms;
            stamp_slot(a, e);
            stamp_slot(b, e);
            stamp_slot(c, e);
            CHECK(slot_state(a.tag, e) == kSlotReady && tag_hash_eq(a.tag, key_hash(ks.body)));
            CHECK(slot_state(b.pad, e) == kSlotReady && slot_state(c.pad, e) == kSlotReady);
            CHECK(same_bytes(canonical_slot(a, true), ks) && same_bytes(canonical_slot(b, true), ps) &&
                  same_bytes(canonical_slot(c, true), ms));
            const KnownSlot zk{};
            const PairSlot zp{};
            const MetaSlot zm{};
            CHECK(same_bytes(canonical_slot(a, false), zk) && same_bytes(canonical_slot(b, false), zp) &&
                  same_bytes(canonical_slot(c, false), zm));
        }
    }
    KnownSlot empty{};
    PairSlot pempty{};
    MetaSlot mempty{};
    stamp_slot(empty, 5u);
    stamp_slot(pempty, 5u);
    stamp_slot(mempty, 5u);
    CHECK(empty.tag == 0ull && pempty.pad == 0ull && mempty.pad == 0ull);  // an empty canonical slot stays empty

    if (failures) {
        std::printf("%lu of %lu checks failed\n", failures, checks);
        return 1;
    }
    std::printf("ok %lu\n", checks);
    return 0;
}
