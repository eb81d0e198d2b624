// Checks rand_peek_randint (procgen_b200/csrc/pg_rng.cuh) against the draw rand_randint then makes: 10^5 draws from
// each of several seeds and level ranges (so every position of a generation, 623 and 624 included, and the state
// straight after mt_seed), and states an older build left half-twisted: the peek is the next draw where word p is
// already twisted, and "unknown" where it is not. Built and run by tests/test_level_lookahead_on_cpu.py; prints
// "OK <draws>" or the first mismatch.
#include <cstdio>
#include <cstdint>
#include <climits>
#include <initializer_list>

#include "pg_rng.cuh"

using namespace pg;

static long checked = 0;

static bool peek_matches(MT19937 &s, int low, int high, const char *what, long i) {
    const int32_t p = s.p;
    int peeked = -1;
    if (!rand_peek_randint(s, low, high, &peeked)) {
        printf("MISMATCH %s draw %ld (p=%d gen=%d): peek reported unknown\n", what, i, p, s.gen);
        return false;
    }
    const int drawn = rand_randint(s, low, high);
    checked++;
    if (peeked != drawn) {
        printf("MISMATCH %s draw %ld (p=%d): peek %d, draw %d\n", what, i, p, peeked, drawn);
        return false;
    }
    return true;
}

int main() {
    static const uint32_t seeds[] = {0u, 1u, 5489u, 0x7fffffffu, 0xffffffffu, 123456789u};
    static const int ranges[][2] = {{0, INT_MAX}, {0, 200}, {1000, 1500}, {0, 1}};
    for (uint32_t seed : seeds)
        for (const auto &r : ranges) {
            MT19937 s;
            mt_seed(s, seed);
            if (s.p != 624) {
                printf("MISMATCH mt_seed leaves p=%d\n", s.p);
                return 1;
            }
            for (long i = 0; i < 100000; i++)
                if (!peek_matches(s, r[0], r[1], "sequence", i))
                    return 1;
        }
    // half-twisted states: an exhausted generation whose words [0, gen) were twisted on demand by an older build
    for (uint32_t seed : seeds)
        for (int gen : {1, 227, 300, 396, 397, 623}) {
            MT19937 base;
            mt_seed(base, seed);
            for (int k = 0; k < 700; k++) (void)mt_next(base);  // into the second generation
            base.p = 624;
            for (int k = 0; k < gen; k++) base.mt[k] = mt_twist_word(base, k);
            base.gen = gen;
            for (int p = 0; p < 624; p++) {
                MT19937 s = base;
                s.p = p;
                int peeked = -1;
                const bool known = rand_peek_randint(s, 0, INT_MAX, &peeked);
                if (p >= gen) {
                    if (known) {
                        printf("MISMATCH half-twisted gen=%d p=%d: word p is not twisted, peek reported %d\n", gen, p, peeked);
                        return 1;
                    }
                    continue;
                }
                if (!known || peeked != rand_randint(s, 0, INT_MAX)) {
                    printf("MISMATCH half-twisted gen=%d p=%d: peek %d (known %d)\n", gen, p, peeked, (int)known);
                    return 1;
                }
                checked++;
                // and the draws after it, through the rest of the generation and into the next
                for (long i = 0; i < 700; i++)
                    if (!peek_matches(s, 0, INT_MAX, "after half-twisted", i))
                        return 1;
            }
        }
    printf("OK %ld\n", checked);
    return 0;
}
