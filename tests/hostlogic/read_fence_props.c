/*
 * tests/hostlogic/read_fence_props.c -- the decisions of a read fence (apus_b200/csrc/apus_fence.h, the very functions
 * the fence kernel uses), checked on the CPU against their definitions:
 *   1. confirmation holds iff at least N/2 + 1 connected members carry a SID of term <= t -- exhaustively for N = 1..13
 *      over every connected mask and every choice of which members sit above t (terms t-1 / t below, t+1 / far above,
 *      with the SID's L and IDX bits varied, for several t, t = 0 included);
 *   2. a member that is not connected never counts, whatever its SID;
 *   3. READY never holds with held < K, with held == 0, with a header of another idx, or with a held entry of a term
 *      below t -- and holds in every other case.
 * Prints "fence ok <cases>"; any violation aborts with a message.
 */
#include <stdio.h>
#include <stdlib.h>
#include "../../apus_b200/csrc/apus_fence.h"

#define CHECK(c, ...) do { if (!(c)) { fprintf(stderr, "FAILED line %d: ", __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); exit(1); } } while (0)

static uint64_t sid_of(uint64_t term, uint32_t i, uint32_t variant)
{
    return (term << 9) | ((uint64_t)(variant & 1) << 8) | ((i + variant) % 13);      /* [TERM|L|IDX] */
}

int main(void)
{
    unsigned long long cases = 0;
    const uint64_t ts[] = {0, 1, 7, 1ull << 40};
    /* 1 and 2: every N, connected mask and "above t" mask */
    for (uint32_t n = 1; n <= 13; n++) {
        const uint32_t full = (1u << n) - 1, quorum = n / 2 + 1;
        for (unsigned q = 0; q < sizeof ts / sizeof ts[0]; q++) {
            const uint64_t t = ts[q];
            if (n > 10 && q != 2) continue;            /* the largest groups: one t (4^13 combinations each) */
            for (uint32_t conn = 0; conn <= full; conn++) {
                for (uint32_t above = 0; above <= full; above++) {
                    uint32_t counted = 0, want = 0;
                    for (uint32_t i = 0; i < n; i++) {
                        const uint32_t v = (conn ^ (above >> 1) ^ i) & 3;
                        const int up = (above >> i) & 1, c = (conn >> i) & 1;
                        uint64_t term;
                        if (up) term = (v & 2) ? t + (1ull << 20) : t + 1;
                        else term = (v & 2) && t ? t - 1 : t;
                        const uint32_t k = rf_member_counts(c, sid_of(term, i, v), t);
                        CHECK(k <= 1, "member counts %u", k);
                        CHECK(c || k == 0, "n %u: member %u is not connected and counts", n, i);
                        CHECK(k == (uint32_t)(c && !up), "n %u t %llu: member %u (connected %d, term %llu) counts %u",
                              n, (unsigned long long)t, i, c, (unsigned long long)term, k);
                        counted += k;
                        want += c && !up;
                    }
                    const int ok = rf_confirmed(counted, n);
                    CHECK(ok == (want >= quorum), "n %u conn %x above %x: confirmed %d with %u of %u", n, conn, above, ok,
                          want, quorum);
                    cases++;
                }
            }
        }
        /* every count of members: the threshold is exactly N/2 + 1 */
        for (uint32_t k = 0; k <= n; k++) CHECK(rf_confirmed(k, n) == (k >= quorum), "n %u, %u members", n, k);
    }
    /* 3: READY */
    for (uint64_t held = 0; held < 40; held++)
        for (uint64_t k = 0; k < 40; k++)
            for (uint64_t t = 0; t < 6; t++)
                for (uint64_t et = 0; et < 8; et++)
                    for (int off = -1; off <= 1; off++) {
                        const uint64_t eidx = held + (uint64_t)off;
                        const int r = rf_ready(held, k, eidx, et, t);
                        if (held < k) CHECK(!r, "READY with held %llu < K %llu", (unsigned long long)held, (unsigned long long)k);
                        if (et < t) CHECK(!r, "READY with a held entry of term %llu < t %llu", (unsigned long long)et, (unsigned long long)t);
                        if (held == 0) CHECK(!r, "READY with nothing held");
                        if (eidx != held) CHECK(!r, "READY on the header of idx %llu for held %llu", (unsigned long long)eidx, (unsigned long long)held);
                        CHECK(r == (held && held >= k && eidx == held && et >= t), "READY %d for held %llu K %llu", r,
                              (unsigned long long)held, (unsigned long long)k);
                        cases++;
                    }
    printf("fence ok %llu\n", cases);
    return 0;
}
