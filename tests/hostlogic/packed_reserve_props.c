/*
 * tests/hostlogic/packed_reserve_props.c -- the payload-ring reservation of a packed device batch
 * (apus_b200/csrc/apus_slot.h: slot_packed_reserve, what apus_submit_device_packed reserves), checked on the CPU.  For
 * random valid batches -- nondecreasing offsets starting anywhere inside a values buffer, lengths 0..65535 with the
 * boundaries 0, 78, 79, 80 (inline / external: an image of 2 + len > APUS_SLOT_INLINE bytes travels in the ring) and
 * 65535 drawn often -- and for values buffers with slack past offsets[n], asserts:
 *   1. the external images of the batch, sum of slot_ext_bytes(slot_image_bytes(SEND, len)), fit the reservation;
 *   2. the reservation is at most n * round16(2 + 65535), the worst case of n maximal requests;
 *   3. the same two for every request type the packing accepts, and with every request rejected (no image at all).
 * Prints "packed ok <batches>"; any violation aborts with a message.
 */
#include <stdio.h>
#include <stdlib.h>
#include "../../include/apus_gpu.h"
#include "../../apus_b200/csrc/apus_slot.h"

#define FAIL(...) do { fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); exit(1); } while (0)

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd(void) { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }

static uint32_t draw_len(uint32_t shape)
{
    static const uint32_t edge[] = {0, 78, 79, 80, 65535};
    if (rnd() % 3 == 0) return edge[rnd() % 5];
    switch (shape) {
    case 0: return (uint32_t)(rnd() % 65536);                                  /* anything */
    case 1: return (uint32_t)(rnd() % 257);                                    /* small: mostly inline */
    case 2: return rnd() % 50 ? (uint32_t)(rnd() % 257) : (uint32_t)(rnd() % 65536);   /* heavy tail */
    default: return 64;                                                        /* uniform, all inline */
    }
}

int main(void)
{
    static const uint32_t types[] = {APUS_CSM, APUS_CONNECT, APUS_SEND, APUS_CLOSE};
    static uint64_t off[4097];
    uint64_t batches = 0;
    for (int it = 0; it < 20000; it++) {
        const uint32_t n = 1 + (uint32_t)(rnd() % (it % 10 == 0 ? 4096 : 64));
        const uint32_t shape = (uint32_t)(rnd() % 4);
        const uint32_t ty = types[rnd() % 4];
        off[0] = rnd() % 1000;                                                 /* a slice: offsets[0] > 0 */
        uint64_t ext = 0;
        for (uint32_t k = 0; k < n; k++) {
            const uint32_t len = draw_len(shape);
            off[k + 1] = off[k] + len;
            ext += slot_ext_bytes(slot_image_bytes(ty, len));
        }
        const uint64_t values_bytes = off[n] + (rnd() % 2 ? 0 : rnd() % 5000);   /* the buffer may be longer */
        const uint64_t res = slot_packed_reserve(n, values_bytes);
        const uint64_t worst = (uint64_t)n * slot_ext_bytes(2u + 65535u);
        if (ext > res)
            FAIL("batch %d (n %u, shape %u): external images take %llu B, the reservation is %llu B", it, n, shape,
                 (unsigned long long)ext, (unsigned long long)res);
        if (res > worst)
            FAIL("batch %d (n %u): the reservation %llu B exceeds n * round16(2 + 65535) = %llu B", it, n,
                 (unsigned long long)res, (unsigned long long)worst);
        if (res % 16) FAIL("batch %d: the reservation %llu B is not a multiple of 16", it, (unsigned long long)res);
        batches++;
    }
    /* every length at its own boundary, one request per batch */
    for (uint32_t len = 0; len <= 65535; len++) {
        const uint64_t ext = slot_ext_bytes(slot_image_bytes(APUS_SEND, len)), res = slot_packed_reserve(1, len);
        if (ext > res || res > slot_ext_bytes(2u + 65535u)) FAIL("len %u: image %llu B, reservation %llu B", len,
                                                               (unsigned long long)ext, (unsigned long long)res);
    }
    if (slot_packed_reserve(3, ~0ull) != 3ull * slot_ext_bytes(2u + 65535u)) FAIL("huge values_bytes: not the worst case");
    if (slot_packed_reserve(0, 0) != 0) FAIL("an empty batch reserves bytes");
    printf("packed ok %llu\n", (unsigned long long)batches);
    return 0;
}
