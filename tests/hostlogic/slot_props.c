/*
 * tests/hostlogic/slot_props.c -- properties of the submission-slot format (apus_b200/csrc/apus_slot.h, the functions
 * the host submit paths and the fill kernels use), checked on the CPU.  A model of the engine's payload accounting
 * (apus_engine.cu: place_image, apus_submit_device) submits random mixes of host requests (lengths 0..1500, inline and
 * external) and device batches (worst-case reservations packed from their start) into a small payload ring, with a
 * consumer that frees space as the leader would, and asserts:
 *   1. every external image lies inside the ring, and inside its device batch's reservation;
 *   2. consecutive external images are contiguous (each round16(image) after the previous) unless the later one
 *      carries APUS_SLOT_WRAP -- the staging rule of the leader kernel;
 *   3. no two live images overlap (space accounting);
 *   4. a slot written for a host submission decodes, field by field, to the apus_slot_t layout of apus_layout.h:
 *      req_id, type_off, len, clt_id, the inline image in inl0/inl1, both stamps = the ticket.
 * Prints "slot ok <images> <wraps>"; any violation aborts with a message.
 */
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../include/apus_gpu.h"
#include "../../apus_b200/csrc/apus_slot.h"

#define FAIL(...) do { fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); exit(1); } while (0)

static uint64_t rng_state = 0x2545F4914F6CDD1Dull;
static uint64_t rnd(void) { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }

#define SLOTS 4096u
#define R (64u * 1024u)
static uint64_t pay_end[SLOTS];           /* as the engine keeps it: counter after ticket's image (or reservation) */
static uint64_t img_pos[SLOTS], img_len[SLOTS];   /* external image of ticket t: ring position, round16 bytes (0 = none) */
static uint32_t img_flags[SLOTS];
static uint64_t res_lo[SLOTS], res_hi[SLOTS];     /* device batch: ring positions [lo, hi) of its reservation (hi = 0: host) */
static uint64_t submitted, consumed, head, images, wraps;
static int wrap_next;

static uint64_t tail(void) { return consumed ? pay_end[(consumed - 1) % SLOTS] : 0; }

/* the leader: consume some tickets in order, checking the staging rule between consecutive external images */
static uint64_t last_ext_pos, last_ext_len, have_last;
static void consume(uint64_t upto)
{
    for (; consumed < upto; consumed++) {
        const uint64_t t = consumed % SLOTS;
        if (!img_len[t]) continue;
        if (img_pos[t] + img_len[t] > R) FAIL("ticket %llu: image [%llu, +%llu) crosses the ring end",
                                              (unsigned long long)consumed + 1, (unsigned long long)img_pos[t], (unsigned long long)img_len[t]);
        if (res_hi[t] && (img_pos[t] < res_lo[t] || img_pos[t] + img_len[t] > res_hi[t]))
            FAIL("ticket %llu: image outside its reservation", (unsigned long long)consumed + 1);
        if (have_last && !(img_flags[t] & APUS_SLOT_WRAP) && img_pos[t] != last_ext_pos + last_ext_len)
            FAIL("ticket %llu: image at %llu does not continue the previous one (%llu + %llu) and carries no WRAP",
                 (unsigned long long)consumed + 1, (unsigned long long)img_pos[t], (unsigned long long)last_ext_pos,
                 (unsigned long long)last_ext_len);
        if (img_flags[t] & APUS_SLOT_WRAP) wraps++;
        last_ext_pos = img_pos[t]; last_ext_len = img_len[t]; have_last = 1;
        images++;
    }
}

/* occupancy map: every live image byte is owned by one ticket */
static uint64_t owner[R];
static void claim_bytes(uint64_t t, uint64_t pos, uint64_t len)
{
    for (uint64_t b = pos; b < pos + len; b++) {
        const uint64_t o = owner[b];
        if (o && o > consumed) FAIL("ticket %llu overwrites live bytes of ticket %llu at %llu", (unsigned long long)t,
                                    (unsigned long long)o, (unsigned long long)b);
        owner[b] = t;
    }
}

/* host path: place_image + write_slot, with the slot decoded back */
static int host_submit(uint32_t type, uint16_t len)
{
    if (submitted - consumed >= SLOTS) return -1;
    const uint32_t nb = slot_image_bytes(type, len), need = slot_ext_bytes(nb);
    uint64_t pos = 0, h = head;
    uint32_t wrap = 0, flags = 0;
    if (need) {
        if (slot_place(R, head, tail(), need, &pos, &h, &wrap)) return -1;
        flags = APUS_SLOT_EXT | ((wrap || wrap_next) ? APUS_SLOT_WRAP : 0u);
        wrap_next = 0;
    }
    const uint32_t to = slot_type_off(type, flags, pos);
    const uint64_t ticket = submitted + 1, rid = rnd();
    const uint16_t conn = (uint16_t)rnd();
    uint8_t cmd[1500], img[1502];
    for (uint32_t i = 0; i < len; i++) cmd[i] = (uint8_t)rnd();
    apus_slot_t slot;
    memset(&slot, 0xA5, sizeof slot);
    slot_put_image(img, type, len, cmd, nb);
    if (!need) slot_put_inline(&slot, img, nb);
    slot_finish(&slot, ticket, to, conn, rid, len);
    /* 4: field-by-field decode through the struct of apus_layout.h */
    if (slot.req_id != rid || slot.type_off != to || slot.len != len || slot.clt_id != conn || slot.stamp0 != ticket ||
        slot.stamp1 != ticket)
        FAIL("ticket %llu: descriptor / stamps do not decode", (unsigned long long)ticket);
    if (((slot.type_off >> APUS_SLOT_TYPE_SHIFT) & APUS_SLOT_TYPE_MASK) != type) FAIL("type field");
    if (need && (uint64_t)(slot.type_off & APUS_SLOT_OFF_MASK) * 16 != pos) FAIL("payload offset field");
    if (!need && (slot.type_off & (APUS_SLOT_EXT | APUS_SLOT_WRAP))) FAIL("inline image flagged external");
    if (img[0] != (uint8_t)len || img[1] != (uint8_t)(len >> 8) || (len && memcmp(img + 2, cmd, len)))
        FAIL("image is not {u16 len; cmd}");
    if (!need) {
        const uint8_t *sb = (const uint8_t *)&slot;
        for (uint32_t i = 0; i < nb; i++) {
            if (sb[slot_inline_off(i)] != img[i]) FAIL("inline byte %u", i);
            const uint32_t off = slot_inline_off(i);
            if (off < offsetof(apus_slot_t, inl0) || (off >= offsetof(apus_slot_t, stamp0) && off < offsetof(apus_slot_t, inl1)) ||
                off >= offsetof(apus_slot_t, stamp1))
                FAIL("inline byte %u at %u is outside inl0 / inl1", i, off);
            if (16u * slot_inline_chunk(i / 16) + (i % 16) != off) FAIL("inline chunk of byte %u", i);
        }
    }
    const uint64_t t = submitted % SLOTS;
    img_len[t] = need; img_pos[t] = pos; img_flags[t] = flags; res_hi[t] = 0;
    if (need) claim_bytes(ticket, pos, need);
    pay_end[t] = h;
    head = h;
    submitted++;
    return 0;
}

/* device path: apus_submit_device's reservation and the packing kernel's placement */
static int device_batch(uint32_t n, uint32_t stride)
{
    if (submitted + n - consumed > SLOTS) return -1;
    const uint64_t per = slot_ext_bytes(2u + stride), res = (uint64_t)n * per;
    if (res > R) return -2;
    const uint64_t head0 = head;
    uint64_t pos = 0, h = head;
    uint32_t wrap = 0;
    if (res && slot_place(R, head, tail(), res, &pos, &h, &wrap)) return -1;
    uint64_t off = 0;
    for (uint32_t k = 0; k < n; k++) {
        const uint64_t t = (submitted + k) % SLOTS;
        const uint32_t type = (rnd() % 8 == 0) ? 9u : APUS_SEND;            /* some rejected: NOOP, no image */
        uint32_t len = (uint32_t)(rnd() % (stride + 1));
        if (rnd() % 16 == 0) len = stride + 1;                              /* len > stride: rejected */
        const int ok = type == APUS_SEND && len <= stride;
        const uint32_t xb = ok ? slot_ext_bytes(slot_image_bytes(APUS_SEND, len)) : 0;
        img_len[t] = xb; res_hi[t] = 0;
        if (xb) {
            img_pos[t] = pos + off;
            img_flags[t] = APUS_SLOT_EXT | (off == 0 ? APUS_SLOT_WRAP : 0u);
            res_lo[t] = pos; res_hi[t] = pos + res;
            claim_bytes(submitted + k + 1, pos + off, xb);
            off += xb;
        }
        pay_end[t] = (k + 1 < n) ? head0 : h;
    }
    if (off > res) FAIL("batch packed %llu B into a reservation of %llu B", (unsigned long long)off, (unsigned long long)res);
    head = h;
    if (res) wrap_next = 1;
    submitted += n;
    return 0;
}

int main(void)
{
    for (int round = 0; round < 200000; round++) {
        const uint64_t r = rnd() % 100;
        if (r < 70) {
            uint16_t len = (uint16_t)(rnd() % 1501);
            if (rnd() % 3 == 0) len = (uint16_t)(rnd() % 79);               /* plenty of inline images */
            const uint32_t type = (rnd() % 20 == 0) ? APUS_CONNECT : APUS_SEND;
            if (host_submit(type, len)) {
                const uint64_t upto = consumed + 1 + rnd() % 64;
                consume(upto > submitted ? submitted : upto);
            }
        } else if (r < 78) {
            const uint32_t stride = (rnd() % 4 == 0) ? (uint32_t)(rnd() % 79) : (uint32_t)(rnd() % 1501);
            const uint32_t n = 1 + (uint32_t)(rnd() % 40);
            const int rc = device_batch(n, stride);
            if (rc == -1) consume(submitted);
        } else {
            const uint64_t upto = consumed + rnd() % 48;
            consume(upto > submitted ? submitted : upto);
        }
    }
    consume(submitted);
    if (images < 100000 || wraps < 1000) FAIL("too few cases: %llu images, %llu wraps", (unsigned long long)images,
                                              (unsigned long long)wraps);
    printf("slot ok %llu %llu\n", (unsigned long long)images, (unsigned long long)wraps);
    return 0;
}
