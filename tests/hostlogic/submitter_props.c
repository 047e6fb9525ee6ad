/*
 * tests/hostlogic/submitter_props.c -- the reservation arithmetic of a resident submitter (include/apus_submitter.cuh:
 * slot_reserve and slot_reserve_pay_end of include/apus_slot_format.h, the functions the device code itself calls),
 * checked on the CPU against the host paths it shares the ring with.  A model of the engine's accounting runs random
 * interleavings of host submits (place_image), device batches (worst-case reservations packed from their start) and
 * attach / reserve / publish / detach cycles of a submitter (exact reservations of 1..600 requests of 0..1500 B, a few
 * up to 64 KiB), over many laps of both rings, with a leader that consumes published tickets lazily, and asserts:
 *   1. space is never over-committed: no live image overlaps another, every image lies inside the ring (and inside its
 *      device batch's reservation);
 *   2. the external images of consecutive tickets are contiguous unless the later one carries APUS_SLOT_WRAP;
 *   3. both hold across the detach hand-back, which drops the reservations never published and hands their ticket
 *      numbers out again.
 * Prints "submitter ok <images> <wraps> <reservations> <dropped>"; any violation aborts with a message.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../include/apus_slot_format.h"

#define FAIL(...) do { fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); exit(1); } while (0)

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd(void) { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }

#define SLOTS 2048u
#define R (256u * 1024u)
static uint64_t pay_end[SLOTS];                   /* the host's array (the submitter's copy while attached: dev_pay_end) */
static uint64_t dev_pay_end[SLOTS];
static uint64_t img_pos[SLOTS], img_len[SLOTS];   /* external image of ticket t: ring position, round16 bytes (0 = none) */
static uint32_t img_flags[SLOTS];
static uint64_t res_lo[SLOTS], res_hi[SLOTS];     /* device batch: ring positions [lo, hi) of its reservation (hi = 0: none) */
static uint64_t submitted, consumed, published, head, images, wraps, reservations, dropped;
static int wrap_next;

/* the leader: consume published tickets in order, checking the staging rule between consecutive external images */
static uint64_t last_ext_pos, last_ext_len, have_last;
static void consume(uint64_t upto)
{
    if (upto > published) upto = published;
    for (; consumed < upto; consumed++) {
        const uint64_t t = consumed % SLOTS;
        if (!img_len[t]) continue;
        if (img_pos[t] + img_len[t] > R) FAIL("ticket %llu: image crosses the ring end", (unsigned long long)consumed + 1);
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
    if (pos + len > R) FAIL("ticket %llu: image [%llu, +%llu) crosses the ring end", (unsigned long long)t,
                            (unsigned long long)pos, (unsigned long long)len);
    for (uint64_t b = pos; b < pos + len; b++) {
        const uint64_t o = owner[b];
        if (o && o > consumed) FAIL("ticket %llu overwrites live bytes of ticket %llu at %llu", (unsigned long long)t,
                                    (unsigned long long)o, (unsigned long long)b);
        owner[b] = t;
    }
}
static void set_image(uint64_t ticket, uint64_t pos, uint64_t xb, uint32_t flags)
{
    const uint64_t t = (ticket - 1) % SLOTS;
    img_len[t] = xb; img_pos[t] = pos; img_flags[t] = flags; res_hi[t] = 0;
    if (xb) claim_bytes(ticket, pos, xb);
}

static uint32_t request_len(void)
{
    if (rnd() % 200 == 0) return (uint32_t)(rnd() % 65536);          /* a few up to 64 KiB */
    if (rnd() % 3 == 0) return (uint32_t)(rnd() % 79);               /* plenty of inline images */
    return (uint32_t)(rnd() % 1501);
}

/* host path: place_image (apus_engine.cu) */
static int host_submit(uint32_t len)
{
    if (submitted - consumed >= SLOTS) return -1;
    const uint32_t need = slot_ext_bytes(slot_image_bytes(APUS_SEND, len));
    uint64_t pos = 0, h = head;
    uint32_t wrap = 0, flags = 0;
    if (need) {
        const uint64_t tail = consumed ? pay_end[(consumed - 1) % SLOTS] : 0;
        if (slot_place(R, head, tail, need, &pos, &h, &wrap)) return -1;
        flags = APUS_SLOT_EXT | ((wrap || wrap_next) ? APUS_SLOT_WRAP : 0u);
        wrap_next = 0;
    }
    set_image(submitted + 1, pos, need, flags);
    pay_end[submitted % SLOTS] = h;
    head = h;
    published = ++submitted;
    return 0;
}

/* device path: apus_submit_device's worst-case reservation, packed from its start */
static int device_batch(uint32_t n, uint32_t stride)
{
    if (submitted + n - consumed > SLOTS) return -1;
    const uint64_t res = (uint64_t)n * slot_ext_bytes(2u + stride);
    if (res > R) return -2;
    const uint64_t head0 = head, tail = consumed ? pay_end[(consumed - 1) % SLOTS] : 0;
    uint64_t pos = 0, h = head, off = 0;
    uint32_t wrap = 0;
    if (res && slot_place(R, head, tail, res, &pos, &h, &wrap)) return -1;
    for (uint32_t k = 0; k < n; k++) {
        const uint32_t len = (uint32_t)(rnd() % (stride + 1));
        const uint32_t xb = (rnd() % 8) ? slot_ext_bytes(slot_image_bytes(APUS_SEND, len)) : 0;   /* some rejected */
        set_image(submitted + k + 1, pos + off, xb, xb ? APUS_SLOT_EXT | (off == 0 ? APUS_SLOT_WRAP : 0u) : 0u);
        if (xb) { res_lo[(submitted + k) % SLOTS] = pos; res_hi[(submitted + k) % SLOTS] = pos + res; }
        off += xb;
        pay_end[(submitted + k) % SLOTS] = (k + 1 < n) ? head0 : h;
    }
    head = h;
    if (res) wrap_next = 1;
    published = submitted += n;
    return 0;
}

/* the submitter's device state while attached (apus_submitter_state_t) */
static uint64_t s_submitted, s_head, s_consumed;
static int s_wrap_next;

/* apus_submitter_try_reserve, the ext_off rule of the puts, then a publish unless `publish` is 0 */
static int submitter_reservation(uint32_t n, int publish)
{
    uint32_t xs[600];                               /* apus_submitter_ext_bytes of each request */
    uint64_t xb = 0;
    for (uint32_t k = 0; k < n; k++) {
        const uint32_t len = request_len();
        xs[k] = (rnd() % 16) ? slot_ext_bytes(slot_image_bytes(APUS_SEND, len)) : 0;  /* rejected: no bytes */
        xb += xs[k];
    }
    if (n > SLOTS || xb > R) return -2;
    uint64_t pos = 0, head_out = 0;
    uint32_t wrap = 0;
    for (int fresh = 0;; fresh++) {
        const uint64_t tail = s_consumed ? dev_pay_end[(s_consumed - 1) % SLOTS] : 0;
        if (slot_reserve(SLOTS, R, s_submitted, s_head, s_consumed, tail, n, xb, &pos, &head_out, &wrap) == 0) break;
        if (fresh) return -1;
        s_consumed = consumed;                      /* the cached bound says full: read the leader's word */
    }
    if (s_consumed > consumed) FAIL("cached consumed ahead of the leader");
    for (uint32_t k = 0; k < n; k++) dev_pay_end[(s_submitted + k) % SLOTS] = slot_reserve_pay_end(k, n, s_head, head_out);
    const uint32_t first_wrap = xb && (wrap || s_wrap_next) ? APUS_SLOT_WRAP : 0u;
    if (xb) s_wrap_next = 0;
    /* the puts: request k's image at pos + the bytes of requests 0 .. k-1 (recomputed from the same lengths) */
    uint64_t off = 0;
    for (uint32_t k = 0; k < n; k++) {
        set_image(s_submitted + k + 1, pos + off, xs[k], xs[k] ? APUS_SLOT_EXT | (off == 0 ? first_wrap : 0u) : 0u);
        off += xs[k];
    }
    s_head = head_out;
    s_submitted += n;
    reservations++;
    if (publish) {
        if (published != s_submitted - n) FAIL("publish out of turn");
        published = s_submitted;
    }
    return 0;
}

static void attach(void)
{
    s_submitted = submitted; s_head = head; s_wrap_next = wrap_next; s_consumed = consumed;
    memcpy(dev_pay_end, pay_end, sizeof pay_end);
}

/* apus_submitter_detach: the doorbell P = published becomes the host's count; reservations past it are dropped */
static void detach(void)
{
    for (uint64_t t = published; t < s_submitted; t++) {         /* dropped: their bytes are nobody's any more */
        const uint64_t i = t % SLOTS;
        for (uint64_t b = img_pos[i]; img_len[i] && b < img_pos[i] + img_len[i]; b++)
            if (owner[b] == t + 1) owner[b] = 0;
        img_len[i] = 0;
        dropped++;
    }
    memcpy(pay_end, dev_pay_end, sizeof pay_end);
    submitted = published;
    head = published ? pay_end[(published - 1) % SLOTS] : 0;
    wrap_next = 1;
}

int main(void)
{
    for (int round = 0; round < 60000; round++) {
        const uint64_t r = rnd() % 100;
        if (r < 55) {
            if (host_submit(request_len() % 1501)) consume(consumed + 1 + rnd() % 64);
        } else if (r < 63) {
            const uint32_t stride = (rnd() % 4 == 0) ? (uint32_t)(rnd() % 79) : (uint32_t)(rnd() % 1501);
            if (device_batch(1 + (uint32_t)(rnd() % 40), stride) == -1) consume(published);
        } else if (r < 80) {
            /* a submitter session: some reservations, published in order; perhaps a dropped tail */
            attach();
            const int nres = 1 + (int)(rnd() % 12);
            const int drop = rnd() % 4 == 0;
            for (int i = 0; i < nres; i++) {
                const uint32_t n = (rnd() % 3 == 0) ? 1u + (uint32_t)(rnd() % 600) : 1u + (uint32_t)(rnd() % 32);
                const int publish = !(drop && i + 1 == nres);
                int rc;
                while ((rc = submitter_reservation(n, publish)) == -1) {
                    if (consumed == published) break;        /* nothing left to free: the ring is too small for it */
                    consume(consumed + 1 + rnd() % 256);
                }
                if (rc) break;
                if (rnd() % 2) consume(consumed + rnd() % 128);
            }
            detach();
        } else {
            consume(consumed + rnd() % 48);
        }
    }
    consume(published);
    if (images < 50000 || wraps < 500 || reservations < 10000 || dropped < 100)
        FAIL("too few cases: %llu images, %llu wraps, %llu reservations, %llu dropped", (unsigned long long)images,
             (unsigned long long)wraps, (unsigned long long)reservations, (unsigned long long)dropped);
    printf("submitter ok %llu %llu %llu %llu\n", (unsigned long long)images, (unsigned long long)wraps,
           (unsigned long long)reservations, (unsigned long long)dropped);
    return 0;
}
