/*
 * tests/hostlogic/slot_writer.c -- the host's side of the submission-slot format, built with gcc against
 * include/apus_slot_format.h as a shared library for tests/test_gpu_header_primitives.py and tests/test_header_probe.py:
 *   sw_put      composes one slot the way the host submit path does: the data image memcpy'd inline at
 *               slot_inline_off, or into the payload ring at `pos`, then slot_finish;
 *   sw_reserve  slot_reserve, and sw_place slot_place, as the header defines them, so that the tests' own statement of
 *               the placement rule can be checked against the header compiled as C.
 */
#include <stdint.h>
#include <string.h>

#include "apus_slot_format.h"

/* the data image of a request of type `type` with a cmd of len bytes ({u16 len; cmd}, or the raw 8 / 16 B image of HEAD
 * and CONFIG, or nothing for NOOP) */
static uint32_t put_image(uint8_t *dst, uint32_t type, uint32_t len, const uint8_t *cmd)
{
    const uint32_t nb = slot_image_bytes(type, len);
    if (type == APUS_NOOP) return 0;
    if (type == APUS_CONFIG || type == APUS_HEAD) {
        memcpy(dst, cmd, nb);
        return nb;
    }
    dst[0] = (uint8_t)len;
    dst[1] = (uint8_t)(len >> 8);
    memcpy(dst + 2, cmd, len);
    return nb;
}

/* Write ticket's slot into slots (ring_slots slots of 128 B) and, for an external image, the image into pay at ring
 * position pos with APUS_SLOT_WRAP when wrap is set.  Returns the image bytes. */
uint32_t sw_put(uint8_t *slots, uint32_t ring_slots, uint8_t *pay, uint64_t ticket, uint64_t pos, uint32_t wrap,
                uint32_t type, uint16_t conn, uint64_t req_id, const uint8_t *cmd, uint32_t len)
{
    apus_slot_t *d = (apus_slot_t *)(slots + (uint64_t)APUS_SLOT_BYTES * ((ticket - 1) & (ring_slots - 1)));
    const uint32_t nb = slot_image_bytes(type, len);
    uint32_t type_off;
    if (slot_ext_bytes(nb)) {
        put_image(pay + pos, type, len, cmd);
        type_off = slot_type_off(type, APUS_SLOT_EXT | (wrap ? APUS_SLOT_WRAP : 0u), pos);
    } else {
        uint8_t img[APUS_SLOT_INLINE];
        put_image(img, type, len, cmd);
        for (uint32_t i = 0; i < nb; i++) ((uint8_t *)d)[slot_inline_off(i)] = img[i];
        type_off = slot_type_off(type, 0, 0);
    }
    d->rsv0 = 0;
    d->rsv1 = 0;
    slot_finish(d, ticket, type_off, conn, req_id, (uint16_t)len);
    return nb;
}

int sw_reserve(uint32_t S, uint64_t R, uint64_t submitted, uint64_t head, uint64_t consumed, uint64_t tail, uint64_t n,
               uint64_t need, uint64_t out[3])
{
    uint32_t wrap = 0;
    const int rc = slot_reserve(S, R, submitted, head, consumed, tail, n, need, &out[0], &out[1], &wrap);
    out[2] = wrap;
    return rc;
}

int sw_place(uint64_t R, uint64_t head, uint64_t tail, uint64_t need, uint64_t out[3])
{
    uint32_t wrap = 0;
    const int rc = slot_place(R, head, tail, need, &out[0], &out[1], &wrap);
    out[2] = wrap;
    return rc;
}
