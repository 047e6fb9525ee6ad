/*
 * apus_slot.h -- what the engine's own writers of the submission ring add to the slot format: the host submit paths
 * (apus_engine.cu: ring_put, apus_submit_uniform) and the device fill kernels (apus_batch.cu: apus_synth_kernel and the
 * packing kernels of apus_submit_device).  The format itself -- the slot, its image placement, the stamp rule and the
 * WRAP rule -- is the public include/apus_slot_format.h, which application kernels compile too.  Checked on the CPU by
 * tests/hostlogic/slot_props.c, which is why it compiles as plain C as well (and includes the public header by a path
 * relative to this one).  The payload bytes of synthetic requests (synth_word) are defined here too, for the fill
 * kernel and the host alike.
 */
#ifndef APUS_SLOT_H
#define APUS_SLOT_H
#include <stdint.h>
#include <string.h>
#include "apus_layout.h"
#include "../../include/apus_slot_format.h"

/* The payload-ring reservation of a packed device batch (apus_submit_device_packed): n requests whose cmds lie in
 * values_bytes bytes.  The host sees neither the lengths nor the types, so it bounds the external images from n and
 * values_bytes alone: an image of a valid request (len <= 65535) takes round16(2 + len) <= len + 17 bytes, the lengths
 * of a batch with nondecreasing offsets sum to at most values_bytes, and no request needs more than round16(2 + 65535). */
APUS_HD uint64_t slot_packed_reserve(uint64_t n, uint64_t values_bytes)
{
    const uint64_t worst = n * slot_ext_bytes(2u + 0xffffu);
    if (values_bytes >= worst) return worst;
    const uint64_t sum = (values_bytes + 17u * n + 15u) & ~15ull;
    return sum < worst ? sum : worst;
}

/* the data image of a request into dst: CONFIG / HEAD carry `cmd` as is, the others {u16 len; cmd[len]} */
APUS_HD void slot_put_image(uint8_t *dst, uint32_t type, uint16_t len, const void *cmd, uint32_t nb)
{
    if (!nb) return;
    if (type == T_CONFIG || type == T_HEAD) {
        memcpy(dst, cmd, nb);
    } else {
        dst[0] = (uint8_t)len; dst[1] = (uint8_t)(len >> 8);       /* sm_cmd_t {u16 len; u8 cmd[]} (dare_sm.h:23-27) */
        if (len) memcpy(dst + 2, cmd, len);
    }
}

/* an inline image of nb bytes into the slot's inl0 / inl1 */
APUS_HD void slot_put_inline(apus_slot_t *d, const uint8_t *img, uint32_t nb)
{
    if (!nb) return;
    memcpy(d->inl0, img, nb < 32 ? nb : 32);
    if (nb > 32) memcpy(d->inl1, img + 32, nb - 32);
}

/* payload byte k of the synthetic request `req_id` (apus_submit_synth): the fill kernel writes it, the host's
 * apus_synth_byte reads it back */
APUS_HD uint32_t synth_word(uint32_t seed, uint64_t req_id, uint32_t w)
{
    uint32_t x = seed ^ ((uint32_t)req_id * 0x9E3779B1u) ^ ((uint32_t)(req_id >> 32) * 0x7F4A7C15u) ^ (w * 0x85EBCA77u);
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
APUS_HD uint8_t synth_byte(uint32_t seed, uint64_t req_id, uint32_t k)
{
    return (uint8_t)(synth_word(seed, req_id, k >> 2) >> (8u * (k & 3u)));
}
#endif /* APUS_SLOT_H */
