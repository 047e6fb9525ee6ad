/*
 * apus_slot.h -- the submission-slot format (DESIGN.md section 2), written by the host submit paths
 * (apus_engine.cu: ring_put, apus_submit_uniform), by the device fill kernels (apus_batch.cu: apus_synth_kernel and
 * the packing kernels of apus_submit_device) and checked on the CPU by tests/hostlogic/slot_props.c, which is why it
 * compiles as plain C as well.  The payload bytes of synthetic requests (synth_word) are defined here too, for the
 * fill kernel and the host alike.
 *
 * A request's data image (sm_cmd_t {u16 len; cmd[]}, the 16 B dare_cid_t of CONFIG, the 8 B offset of HEAD) travels
 * inline in its 128 B slot when it has at most APUS_SLOT_INLINE bytes, else in the payload byte ring at a 16 B aligned
 * position (APUS_SLOT_EXT).  An image never wraps the payload ring: one that would cross its end starts at 0 instead.
 *
 * The invariant the leader kernel relies on (t1_scan, leader_place and place_fast stage the range
 * [ext_base, ext_base + cum_xb) of a claim with one copy): the external images of consecutive tickets lie
 * contiguously in the payload ring, each round16(image) bytes after the previous one, and every discontinuity is
 * marked with APUS_SLOT_WRAP on the image AFTER it.  A WRAP where the images happen to be contiguous is harmless: it
 * only cuts a sub-tile there.  Discontinuities come from the restart at 0 and from device batches
 * (apus_submit_device), whose images fill their worst-case reservation from its start but may end before it does:
 * the first external image of a device batch, and the first one submitted after it by any path, carry WRAP.
 */
#ifndef APUS_SLOT_H
#define APUS_SLOT_H
#include <stdint.h>
#include <string.h>
#include "apus_layout.h"
#ifndef APUS_HD
#ifdef __CUDACC__
#define APUS_HD __host__ __device__ __forceinline__
#else
#define APUS_HD static inline
#endif
#endif

/* bytes of the data image of a request: NOOP none, CONFIG a dare_cid_t, HEAD a head offset, others {u16 len; cmd} */
APUS_HD uint32_t slot_image_bytes(uint32_t type, uint32_t len)
{
    if (type == T_NOOP) return 0;
    if (type == T_CONFIG) return 16;
    if (type == T_HEAD) return 8;
    return 2u + len;
}

/* payload-ring bytes an image of nb bytes takes: 0 when it travels inline */
APUS_HD uint32_t slot_ext_bytes(uint32_t nb) { return nb > APUS_SLOT_INLINE ? (nb + 15u) & ~15u : 0u; }

/* the type_off word: WRAP | EXT | type << 24 | payload position in 16 B units (flags = 0, or APUS_SLOT_EXT [| WRAP]) */
APUS_HD uint32_t slot_type_off(uint32_t type, uint32_t flags, uint64_t pos)
{
    return ((type & APUS_SLOT_TYPE_MASK) << APUS_SLOT_TYPE_SHIFT) | flags | ((flags & APUS_SLOT_EXT) ? (uint32_t)(pos / 16) : 0u);
}

/* Place `need` bytes (one external image, or a device batch's reservation) in a payload ring of R bytes.  Space is
 * counted with monotone byte counters: `head` = bytes handed out so far (skip gaps included), `tail` = the counter
 * value after the last image the leader has consumed.  A range that would cross the end of the ring restarts at 0.
 * Returns -1 (no room) or 0 with *pos = ring position, *head_out = the counter after the range and *wrap = 1 when the
 * range does not continue the previous one (the restart, or a range that starts the ring anew at 0). */
APUS_HD int slot_place(uint64_t R, uint64_t head, uint64_t tail, uint64_t need, uint64_t *pos, uint64_t *head_out,
                       uint32_t *wrap)
{
    const uint64_t p = head % R;
    const uint64_t skip = (p + need > R) ? (R - p) : 0;
    if ((head - tail) + skip + need > R && !(head == tail && need <= R)) return -1;   /* (an empty ring takes any fit) */
    head += skip;
    *pos = head % R;
    *wrap = (skip || (*pos == 0 && head != 0)) ? 1u : 0u;
    *head_out = head + need;
    return 0;
}

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

/* offset inside the 128 B slot of inline image byte i (i < APUS_SLOT_INLINE): bytes 0..31 in inl0, 32..79 in inl1 */
APUS_HD uint32_t slot_inline_off(uint32_t i) { return i < 32u ? 16u + i : 32u + i; }
/* the slot's 16 B chunk that holds inline image chunk q (q < 5); chunk 0 is the descriptor, 3 and 7 the stamps */
APUS_HD uint32_t slot_inline_chunk(uint32_t q) { return q < 2u ? q + 1u : q + 2u; }

/* the descriptor chunk (slot bytes 0..15) as four little-endian words */
APUS_HD void slot_desc_words(uint32_t w[4], uint64_t req_id, uint32_t type_off, uint32_t len, uint32_t conn)
{
    w[0] = (uint32_t)req_id;
    w[1] = (uint32_t)(req_id >> 32);
    w[2] = type_off;
    w[3] = (len & 0xffffu) | ((conn & 0xffffu) << 16);
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

/* Writing a slot: the image first (inline or in the payload ring), then the descriptor, then the two stamps.  Each
 * 64 B half is complete once its stamp holds the ticket, so a reader that polls the slot itself (host-mapped ring)
 * sees a whole request or none. */
APUS_HD void slot_finish(apus_slot_t *d, uint64_t ticket, uint32_t type_off, uint16_t conn, uint64_t req_id, uint16_t len)
{
    uint32_t w[4];
    slot_desc_words(w, req_id, type_off, len, conn);
    memcpy(d, w, sizeof w);
#ifdef __CUDA_ARCH__
    *(volatile uint64_t *)&d->stamp1 = ticket;
    *(volatile uint64_t *)&d->stamp0 = ticket;
#else
    __atomic_store_n(&d->stamp1, ticket, __ATOMIC_RELEASE);
    __atomic_store_n(&d->stamp0, ticket, __ATOMIC_RELEASE);
#endif
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
