/*
 * apus_slot_format.h -- the submission-slot format of a leader's ring (DESIGN.md section 2): one definition for every
 * writer of the ring.  The host submit paths (apus_engine.cu), the fill and packing kernels (apus_batch.cu), an
 * application's resident submitter (include/apus_submitter.cuh) and the CPU property tests (tests/hostlogic) all write
 * and check slots with these functions, so it compiles as plain C as well as CUDA.  It includes only stdint, string and
 * apus_gpu.h.
 *
 * A request's data image (sm_cmd_t {u16 len; cmd[]}, the 16 B dare_cid_t of CONFIG, the 8 B offset of HEAD) travels
 * inline in its 128 B slot when it has at most APUS_SLOT_INLINE bytes, else in the payload byte ring at a 16 B aligned
 * position (APUS_SLOT_EXT).  An image never wraps the payload ring: one that would cross its end starts at 0 instead.
 *
 * The stamp rule.  A slot is written image first (inline or in the payload ring), then its descriptor (bytes 0..15),
 * then stamp1, then stamp0.  Each 64 B half is complete once its stamp holds the ticket, so a reader that polls the slot
 * itself (host-mapped ring) sees a whole request or none; a reader of the device ring relies on the doorbell instead.
 *
 * The WRAP rule, the invariant the leader kernel relies on (t1_scan, leader_place and place_fast stage the range
 * [ext_base, ext_base + cum_xb) of a claim with one copy): the external images of consecutive tickets lie contiguously
 * in the payload ring, each round16(image) bytes after the previous one, and every discontinuity is marked with
 * APUS_SLOT_WRAP on the image AFTER it.  A WRAP where the images happen to be contiguous is harmless: it only cuts a
 * sub-tile there.  Discontinuities come from the restart at 0 and from reservations whose images may end before the
 * reservation does (device batches reserve their worst case): the first external image of a device batch, and the first
 * one submitted after it by any path, carry WRAP.  A resident submitter's reservation is exact (slot_reserve), so only
 * its first external image may carry WRAP, when the reservation does not continue the previous one.
 *
 * Space is counted with monotone counters.  Tickets: `submitted` handed out, `consumed` taken by the leader kernel; a
 * ring of S slots holds submitted - consumed <= S.  Payload bytes: `head` handed out (skip gaps included), and the
 * counter after the last image the leader has consumed, pay_end[(consumed - 1) % S], where pay_end[t % S] is the head
 * after ticket t's image (or after its reservation, for a reservation's last ticket; the head before it for the others).
 */
#ifndef APUS_SLOT_FORMAT_H
#define APUS_SLOT_FORMAT_H
#include <stdint.h>
#include <string.h>

#include "apus_gpu.h"

#ifndef APUS_HD
#ifdef __CUDACC__
#define APUS_HD __host__ __device__ __forceinline__
#else
#define APUS_HD static inline
#endif
#endif

/* submission slot, 128 B: the fields of tailq_entry_t (message.h:11-17).  Requests whose data image is at most 80 B
 * travel inline, so that one coalesced read brings descriptor and payload; larger images live in the payload byte ring
 * at pay_off16 * 16.  Each 64 B half carries the slot's ticket number as a stamp, written last (the stamp rule). */
#define APUS_SLOT_BYTES   128u
#define APUS_SLOT_INLINE  80u
#define APUS_SLOT_OFF_MASK 0x00ffffffu
#define APUS_SLOT_TYPE_SHIFT 24
#define APUS_SLOT_TYPE_MASK 0x1fu
#define APUS_SLOT_EXT   (1u << 29)   /* image is in the payload ring */
#define APUS_SLOT_WRAP  (1u << 30)   /* the payload ring restarted at 0 with this image */
typedef struct apus_slot {
    uint64_t req_id;
    uint32_t type_off;           /* WRAP | EXT | type << 24 | payload offset in 16 B units */
    uint16_t len;                /* cmd length (CSM-like) */
    uint16_t clt_id;             /* connection_id */
    uint8_t  inl0[32];           /* image bytes 0..31 */
    uint64_t stamp0, rsv0;       /* ticket number (1-based position in the submission order) */
    uint8_t  inl1[48];           /* image bytes 32..79 */
    uint64_t stamp1, rsv1;
} apus_slot_t;

/* bytes of the data image of a request: NOOP none, CONFIG a dare_cid_t, HEAD a head offset, others {u16 len; cmd} */
APUS_HD uint32_t slot_image_bytes(uint32_t type, uint32_t len)
{
    if (type == APUS_NOOP) return 0;
    if (type == APUS_CONFIG) return 16;
    if (type == APUS_HEAD) return 8;
    return 2u + len;
}

/* payload-ring bytes an image of nb bytes takes: 0 when it travels inline */
APUS_HD uint32_t slot_ext_bytes(uint32_t nb) { return nb > APUS_SLOT_INLINE ? (nb + 15u) & ~15u : 0u; }

/* the type_off word: WRAP | EXT | type << 24 | payload position in 16 B units (flags = 0, or APUS_SLOT_EXT [| WRAP]) */
APUS_HD uint32_t slot_type_off(uint32_t type, uint32_t flags, uint64_t pos)
{
    return ((type & APUS_SLOT_TYPE_MASK) << APUS_SLOT_TYPE_SHIFT) | flags | ((flags & APUS_SLOT_EXT) ? (uint32_t)(pos / 16) : 0u);
}

/* Place `need` bytes (one external image, or a reservation) in a payload ring of R bytes.  `head` = bytes handed out so
 * far (skip gaps included), `tail` = the counter value after the last image the leader has consumed.  A range that
 * would cross the end of the ring restarts at 0.  Returns -1 (no room) or 0 with *pos = ring position, *head_out = the
 * counter after the range and *wrap = 1 when the range does not continue the previous one (the restart, or a range
 * that starts the ring anew at 0). */
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

/* A reservation of n consecutive tickets after `submitted` and of `need` payload bytes (the exact sum of the
 * slot_ext_bytes of its images) in a ring of S slots and R bytes, where `consumed` tickets have been taken and `tail` is
 * the payload counter after them.  Returns -1 (no room now) or 0 with *pos, *head_out and *wrap as slot_place gives them
 * (*pos = 0, *head_out = head and *wrap = 0 when need is 0).  The caller then sets pay_end of the n tickets: head for
 * all but the last, *head_out for the last (slot_reserve_pay_end). */
APUS_HD int slot_reserve(uint32_t S, uint64_t R, uint64_t submitted, uint64_t head, uint64_t consumed, uint64_t tail,
                         uint64_t n, uint64_t need, uint64_t *pos, uint64_t *head_out, uint32_t *wrap)
{
    if (submitted + n - consumed > S) return -1;
    if (!need) { *pos = 0; *head_out = head; *wrap = 0; return 0; }
    return slot_place(R, head, tail, need, pos, head_out, wrap);
}
/* pay_end of ticket k (0-based) of an n-ticket reservation placed from head to head_out: its space is freed only once
 * the whole reservation has been consumed */
APUS_HD uint64_t slot_reserve_pay_end(uint64_t k, uint64_t n, uint64_t head, uint64_t head_out)
{
    return k + 1 == n ? head_out : head;
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

/* The end of a slot written by one thread, by the stamp rule: the descriptor, then stamp1, then stamp0 (the image is
 * already in place). */
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

#endif /* APUS_SLOT_FORMAT_H */
