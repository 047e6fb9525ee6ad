/*
 * apus_submitter.cuh -- device API of a resident submitter: an application's own persistent kernel, on the leader's
 * GPU, that reserves tickets, writes slots and payload images straight into the leader's HBM submission ring and rings
 * the doorbell, beside the resident replica kernels (apus_submitter_attach).  The replica kernels are unchanged: they
 * read the device ring up to the doorbell word, which the publish below stores.
 *
 * Self-contained: it includes only CUDA and stdint headers, apus_gpu.h, the slot format (apus_slot_format.h) and
 * apus_consumer.cuh for the system-scope loaders and the back-off, and everything here is __device__ __forceinline__, so
 * an application compiles it into its own kernels without relocatable device code.  Any thread of any CTA may call it;
 * the calls of one reservation are made as below.
 *
 *     one thread:   xb = sum over the requests of apus_submitter_ext_bytes(type, len)
 *                   res = apus_submitter_reserve(v, n, xb, timeout_ns)            -- n consecutive tickets and xb bytes
 *     __syncthreads()                                -- hands res to the threads that put
 *     any thread,   apus_submitter_put(v, res, k, ext_off_k, type, conn, req_id, cmd, len)   -- request k of n, where
 *     each k once:  ext_off_k = the sum of apus_submitter_ext_bytes of requests 0 .. k-1 of the reservation
 *     __syncthreads()                                -- every put of the reservation is done (across CTAs: the
 *                                                       application's own synchronisation)
 *     one thread:   apus_submitter_publish(v, res, timeout_ns)                    -- in ticket order, then the doorbell
 *     any thread:   apus_submitter_committed(v) / apus_submitter_wait_committed(v, ticket, timeout_ns)
 *
 * Reservations.  A lock in the submitter's device state serialises them, so tickets and payload positions are handed
 * out in one order.  Room is checked as the host checks it (slot_reserve): the slots against `consumed` (the leader's
 * pinned word, re-read over PCIe only when the cached value says the ring is full) and the payload ring against
 * pay_end[(consumed - 1) % ring_slots].  A reservation's images lie contiguously from its position, so only its first
 * external image may carry APUS_SLOT_WRAP: the invariant of the leader's staging (apus_slot_format.h, the WRAP rule).
 * Requests whose type is not CSM, CONNECT, SEND or CLOSE, or whose cmd is longer than 65535 B (the descriptor's 16-bit
 * length, APUS_SUBMITTER_MAX_LEN), are written as the NOOP apus_submit(APUS_NOOP, ...) would write
 * at that ticket and counted (apus_device_submit_status); apus_submitter_ext_bytes gives them 0 bytes.
 *
 * Publishing.  Reservations become visible in ticket order: a publish waits until the doorbell equals the ticket before
 * its first (the doorbell is its turn word), then stores the doorbell past its last ticket.  A reservation that is
 * never published holds back every later one; their publishes end TIMED_OUT, or STOPPED when the submitter is detached,
 * and apus_submitter_detach drops them.
 *
 * Memory order.  The puts store slots and payload bytes with plain stores from any thread.  The application's barrier
 * over every put of a reservation, then the publishing thread's release store of the doorbell (as apus_consumer_advance
 * releases the cursor), orders all of them before the doorbell; the leader kernel acquires the doorbell at system scope
 * and reads the slots after it.  The turn wait acquires the previous publish, so a later doorbell value also covers the
 * earlier reservations' stores.  Commits are read with an acquire of the committed-tickets word (pinned, over PCIe).
 *
 * Take-overs.  A submitter may be attached to a follower too (apus_submitter_attach): it is then dormant, and every
 * reserve returns APUS_SUBMITTER_NOT_LEADER at once, writing nothing, while the host paths of that replica stay open.
 * The first apus_replicas_launch that runs the replica as leader hands the ring over before the launch: the host's
 * submissions (the winner's blank CONFIG) reach the ring, the accounting is copied into the state, lead_term becomes
 * the term of that leadership, and the host releases the lock.  From then on reservations are OK and carry that term (res.term), and
 * apus_submitter_leading returns it.  So one persistent kernel per replica, launched once, writes through any number of
 * take-overs: it waits out NOT_LEADER on the followers and, after a take-over, compares the term of its reservations
 * with the one it wrote under to decide what to resubmit.  The rows carry (conn, req_id); the engine removes no
 * duplicates.
 *
 * An active submitter does not step down: apus_replica_set_role refuses its replica, and a deposed or stopped leader
 * detaches its submitter before it rejoins as a follower (then attaches again, dormant).  The application's threads may
 * be delayed without bound between reserve, put and publish, so a put or publish of an earlier leadership could land in
 * the ring after a later hand-over, and nothing in the engine could fence it off: only the stop word, which detach
 * moves and then waits for the submitter's stream, ends every such thread before the ring changes hands.
 *
 * The hand-over's memory order.  While dormant, the lock word holds APUS_SUBMITTER_HOST_HELD: the host holds the lock,
 * so no kernel thread does, and a reserve's CAS fails on that value and ends NOT_LEADER.  The host writes the
 * accounting words (submitted .. consumed) and pay_end in one copy, synchronises, writes lead_term in a copy of its
 * own, synchronises, and only then writes 0 into the lock word: the release.  It writes the lock word at no other
 * time once a kernel may run.  The reserving thread's CAS acquires the lock (atom.acquire.gpu) only once it reads
 * that 0, so the accounting it then reads under the lock, and the term it reads after it, are the host's.  An active
 * reservation's critical section is the one it was before the hand-over existed; the term is one load after unlock.
 *
 * The L1 rule.  The submitter never reads ring bytes.  Its state (the lock, counters and pay_end) is read and written
 * only by the reserving thread under the lock, with volatile accesses that bypass L1, and the leader's words are read
 * with system-scope loads, which bypass L1 as well; an application that reads the ring itself must do the same.
 */
#ifndef APUS_SUBMITTER_CUH
#define APUS_SUBMITTER_CUH

#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_gpu.h"
#include "apus_slot_format.h"
#include "apus_consumer.cuh"

/* outcomes of reserve, publish and the commit waits */
#define APUS_SUBMITTER_OK          0u
#define APUS_SUBMITTER_TIMED_OUT   1u
#define APUS_SUBMITTER_STOPPED     2u   /* the stop word moved: apus_submitter_detach or apus_replica_destroy */
#define APUS_SUBMITTER_NEVER_FITS  3u   /* reserve only: n is 0 or above ring_slots, or the bytes exceed ring_bytes */
#define APUS_SUBMITTER_NOT_LEADER  4u   /* reserve only: the submitter is dormant (its replica has not led since attach) */

typedef struct apus_submitter_res {
    uint64_t first_ticket;  /* tickets first_ticket .. first_ticket + n - 1 */
    uint64_t pos;           /* payload-ring position of the reservation's first external image */
    uint32_t n;
    uint32_t wrap;          /* 1: the first external image carries APUS_SLOT_WRAP */
    uint32_t outcome;       /* APUS_SUBMITTER_*; the other fields are meaningful only for APUS_SUBMITTER_OK */
    uint32_t pad;
    uint64_t term;          /* the term the submitter held the ring in when it made the reservation */
} apus_submitter_res_t;

// ---------------------------------------------------------------------------------
// request format
// ---------------------------------------------------------------------------------
#define APUS_SUBMITTER_MAX_LEN 0xffffu   /* the descriptor's cmd length is 16 bits: a longer cmd is rejected */

// the request is written as it is: a type of CSM, CONNECT, SEND or CLOSE with a cmd of at most APUS_SUBMITTER_MAX_LEN
// bytes.  Any other request is written as the NOOP apus_submit(APUS_NOOP, conn, req_id, NULL, 0) writes at its ticket
// and counted, the rule of device batches (apus_submit_device_packed rejects a cmd above 65535 B the same way).
__device__ __forceinline__ bool apus_submitter_accepts(uint32_t type, uint32_t len)
{
    return (type == APUS_CSM || type == APUS_CONNECT || type == APUS_SEND || type == APUS_CLOSE) &&
           len <= APUS_SUBMITTER_MAX_LEN;
}
// payload-ring bytes of one request as apus_submitter_put writes it (0 when inline, or rejected)
__device__ __forceinline__ uint32_t apus_submitter_ext_bytes(uint32_t type, uint32_t len)
{
    return apus_submitter_accepts(type, len) ? slot_ext_bytes(slot_image_bytes(type, len)) : 0u;
}

// ---------------------------------------------------------------------------------
// the words the submitter shares with the leader kernel
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t apus_ld_acquire_gpu(const volatile void *p)
{
    uint64_t v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t apus_ld_acquire_sys_u64(const volatile void *p)
{
    uint64_t v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void apus_st_release_gpu(volatile void *p, uint64_t v)
{
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// one poll of the stop word (read over PCIe at most every APUS_WAIT_RELEASE_POLL_NS)
__device__ __forceinline__ bool apus_submitter_should_stop(const apus_submitter_view_t &v, apus_consumer_poll_t &p)
{
    return apus_poll_word_moved(v.stop, v.stop_epoch, apus_globaltimer_ns(), p.t_chk);
}

// ---------------------------------------------------------------------------------
// reserve: n consecutive tickets and ext_bytes of the payload ring, one thread
// ---------------------------------------------------------------------------------
// one try at the lock: the word it held (0: taken now; APUS_SUBMITTER_HOST_HELD: the submitter is dormant)
__device__ __forceinline__ uint32_t apus_submitter_try_lock(apus_submitter_state_t *s)
{
    uint32_t old;
    asm volatile("{ .reg .u64 o; atom.acquire.gpu.global.cas.b64 o, [%1], 0, 1; cvt.u32.u64 %0, o; }"
                 : "=r"(old) : "l"(&s->lock) : "memory");
    return old;
}
__device__ __forceinline__ bool apus_submitter_lock(apus_submitter_state_t *s) { return apus_submitter_try_lock(s) == 0; }
__device__ __forceinline__ void apus_submitter_unlock(apus_submitter_state_t *s) { apus_st_release_gpu(&s->lock, 0); }

// under the lock: room for the reservation in both rings, placed and accounted; false when there is none now
__device__ __forceinline__ bool apus_submitter_try_reserve(const apus_submitter_view_t &v, uint32_t n, uint64_t ext_bytes,
                                                          apus_submitter_res_t *res)
{
    volatile apus_submitter_state_t *s = v.state;
    volatile uint64_t *pay_end = v.pay_end;
    const uint32_t mask = v.ring_slots - 1;
    const uint64_t sub = s->submitted, head = s->pay_head;
    uint64_t consumed = s->consumed, pos = 0, head_out = 0;
    uint32_t wrap = 0;
    for (int fresh = 0;; fresh++) {
        const uint64_t tail = consumed ? pay_end[(consumed - 1) & mask] : 0;
        if (slot_reserve(v.ring_slots, v.ring_bytes, sub, head, consumed, tail, n, ext_bytes, &pos, &head_out, &wrap) == 0)
            break;
        if (fresh) return false;
        consumed = apus_ld_acquire_sys_u64(v.consumed);   // the cached bound says full: read the leader's word
        s->consumed = consumed;
    }
    for (uint32_t k = 0; k < n; k++) pay_end[(sub + k) & mask] = slot_reserve_pay_end(k, n, head, head_out);
    res->first_ticket = sub + 1;
    res->pos = pos;
    res->n = n;
    res->wrap = ext_bytes && (wrap || s->wrap_next) ? 1u : 0u;
    if (ext_bytes) s->wrap_next = 0;
    s->pay_head = head_out;
    s->submitted = sub + n;
    return true;
}

// the term the submitter holds the ring in, or 0 while it is dormant
__device__ __forceinline__ uint64_t apus_submitter_leading(const apus_submitter_view_t &v)
{
    const uint64_t t = apus_ld_relaxed_sys(&v.state->lead_term);
    return t == APUS_SUBMITTER_DORMANT ? 0 : t;
}

// Reserve n consecutive tickets and ext_bytes payload-ring bytes (the sum of apus_submitter_ext_bytes of the n
// requests), waiting while either ring is full, until the stop word moves or timeout_ns has passed.  A dormant
// submitter gets APUS_SUBMITTER_NOT_LEADER at once, with nothing written.
__device__ __forceinline__ apus_submitter_res_t apus_submitter_reserve(const apus_submitter_view_t &v, uint32_t n,
                                                                       uint64_t ext_bytes, uint64_t timeout_ns)
{
    apus_submitter_res_t res;
    res.first_ticket = 0; res.pos = 0; res.n = 0; res.wrap = 0; res.pad = 0; res.term = 0;
    res.outcome = APUS_SUBMITTER_NEVER_FITS;
    if (n == 0 || n > v.ring_slots || ext_bytes > v.ring_bytes) return res;
    apus_consumer_poll_t p = apus_consumer_poll_init();
    const uint64_t t0 = p.t_chk;
    for (;;) {
        const uint32_t held = apus_submitter_try_lock(v.state);
        if (held == 0) {
            const bool ok = apus_submitter_try_reserve(v, n, ext_bytes, &res);
            apus_submitter_unlock(v.state);
            if (ok) {
                // after the acquire, so the host's term; outside the lock, which it does not lengthen
                res.term = apus_ld_relaxed_sys(&v.state->lead_term);
                res.outcome = APUS_SUBMITTER_OK;
                return res;
            }
        } else if (held == APUS_SUBMITTER_HOST_HELD) {     // dormant: nothing taken, nothing written
            res.outcome = APUS_SUBMITTER_NOT_LEADER;
            return res;
        }
        if (apus_submitter_should_stop(v, p)) { res.outcome = APUS_SUBMITTER_STOPPED; return res; }
        if (apus_globaltimer_ns() - t0 >= timeout_ns) { res.outcome = APUS_SUBMITTER_TIMED_OUT; return res; }
        apus_poll_sleep(p.sleep);
    }
}

// ---------------------------------------------------------------------------------
// put: request k of a reservation, any thread
// ---------------------------------------------------------------------------------
// bytes [16q, 16q + 16) of the image {u16 len; cmd[len]} (nb = 2 + len bytes) of a cmd in device memory, any alignment
__device__ __forceinline__ uint4 apus_submitter_image_chunk(const uint8_t *cmd, uint32_t len, uint32_t nb, uint32_t q)
{
    uint32_t w[4] = {0, 0, 0, 0};
    for (uint32_t i = 0; i < 16; i++) {
        const uint32_t j = 16u * q + i;
        uint32_t b = 0;
        if (j == 0) b = len & 0xffu;
        else if (j == 1) b = (len >> 8) & 0xffu;
        else if (j < nb) b = cmd[j - 2];
        w[i >> 2] |= b << (8u * (i & 3u));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// Write request k (k < res.n) of the reservation: its image inline or at res.pos + ext_off in the payload ring (ext_off
// = the sum of apus_submitter_ext_bytes of requests 0 .. k-1), then the descriptor, then stamp1 and stamp0.  cmd: len
// bytes of device memory.  A request apus_submitter_accepts refuses (a type that is not CSM, CONNECT, SEND or CLOSE, or a
// cmd above APUS_SUBMITTER_MAX_LEN bytes) becomes a NOOP with len 0, and is counted.
__device__ __forceinline__ void apus_submitter_put(const apus_submitter_view_t &v, const apus_submitter_res_t &res,
                                                   uint32_t k, uint64_t ext_off, uint32_t type, uint32_t conn,
                                                   uint64_t req_id, const uint8_t *cmd, uint32_t len)
{
    const uint64_t ticket = res.first_ticket + k;
    if (!apus_submitter_accepts(type, len)) {
        atomicAdd(reinterpret_cast<unsigned long long *>(&v.state->rejected), 1ull);
        atomicMin(reinterpret_cast<unsigned long long *>(&v.state->first_rejected), (unsigned long long)ticket);
        type = APUS_NOOP;
        len = 0;
    }
    const uint32_t nb = slot_image_bytes(type, len), xb = slot_ext_bytes(nb);
    uint4 *d = reinterpret_cast<uint4 *>(v.slots + APUS_SLOT_BYTES * ((ticket - 1) & (v.ring_slots - 1)));
    uint32_t type_off;
    if (xb) {
        const uint64_t pos = res.pos + ext_off;
        uint4 *p = reinterpret_cast<uint4 *>(v.pay + pos);
        for (uint32_t q = 0; 16u * q < nb; q++) p[q] = apus_submitter_image_chunk(cmd, len, nb, q);
        type_off = slot_type_off(type, APUS_SLOT_EXT | (ext_off == 0 && res.wrap ? APUS_SLOT_WRAP : 0u), pos);
    } else {
        for (uint32_t q = 0; 16u * q < nb; q++) d[slot_inline_chunk(q)] = apus_submitter_image_chunk(cmd, len, nb, q);
        type_off = slot_type_off(type, 0, 0);
    }
    uint32_t w[4];
    slot_desc_words(w, req_id, type_off, len, conn);
    apus_st_v4(&d[0], make_uint4(w[0], w[1], w[2], w[3]));
    apus_st_v4(&d[7], make_uint4((uint32_t)ticket, (uint32_t)(ticket >> 32), 0u, 0u));   // stamp1
    apus_st_v4(&d[3], make_uint4((uint32_t)ticket, (uint32_t)(ticket >> 32), 0u, 0u));   // stamp0
}

// ---------------------------------------------------------------------------------
// publish: one thread, after the application's barrier over every put of the reservation
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t apus_submitter_publish(const apus_submitter_view_t &v, const apus_submitter_res_t &res,
                                                           uint64_t timeout_ns)
{
    const uint64_t want = res.first_ticket - 1;
    apus_consumer_poll_t p = apus_consumer_poll_init();
    const uint64_t t0 = p.t_chk;
    while (apus_ld_acquire_gpu(v.doorbell) != want) {         // the turn: every earlier reservation is published
        if (apus_submitter_should_stop(v, p)) return APUS_SUBMITTER_STOPPED;
        if (apus_globaltimer_ns() - t0 >= timeout_ns) return APUS_SUBMITTER_TIMED_OUT;
        apus_poll_sleep(p.sleep);
    }
    apus_st_release_gpu(v.doorbell, want + res.n);
    return APUS_SUBMITTER_OK;
}

// ---------------------------------------------------------------------------------
// commits: the leader's committed-tickets word, any thread
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t apus_submitter_committed(const apus_submitter_view_t &v)
{
    return apus_ld_acquire_sys_u64(v.committed);
}
// wait until `ticket` is committed: APUS_SUBMITTER_OK, _TIMED_OUT after timeout_ns, _STOPPED when the stop word moves
__device__ __forceinline__ uint32_t apus_submitter_wait_committed(const apus_submitter_view_t &v, uint64_t ticket,
                                                                  uint64_t timeout_ns)
{
    apus_consumer_poll_t p = apus_consumer_poll_init();
    const uint64_t t0 = p.t_chk;
    while (apus_submitter_committed(v) < ticket) {
        if (apus_submitter_should_stop(v, p)) return APUS_SUBMITTER_STOPPED;
        if (apus_globaltimer_ns() - t0 >= timeout_ns) return APUS_SUBMITTER_TIMED_OUT;
        apus_poll_sleep(p.sleep);
    }
    return APUS_SUBMITTER_OK;
}

#endif /* APUS_SUBMITTER_CUH */
