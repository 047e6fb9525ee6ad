/*
 * apus_consumer.cuh -- device API of a resident consumer: an application's own persistent kernel that applies the
 * committed entries of a replica's log in place, beside the resident replica kernels (apus_consumer_attach).
 *
 * Self-contained: it includes only CUDA and stdint headers and apus_gpu.h, and everything here is
 * __device__ __forceinline__, so an application compiles it into its own kernels without relocatable device code.
 * The engine's stream-ordered consume kernels (apus_consume_device*, apus_consume_wait, apus_read_fence) use the same
 * definitions, so that the two paths agree on which entries are committed and where the cursor goes.
 *
 * A consumer loop, one CTA (several CTAs synchronise among themselves where the CTA barrier stands below):
 *
 *     thread 0: pos = apus_consumer_position(v); n = apus_consumer_available(v, pos, &committed)
 *     __syncthreads()                                -- hands thread 0's acquire to the rest of the CTA
 *     any thread, k < n: e = apus_consumer_entry(v, pos, committed, k); read its bytes with apus_consumer_copy_cmd or
 *                        the apus_ld_*_any loaders
 *     __syncthreads()                                -- every read of the examined entries is done
 *     thread 0: pos = apus_consumer_advance(v, pos, committed, examined)
 *     thread 0, when n == 0: apus_consumer_backoff(p); apus_consumer_should_stop(v, p) ends the loop
 *     __syncthreads()                                -- before thread 0 overwrites what the CTA shares of this pass
 *
 * Memory order.  The consumer record is stored with a release by the replica kernel (a follower's thread 0 at .sys, a
 * leader's commit warp at .gpu) after the entry bytes and index words it covers; apus_consumer_available acquires it,
 * and the application's barrier carries that to the threads that read the entries.  In the other direction,
 * apus_consumer_advance stores the cursor with a release after the application's barrier over every read of the
 * examined bytes; the replica kernel forwards the cursor to the leader's pruning rule, and only then may the leader
 * overwrite those bytes.
 *
 * The L1 rule.  A persistent kernel must read log bytes and index words only with the system-scope relaxed loads
 * below (ld.relaxed.sys bypasses L1), never with plain loads: the ring is rewritten lap after lap at the same
 * addresses, and a line one lap cached in L1 could be served for the next lap.
 */
#ifndef APUS_CONSUMER_CUH
#define APUS_CONSUMER_CUH

#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_gpu.h"

/* entry header fields (the reference's dare_log_entry_t, dare_log.h:33-48) */
#define APUS_ENT_IDX    0
#define APUS_ENT_TERM   8
#define APUS_ENT_REQID 16
#define APUS_ENT_CLTID 24
#define APUS_ENT_TYPE  26
#define APUS_ENT_DATA  48     /* CSM-like: u16 cmd length */
#define APUS_ENT_CMD   50     /* CSM-like: the cmd bytes */
#define APUS_INDEX_HEAD_BIT 0x80000000u   /* offset-index word: the entry is a HEAD entry */

/* what apus_cons_locate finds for an entry */
#define APUS_CONS_OK     0u
#define APUS_CONS_LATER  1u   /* not committed (yet) */
#define APUS_CONS_BAD    2u   /* the index word names no entry carrying the expected idx: APUS_CONSUME_BAD_IDX */

/* back-off of every poll of the consumer record: stream-ordered waits and fences, and resident consumers */
#define APUS_WAIT_SLEEP_MIN_NS     32u
#define APUS_WAIT_SLEEP_MAX_NS     1024u      /* bounds the delay a poll adds to commit-to-applied latency */
#define APUS_WAIT_RELEASE_POLL_NS  20000ull   /* the host's words are read over PCIe at most this often */

// ---------------------------------------------------------------------------------
// system-scope loads and stores: peers and the host observe these, and they bypass L1
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t apus_ld_relaxed_sys(const volatile void *p)
{
    uint64_t v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t apus_ld_relaxed_sys_u32(const volatile void *p)
{
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void apus_ld_acquire_sys_2x64(const volatile void *p, uint64_t &a, uint64_t &b)
{
    // an acquire LOAD is far cheaper than a system fence (tools/ubench measures both)
    asm volatile("ld.acquire.sys.global.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ uint4 apus_ld_relaxed_sys_v4(const void *p)
{
    uint4 v;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ void apus_st_relaxed_sys(volatile void *p, uint64_t v)
{
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void apus_st_relaxed_sys_2x64(volatile void *p, uint64_t a, uint64_t b)
{
    asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}
__device__ __forceinline__ void apus_st_release_sys_2x64(volatile void *p, uint64_t a, uint64_t b)
{
    asm volatile("st.release.sys.global.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}
__device__ __forceinline__ void apus_st_v4(void *p, uint4 v)
{
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}
__device__ __forceinline__ void apus_st_u8(void *p, uint32_t v)
{
    asm volatile("st.global.u8 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t apus_globaltimer_ns()
{
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ---------------------------------------------------------------------------------
// log bytes of any alignment (entries: the log ring, at: a log offset)
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t apus_ld_u8_any(const uint8_t *entries, uint64_t at)
{
    return (apus_ld_relaxed_sys_u32(entries + (at & ~3ull)) >> (8 * (at & 3ull))) & 0xffu;
}
__device__ __forceinline__ uint32_t apus_ld_u16_any(const uint8_t *entries, uint64_t at)
{
    return apus_ld_u8_any(entries, at) | (apus_ld_u8_any(entries, at + 1) << 8);
}
// one 8 B load, or eight byte reads out of 4 B-aligned words
__device__ __forceinline__ uint64_t apus_ld_u64_any(const uint8_t *entries, uint64_t at)
{
    uint64_t v = apus_ld_relaxed_sys(entries + (at & ~7ull));
    if (at & 7ull) {
        v = 0;
        for (int q = 7; q >= 0; q--) v = (v << 8) | (uint64_t)(apus_ld_relaxed_sys_u32(entries + ((at + q) & ~3ull)) >> (8 * ((at + q) & 3ull)) & 0xffu);
    }
    return v;
}

// `len` bytes from src (log bytes, any alignment) to dst (any alignment), by the `nthr` threads `c` of a group: each
// writes 16 B-aligned destination chunks, built from the one or two aligned 16 B source chunks that hold them.  Only
// chunks holding a wanted byte are loaded (they lie inside the entry); destination bytes outside [dst, dst + len) are
// not written.
__device__ __forceinline__ void apus_copy_cmd(uint8_t *dst, const uint8_t *src, uint32_t len, uint32_t c, uint32_t nthr)
{
    if (!len) return;
    const uint64_t d = (uint64_t)(uintptr_t)dst, d16 = d & ~15ull, de = d + len;
    const uint64_t sb = (uint64_t)(uintptr_t)src - (d - d16);         // source address of destination byte d16
    const uint64_t s_lo = (uint64_t)(uintptr_t)src, s_hi = s_lo + len;
    const uint32_t nch = (uint32_t)(((de + 15ull) & ~15ull) - d16) >> 4;
    for (uint32_t q = c; q < nch; q += nthr) {
        const uint64_t s = sb + 16ull * q, s16 = s & ~15ull;
        const uint32_t sh = (uint32_t)(s & 15ull);
        const uint64_t want_lo = s > s_lo ? s : s_lo, want_hi = (s + 16 < s_hi) ? s + 16 : s_hi;
        uint4 c0 = make_uint4(0, 0, 0, 0), c1 = make_uint4(0, 0, 0, 0);
        if (want_lo < s16 + 16) c0 = apus_ld_relaxed_sys_v4(reinterpret_cast<const void *>(s16));
        if (sh && want_hi > s16 + 16) c1 = apus_ld_relaxed_sys_v4(reinterpret_cast<const void *>(s16 + 16));
        const uint64_t a0 = c0.x | ((uint64_t)c0.y << 32), a1 = c0.z | ((uint64_t)c0.w << 32);
        const uint64_t a2 = c1.x | ((uint64_t)c1.y << 32), a3 = c1.z | ((uint64_t)c1.w << 32);
        const uint32_t k = sh >> 3, b = 8u * (sh & 7u);
        const uint64_t w0 = k ? a1 : a0, w1 = k ? a2 : a1, w2 = k ? a3 : a2;
        const uint64_t r0 = b ? (w0 >> b) | (w1 << (64u - b)) : w0, r1 = b ? (w1 >> b) | (w2 << (64u - b)) : w1;
        const uint64_t o = d16 + 16ull * q;
        if (o >= d && o + 16 <= de) {
            apus_st_v4(reinterpret_cast<void *>(o), make_uint4((uint32_t)r0, (uint32_t)(r0 >> 32), (uint32_t)r1, (uint32_t)(r1 >> 32)));
        } else {
            for (uint32_t i = 0; i < 16; i++)
                if (o + i >= d && o + i < de) apus_st_u8(reinterpret_cast<void *>(o + i), (uint32_t)(((i < 8 ? r0 : r1) >> (8 * (i & 7))) & 0xffu));
        }
    }
}

// ---------------------------------------------------------------------------------
// entry format
// ---------------------------------------------------------------------------------
__device__ __forceinline__ bool apus_has_cmd(uint32_t type)
{
    return !(type == APUS_NOOP || type == APUS_CONFIG || type == APUS_HEAD);
}
__device__ __forceinline__ uint32_t apus_entry_stride(uint32_t type, uint32_t len)
{
    return apus_has_cmd(type) ? APUS_ENTRY_HDR + len : APUS_ENTRY_HDR;   // dare_log.h:228-234
}
__device__ __forceinline__ uint64_t apus_ring_dist(uint64_t from, uint64_t to, uint64_t L)
{
    return to >= from ? to - from : L - (from - to);
}

// ---------------------------------------------------------------------------------
// the consumer record {committed-and-held offset, entries held} and the cursor {offset, idx of the next entry}
// ---------------------------------------------------------------------------------
__device__ __forceinline__ void apus_cons_read(const volatile uint64_t *rec, uint64_t &held_off, uint64_t &held_entries)
{
    apus_ld_acquire_sys_2x64(rec, held_off, held_entries);
}
// committed entries past the cursor: the record holds entries 1 .. held_entries, the cursor stands at idx next_idx
__device__ __forceinline__ uint64_t apus_cons_avail(uint64_t held_entries, uint64_t next_idx)
{
    return held_entries + 1 > next_idx ? held_entries + 1 - next_idx : 0;
}
// the entry with idx `idx`: its offset from the index word, then whether it is committed (within [cursor, committed) of
// the one lap the cursor bounds), carries that idx, and fits the log.  *ty and *len are set for a committed entry.
__device__ __forceinline__ uint32_t apus_cons_locate(const uint8_t *entries, const uint32_t *index, uint32_t idx_mask,
                                                     uint64_t L, uint64_t cursor, uint64_t committed, uint64_t idx,
                                                     uint64_t *off, uint32_t *ty, uint32_t *len)
{
    const uint64_t o = apus_ld_relaxed_sys_u32(&index[(uint32_t)idx & idx_mask]) & ~APUS_INDEX_HEAD_BIT;
    *off = o;
    if (apus_ring_dist(cursor, o, L) >= apus_ring_dist(cursor, committed, L)) return APUS_CONS_LATER;
    if (o + APUS_ENTRY_HDR > L || apus_ld_u64_any(entries, o + APUS_ENT_IDX) != idx) return APUS_CONS_BAD;
    *ty = apus_ld_u8_any(entries, o + APUS_ENT_TYPE);
    if (apus_has_cmd(*ty)) {
        *len = apus_ld_u16_any(entries, o + APUS_ENT_DATA);
        if (o + apus_entry_stride(*ty, *len) > L) return APUS_CONS_BAD;   // not an entry this log could hold
    }
    return APUS_CONS_OK;
}
// the cursor past an examined entry: its end, where L is 0
__device__ __forceinline__ uint64_t apus_cons_cursor_after(uint64_t off, uint32_t ty, uint32_t len, uint64_t L)
{
    const uint64_t cur = off + apus_entry_stride(ty, len);
    return cur == L ? 0 : cur;
}
// one poll of a host word that ends a poll loop, at most every APUS_WAIT_RELEASE_POLL_NS (t_chk: when it was read last):
// true when it no longer holds `epoch`
__device__ __forceinline__ bool apus_poll_word_moved(const volatile uint64_t *word, uint64_t epoch, uint64_t now, uint64_t &t_chk)
{
    if (now - t_chk >= APUS_WAIT_RELEASE_POLL_NS) {
        t_chk = now;
        if (apus_ld_relaxed_sys(word) != epoch) return true;
    }
    return false;
}
// the sleep between two polls: `sleep` doubles from APUS_WAIT_SLEEP_MIN_NS up to APUS_WAIT_SLEEP_MAX_NS
__device__ __forceinline__ void apus_poll_sleep(uint32_t &sleep)
{
    __nanosleep(sleep);
    if (sleep < APUS_WAIT_SLEEP_MAX_NS) sleep <<= 1;
}

// ---------------------------------------------------------------------------------
// the resident consumer's API over an apus_consumer_view_t (apus_consumer_attach)
// ---------------------------------------------------------------------------------
typedef struct apus_consumer_pos {
    uint64_t cursor;        /* log offset where the next entry starts (or the wrap gap before it) */
    uint64_t next_idx;      /* idx of the next entry */
} apus_consumer_pos_t;

typedef struct apus_consumer_entry {
    uint64_t idx, req_id;
    uint64_t cmd_off;       /* log offset of the cmd bytes (CSM-like entries) */
    uint64_t off;           /* log offset of the entry */
    uint32_t type, len;     /* len: cmd length (CSM-like entries, else 0) */
    uint32_t clt_id;
    uint32_t status;        /* APUS_CONS_OK; APUS_CONS_LATER: not committed yet as its index word shows it, examine up to
                               it and poll again; APUS_CONS_BAD: the consumer is stopped for good (APUS_CONSUME_BAD_IDX) */
} apus_consumer_entry_t;

typedef struct apus_consumer_poll {
    uint64_t t_chk;         /* %globaltimer when the stop word was read last */
    uint32_t sleep;         /* next back-off sleep (ns) */
} apus_consumer_poll_t;

// the consumer's position (one writer: the resident consumer itself, through apus_consumer_advance).  It is also what a
// snapshot of the application's state records: apus_consume_seed starts a replacement there.
__device__ __forceinline__ apus_consumer_pos_t apus_consumer_position(const apus_consumer_view_t &v)
{
    apus_consumer_pos_t p;
    p.cursor = apus_ld_relaxed_sys(&v.cur[0]);
    p.next_idx = apus_ld_relaxed_sys(&v.cur[1]);
    return p;
}
// committed entries past `p` (0 once the consumer is stopped by APUS_CONSUME_BAD_IDX); *committed receives the
// committed-and-held offset that apus_consumer_entry and apus_consumer_advance take.  One thread: its acquire of the
// record reaches the other threads through the application's barrier after it.
__device__ __forceinline__ uint64_t apus_consumer_available(const apus_consumer_view_t &v, apus_consumer_pos_t p,
                                                            uint64_t *committed)
{
    uint64_t held;
    apus_cons_read(v.rec, *committed, held);
    if (*(const volatile uint64_t *)v.error) return 0;
    return apus_cons_avail(held, p.next_idx);
}
// entry k past `p`, k < apus_consumer_available(): any thread, concurrently.  The examination stops before the first
// entry whose status is not APUS_CONS_OK, as the stream-ordered consume calls stop: APUS_CONS_LATER quietly (the next
// poll goes on there), APUS_CONS_BAD for good -- an entry that does not carry the idx its index word promises sets the
// sticky error and its status word, and apus_consumer_available reports nothing from then on.
__device__ __forceinline__ apus_consumer_entry_t apus_consumer_entry(const apus_consumer_view_t &v, apus_consumer_pos_t p,
                                                                     uint64_t committed, uint64_t k)
{
    apus_consumer_entry_t e;
    e.idx = p.next_idx + k;
    e.type = APUS_NOOP; e.len = 0; e.clt_id = 0; e.req_id = 0;
    e.status = apus_cons_locate(v.entries, v.index, v.idx_mask, v.log_len, p.cursor, committed, e.idx, &e.off, &e.type,
                                &e.len);
    if (e.status == APUS_CONS_LATER) return e;
    if (e.status == APUS_CONS_BAD) {
        *(volatile uint64_t *)v.error = APUS_CONSUME_BAD_IDX;
        apus_st_relaxed_sys(&v.status[3], APUS_CONSUME_BAD_IDX);
        return e;
    }
    e.cmd_off = e.off + APUS_ENT_CMD;
    if (apus_has_cmd(e.type)) {
        e.clt_id = apus_ld_u16_any(v.entries, e.off + APUS_ENT_CLTID);
        e.req_id = apus_ld_u64_any(v.entries, e.off + APUS_ENT_REQID);
    } else {
        e.len = 0;
    }
    return e;
}
// the cmd of a CSM-like entry into dst (any alignment), by the nthr threads c of a group
__device__ __forceinline__ void apus_consumer_copy_cmd(const apus_consumer_view_t &v, const apus_consumer_entry_t &e,
                                                       uint8_t *dst, uint32_t c, uint32_t nthr)
{
    apus_copy_cmd(dst, v.entries + e.cmd_off, e.len, c, nthr);
}
// Move past the first n entries after `p` (n examined, each of them APUS_CONS_OK) and return the new position.  One
// thread, after the application's barrier over every read of those entries (across CTAs: after the application's own
// synchronisation).  The cursor is the end of the last examined entry, 0 for the log's end, stored with a release: the
// leader may prune and overwrite everything behind it.  The status words apus_consume_status reads follow.
__device__ __forceinline__ apus_consumer_pos_t apus_consumer_advance(const apus_consumer_view_t &v, apus_consumer_pos_t p,
                                                                     uint64_t committed, uint64_t n)
{
    if (n == 0) return p;
    uint64_t off = 0;
    uint32_t ty = APUS_NOOP, len = 0;
    apus_cons_locate(v.entries, v.index, v.idx_mask, v.log_len, p.cursor, committed, p.next_idx + n - 1, &off, &ty, &len);
    apus_consumer_pos_t q;
    q.cursor = apus_cons_cursor_after(off, ty, len, v.log_len);
    q.next_idx = p.next_idx + n;
    apus_st_release_sys_2x64(v.cur, q.cursor, q.next_idx);
    apus_st_relaxed_sys(&v.status[0], q.cursor);
    apus_st_relaxed_sys(&v.status[1], q.next_idx);
    apus_st_relaxed_sys(&v.status[2], 0);
    apus_st_relaxed_sys(&v.status[3], *(const volatile uint64_t *)v.error);
    return q;
}
__device__ __forceinline__ apus_consumer_poll_t apus_consumer_poll_init()
{
    apus_consumer_poll_t p;
    p.t_chk = apus_globaltimer_ns();
    p.sleep = APUS_WAIT_SLEEP_MIN_NS;
    return p;
}
// true once apus_consumer_detach or apus_replica_destroy has asked the consumer to end (the stop word is read over PCIe
// at most every APUS_WAIT_RELEASE_POLL_NS); the consumer then returns without touching the view again
__device__ __forceinline__ bool apus_consumer_should_stop(const apus_consumer_view_t &v, apus_consumer_poll_t &p)
{
    return apus_poll_word_moved(v.stop, v.stop_epoch, apus_globaltimer_ns(), p.t_chk);
}
// back off after a poll that found nothing; apus_consumer_found resets the back-off once entries arrive
__device__ __forceinline__ void apus_consumer_backoff(apus_consumer_poll_t &p) { apus_poll_sleep(p.sleep); }
__device__ __forceinline__ void apus_consumer_found(apus_consumer_poll_t &p) { p.sleep = APUS_WAIT_SLEEP_MIN_NS; }

#endif /* APUS_CONSUMER_CUH */
