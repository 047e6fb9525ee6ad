/*
 * apus_reader.cuh -- device API of a resident reader: read fences that an application's own persistent kernel runs
 * beside the replica kernels, with no host call per fence (apus_reader_attach).  A READY fence gives the read index F:
 * a state that has applied through idx F answers a read that is linearizable with respect to every commit the leader's
 * consumer record had published when the fence began (the contract of apus_read_fence, apus_gpu.h).
 *
 * Self-contained: it includes only CUDA and stdint headers, apus_gpu.h, apus_fence_rule.h and apus_consumer.cuh, and
 * everything here is __device__ __forceinline__.  The engine's stream fence kernel (apus_read_fence) is written on the
 * same three steps, so that the two paths cannot disagree:
 *   1. take K: the leader's consumer flag must be 2 (a record in every role), then the acquire of its consumer record
 *      gives K, the entries it has committed;
 *   2. confirm: after that acquire, the SID of every mapped member; at least N/2 + 1 at term <= t (rf_confirmed);
 *   3. ready: polled on this replica's own record until rf_ready -- it holds the committed entries through K and the
 *      entry at that count is of term >= t.  F := the entries held.
 *
 * One fence, one thread (several threads fence at once on distinct slots s < APUS_READER_SLOTS):
 *
 *     apus_reader_fence_t f;
 *     apus_reader_begin(v, s, timeout_ns, f);        -- steps 1 and 2
 *     while (apus_reader_poll(v, f) == APUS_READER_PENDING) { other work, or apus_poll_sleep(f.sleep) }
 *     READY: apply through f.F (apus_consumer_position's next_idx - 1 >= f.F), then answer the read
 *
 * or apus_reader_fence(v, s, timeout_ns, &F), which does exactly that and sleeps between polls.
 *
 * The peer-lifetime handshake.  Steps 1 and 2 read other replicas' regions through the member words of a pinned block
 * the host keeps, and the host may clear a word (apus_replica_disconnect, the destroy of a peer) while fences run.  No
 * fence may read a region after the call that cleared its word has returned; Dekker's exclusion gives that:
 *   device, per fence in slot s: store busy[s] odd; fence.sc.sys; load the release epoch, the role word and member[];
 *                                steps 1 and 2; store busy[s] even with st.release.sys (after every load above);
 *   host, per cleared word:      store 0; full barrier (__sync_synchronize); for each busy word that is odd, spin until
 *                                it changes.
 * Either the fence's load of the word comes after the host's store in the single order of the two sequentially
 * consistent fences, and it reads 0; or the host's load of busy[s] comes after the device's odd store, and the host
 * waits until the release store that follows the fence's last load of that region.  Step 3 polls only this replica's
 * own region and runs outside the window, so the window is the N + 2 remote loads of steps 1 and 2, never a wait.
 * The role word is read in the window too, after an acquire of the release epoch: a fence that read the role word as
 * it was before a take-over's apus_replica_set_role read the epoch before that call's release, and ends RELEASED.
 */
#ifndef APUS_READER_CUH
#define APUS_READER_CUH

#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_gpu.h"
#include "apus_fence_rule.h"
#include "apus_consumer.cuh"

#define APUS_READER_PENDING 0xffffffffu   /* apus_reader_poll: the fence has not ended yet (not an APUS_WAIT_* outcome) */

// ---------------------------------------------------------------------------------
// the three steps of a fence, on raw region addresses (the stream fence kernel takes them too)
// ---------------------------------------------------------------------------------
// 1. K from the leader's region `lead` (NULL: not connected): false unless its consumer flag at on_off is 2; otherwise
//    the acquire of its record at rec_off, which orders every load after it
__device__ __forceinline__ bool apus_fence_take_k(const uint8_t *lead, uint32_t on_off, uint32_t rec_off, uint64_t &K)
{
    if (!lead || apus_ld_relaxed_sys(lead + on_off) != 2) return false;
    uint64_t k_off;
    apus_cons_read(reinterpret_cast<const volatile uint64_t *>(lead + rec_off), k_off, K);
    return true;
}
// 2. the confirmation, after step 1: the SID word (at sid_off) of every member i < n whose region is mapped; `mask`
//    receives the members counted (bit i), the result is rf_confirmed of their number
__device__ __forceinline__ bool apus_fence_confirm(const uint8_t *const *member, uint32_t n, uint32_t sid_off, uint64_t t,
                                                   uint32_t &mask)
{
    mask = 0;
#pragma unroll
    for (uint32_t i = 0; i < APUS_MAX_SERVER_COUNT; i++)
        if (i < n && member[i] && rf_member_counts(1, apus_ld_relaxed_sys(member[i] + sid_off), t)) mask |= 1u << i;
    return rf_confirmed((uint32_t)__popc(mask), n);
}
// 3. one poll of this replica's own record `rec`: `held` receives the entries it holds; true once rf_ready.  The header
//    the offset index names for idx `held` is read idx, term, idx, so that a term torn from an entry of a later lap is
//    not taken.
__device__ __forceinline__ bool apus_fence_ready(const uint8_t *entries, const uint32_t *index, uint32_t idx_mask,
                                                 uint64_t log_len, const volatile uint64_t *rec, uint64_t K, uint64_t t,
                                                 uint64_t &held)
{
    uint64_t held_off, e_idx = 0, e_term = 0;
    apus_cons_read(rec, held_off, held);
    if (held && held >= K) {
        const uint64_t off = apus_ld_relaxed_sys_u32(&index[(uint32_t)held & idx_mask]) & ~APUS_INDEX_HEAD_BIT;
        if (off + APUS_ENTRY_HDR <= log_len) {
            e_idx = apus_ld_u64_any(entries, off + APUS_ENT_IDX);
            e_term = apus_ld_u64_any(entries, off + APUS_ENT_TERM);
            if (apus_ld_u64_any(entries, off + APUS_ENT_IDX) != e_idx) e_idx = 0;
        }
    }
    return rf_ready(held, K, e_idx, e_term, t);
}

// ---------------------------------------------------------------------------------
// the resident reader's API over an apus_reader_view_t (apus_reader_attach)
// ---------------------------------------------------------------------------------
typedef struct apus_reader_fence {
    uint64_t t0;            /* %globaltimer when the fence began */
    uint64_t t_chk;         /* ... and when the release and stop words were read last */
    uint64_t timeout_ns;
    uint64_t epoch;         /* the release epoch the fence began under */
    uint64_t term;          /* t: the term of the role word when the fence began ... */
    uint32_t leader;        /* ... and L, its leader */
    uint32_t mask;          /* the members counted by the confirmation (bit i) */
    uint64_t K;             /* the leader's committed entries, taken in step 1 */
    uint64_t F;             /* READY: the read index */
    uint32_t outcome;       /* APUS_WAIT_* once ended, APUS_READER_PENDING before */
    uint32_t sleep;         /* the next back-off sleep (ns), for apus_poll_sleep */
} apus_reader_fence_t;

__device__ __forceinline__ uint64_t apus_reader_ld_acquire(const volatile void *p)
{
    uint64_t v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void apus_reader_st_release(volatile void *p, uint64_t v)
{
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Begin a fence in slot `slot` (< APUS_READER_SLOTS; one fence per slot at a time): steps 1 and 2 inside the handshake's
// window.  f.outcome is APUS_WAIT_NOT_LEADER when the leader could not be confirmed, APUS_READER_PENDING otherwise.
__device__ __forceinline__ void apus_reader_begin(const apus_reader_view_t &v, uint32_t slot, uint64_t timeout_ns,
                                                  apus_reader_fence_t &f)
{
    f.t0 = apus_globaltimer_ns();
    f.t_chk = f.t0;
    f.timeout_ns = timeout_ns;
    f.K = 0; f.F = 0; f.mask = 0;
    f.outcome = APUS_WAIT_NOT_LEADER;
    f.sleep = APUS_WAIT_SLEEP_MIN_NS;
    uint64_t *busy = v.busy + slot;
    const uint64_t seq = apus_ld_relaxed_sys(busy);          // even: only this slot's fences write it
    apus_st_relaxed_sys(busy, seq + 1);
    asm volatile("fence.sc.sys;" ::: "memory");
    f.epoch = apus_reader_ld_acquire(v.release);
    const uint64_t role = apus_ld_relaxed_sys(v.role);
    f.term = APUS_SID_TERM(role);
    f.leader = (uint32_t)(role & 0xffu);
    const uint8_t *member[APUS_MAX_SERVER_COUNT];
    const uint8_t *lead = NULL;
#pragma unroll
    for (uint32_t i = 0; i < APUS_MAX_SERVER_COUNT; i++) {
        member[i] = i < v.n ? reinterpret_cast<const uint8_t *>(apus_ld_relaxed_sys(v.member + i)) : NULL;
        if (i == f.leader) lead = member[i];
    }
    uint64_t K = 0;
    if (apus_fence_take_k(lead, v.on_off, v.rec_off, K) && apus_fence_confirm(member, v.n, v.sid_off, f.term, f.mask)) {
        f.K = K;
        f.outcome = APUS_READER_PENDING;
    }
    apus_reader_st_release(busy, seq + 2);                   // after every load of another replica's region
}
// One poll of a fence begun with apus_reader_begin: APUS_WAIT_READY (f.F is the read index), APUS_WAIT_TIMED_OUT
// (timeout_ns after it began), APUS_WAIT_RELEASED (a release point of consume waits and fences, or the reader's stop
// word; both words are read over PCIe at most every APUS_WAIT_RELEASE_POLL_NS), APUS_WAIT_NOT_LEADER (from begin), or
// APUS_READER_PENDING.  Only this replica's own region is read.
__device__ __forceinline__ uint32_t apus_reader_poll(const apus_reader_view_t &v, apus_reader_fence_t &f)
{
    if (f.outcome != APUS_READER_PENDING) return f.outcome;
    uint64_t held;
    if (apus_fence_ready(v.entries, v.index, v.idx_mask, v.log_len, v.rec, f.K, f.term, held)) {
        f.F = held;
        return f.outcome = APUS_WAIT_READY;
    }
    const uint64_t now = apus_globaltimer_ns();
    if (now - f.t_chk >= APUS_WAIT_RELEASE_POLL_NS) {
        f.t_chk = now;
        if (apus_ld_relaxed_sys(v.release) != f.epoch || apus_ld_relaxed_sys(v.stop) != v.stop_epoch)
            return f.outcome = APUS_WAIT_RELEASED;
    }
    if (now - f.t0 >= f.timeout_ns) return f.outcome = APUS_WAIT_TIMED_OUT;
    return APUS_READER_PENDING;
}
// A whole fence in slot `slot`: begin, then poll with the back-off of consume waits until it ends.  Returns its
// APUS_WAIT_* outcome; *F receives the read index on READY.
__device__ __forceinline__ uint32_t apus_reader_fence(const apus_reader_view_t &v, uint32_t slot, uint64_t timeout_ns,
                                                      uint64_t *F)
{
    apus_reader_fence_t f;
    apus_reader_begin(v, slot, timeout_ns, f);
    uint32_t o;
    while ((o = apus_reader_poll(v, f)) == APUS_READER_PENDING) apus_poll_sleep(f.sleep);
    if (o == APUS_WAIT_READY) *F = f.F;
    return o;
}
// true once apus_reader_detach or apus_replica_destroy has asked the reader to end (one load over PCIe): the reader then
// returns without touching the view again
__device__ __forceinline__ bool apus_reader_should_stop(const apus_reader_view_t &v)
{
    return apus_ld_relaxed_sys(v.stop) != v.stop_epoch;
}

#endif /* APUS_READER_CUH */
