/*
 * resident_reads.cu -- a resident reader for the tests and tools/resident_read_bench.py, written against the public
 * headers alone: one CTA whose warps fence at once, lane 0 of warp w on slot slot0 + w, one fence after the other.
 * For each fence it reads the leader's committed-tickets word (T0), fences (apus_reader_begin / apus_reader_poll), and
 * on READY, when it has the same replica's consumer view, waits until that consumer has applied through F
 * (apus_consumer_position's next_idx - 1 >= F).  It then logs RD_LOG_WORDS words per fence:
 *     {slot, seq, t, L, K, member mask, outcome, F, applied, T0, t_begin, t_end}   (%globaltimer ns)
 * Before each fence it stores seq + 1 to the slot's pinned `begun` word: a host that reads b there after a call has
 * returned knows that fences seq >= b began after it (the store precedes the fence's fence.sc.sys).
 * A slot ends on the reader's stop word (apus_reader_detach / apus_replica_destroy), after `target` fences, or
 * `deadline_ns` after the launch started: every launch ends by itself.  out[2 w] = fences logged by slot w (up to
 * log_cap), out[2 w + 1] = why it ended (RD_END_*).
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_reader.cuh"

#define RD_LOG_WORDS 12u
#define RD_END_STOP     1u
#define RD_END_TARGET   2u
#define RD_END_DEADLINE 3u

struct rd_args {
    const volatile uint64_t *t0_word;  /* pinned: the leader's committed tickets (NULL: T0 = 0) */
    uint64_t *log;                     /* device: log_cap fences of RD_LOG_WORDS words per slot */
    uint64_t log_cap;
    uint64_t target;                   /* fences per slot */
    uint64_t timeout_ns;               /* of each fence */
    uint64_t deadline_ns;              /* of the launch */
    uint64_t gap_ns;                   /* pause after each fence */
    volatile uint64_t *begun;          /* pinned: [w] fences begun by slot w */
    uint64_t *out;                     /* device: 2 words per slot */
    uint32_t slot0, has_cv;
};

__global__ void resident_reads_kernel(const apus_reader_view_t v, const apus_consumer_view_t cv, const rd_args a)
{
    if ((threadIdx.x & 31u) != 0) return;
    const uint32_t w = threadIdx.x >> 5, slot = a.slot0 + w;
    const uint64_t t_start = apus_globaltimer_ns();
    uint64_t seq = 0;
    uint32_t why;
    for (;;) {
        if (seq >= a.target) { why = RD_END_TARGET; break; }
        if (apus_reader_should_stop(v)) { why = RD_END_STOP; break; }
        if (apus_globaltimer_ns() - t_start >= a.deadline_ns) { why = RD_END_DEADLINE; break; }
        const uint64_t T0 = a.t0_word ? *a.t0_word : 0;
        a.begun[w] = seq + 1;
        apus_reader_fence_t f;
        apus_reader_begin(v, slot, a.timeout_ns, f);
        uint32_t o;
        while ((o = apus_reader_poll(v, f)) == APUS_READER_PENDING) apus_poll_sleep(f.sleep);
        uint64_t applied = 0;
        if (o == APUS_WAIT_READY && a.has_cv) {
            uint32_t sleep = APUS_WAIT_SLEEP_MIN_NS;
            for (;;) {
                applied = apus_consumer_position(cv).next_idx - 1;
                if (applied >= f.F || apus_globaltimer_ns() - t_start >= a.deadline_ns) break;
                apus_poll_sleep(sleep);
            }
        }
        const uint64_t t_end = apus_globaltimer_ns();
        if (seq < a.log_cap) {
            uint64_t *e = a.log + ((uint64_t)w * a.log_cap + seq) * RD_LOG_WORDS;
            e[0] = slot; e[1] = seq; e[2] = f.term; e[3] = f.leader; e[4] = f.K; e[5] = f.mask;
            e[6] = o; e[7] = f.F; e[8] = applied; e[9] = T0; e[10] = f.t0; e[11] = t_end;
        }
        seq++;
        if (a.gap_ns) {
            const uint64_t t = apus_globaltimer_ns();
            while (apus_globaltimer_ns() - t < a.gap_ns) __nanosleep(1000);
        }
    }
    a.out[2 * w] = seq < a.log_cap ? seq : a.log_cap;
    a.out[2 * w + 1] = why;
}

extern "C" int rd_launch(const apus_reader_view_t *v, const apus_consumer_view_t *cv, const rd_args *a, unsigned slots,
                         void *stream)
{
    resident_reads_kernel<<<1, 32 * slots, 0, (cudaStream_t)stream>>>(*v, *cv, *a);
    return (int)cudaGetLastError();
}

// loaded before any replica kernel is resident: a lazy load beside them may wait for them
extern "C" int rd_load(void)
{
    cudaFuncAttributes fa;
    return (int)cudaFuncGetAttributes(&fa, resident_reads_kernel);
}

extern "C" unsigned rd_args_size(void) { return (unsigned)sizeof(rd_args); }
