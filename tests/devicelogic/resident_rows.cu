/*
 * resident_rows.cu -- a resident consumer for the tests and tools/resident_consumer_bench.py, written against the public
 * header alone: one persistent CTA of RR_THREADS threads that polls its replica's consumer record, examines up to
 * `max_pass` committed entries per pass, writes the CSM-like ones as rows in the strided layout of
 * apus_consume_device (idx, type, clt_id, req_id, len, cmd at row * stride), advances, publishes its row count, and logs
 * every cursor it advanced to, with its row count and %globaltimer.
 *
 * Host control word ctl[0] (pinned): 1 asks the consumer to stop examining and write its position {cursor offset, next
 * idx} and its row count to pos[0..2], then it acknowledges with ctl[1] = 1 and examines nothing until ctl[0] is 2.
 * The kernel ends on the stop word (apus_consumer_detach / apus_replica_destroy), once it has written `target` rows,
 * on a sticky APUS_CONSUME_BAD_IDX, on a full row buffer, or `deadline_ns` after it started: every launch ends by
 * itself.  out[0] says why (RR_END_*), out[1] the rows written, out[2] the cursor log's length.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_consumer.cuh"

#define RR_THREADS 256u
#define RR_END_STOP     1u
#define RR_END_TARGET   2u
#define RR_END_BAD_IDX  3u
#define RR_END_FULL     4u
#define RR_END_DEADLINE 5u

struct rr_args {
    uint64_t *idx;
    uint8_t *types;
    uint16_t *conns;
    uint64_t *req_ids;
    uint16_t *lens;
    uint8_t *payloads;
    uint64_t stride, row_cap, target;
    uint32_t max_pass, pad;
    uint64_t delay_ns, deadline_ns;
    volatile uint64_t *rows_pub;   /* pinned: rows written so far */
    uint64_t *log;                 /* device: {cursor, rows, %globaltimer} per advance */
    uint64_t log_cap;
    volatile uint32_t *ctl;        /* pinned: snapshot request / acknowledgement */
    volatile uint64_t *pos;        /* pinned: {cursor, next idx, rows} written on request */
    uint64_t *out;                 /* device: {why it ended, rows, log length} */
};

__global__ void __launch_bounds__(RR_THREADS) resident_rows_kernel(const apus_consumer_view_t v, const rr_args a)
{
    __shared__ apus_consumer_pos_t s_pos;
    __shared__ uint64_t s_committed, s_rows, s_logn;
    __shared__ uint32_t s_m, s_end, s_first_bad;
    __shared__ uint32_t s_flag[RR_THREADS / 32];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    apus_consumer_poll_t poll;
    const uint64_t t_start = apus_globaltimer_ns();
    if (tid == 0) { s_rows = 0; s_logn = 0; s_end = 0; poll = apus_consumer_poll_init(); }
    for (;;) {
        __syncthreads();                       // every thread has read the previous pass's shared words
        if (tid == 0) {
            const uint64_t now = apus_globaltimer_ns();
            uint32_t m = 0;
            if (a.ctl[0] == 1u) {
                if (a.ctl[1] == 0u) {
                    const apus_consumer_pos_t p = apus_consumer_position(v);
                    a.pos[0] = p.cursor; a.pos[1] = p.next_idx; a.pos[2] = s_rows;
                    __threadfence_system();
                    a.ctl[1] = 1u;
                }
            } else {
                s_pos = apus_consumer_position(v);
                const uint64_t n = apus_consumer_available(v, s_pos, &s_committed);
                m = (uint32_t)(n < a.max_pass ? n : a.max_pass);
                if (*(const volatile uint64_t *)v.error) s_end = RR_END_BAD_IDX;
            }
            if (s_rows >= a.target) s_end = RR_END_TARGET;
            if (now - t_start >= a.deadline_ns) s_end = RR_END_DEADLINE;
            if (apus_consumer_should_stop(v, poll)) s_end = RR_END_STOP;
            if (m == 0 && !s_end) apus_consumer_backoff(poll);
            if (m) apus_consumer_found(poll);
            s_m = s_end ? 0 : m;
            s_first_bad = 0xffffffffu;
        }
        __syncthreads();                       // hands thread 0's acquire of the record to every thread
        if (s_end) break;
        const uint32_t m = s_m;
        if (m == 0) continue;
        apus_consumer_entry_t e;
        e.status = APUS_CONS_LATER;
        if (tid < m) {
            e = apus_consumer_entry(v, s_pos, s_committed, tid);
            if (e.status != APUS_CONS_OK) atomicMin(&s_first_bad, tid);
        }
        __syncthreads();
        const uint32_t exam = m < s_first_bad ? m : s_first_bad;   // stops before an entry not committed yet, or bad
        const bool row = tid < exam && apus_has_cmd(e.type);
        const uint32_t b = __ballot_sync(0xffffffffu, row);
        if (lane == 0) s_flag[w] = __popc(b);
        __syncthreads();
        uint32_t before = 0, total = 0;
        for (uint32_t i = 0; i < RR_THREADS / 32; i++) {
            if (i < w) before += s_flag[i];
            total += s_flag[i];
        }
        const uint64_t r = s_rows + before + __popc(b & ((1u << lane) - 1u));
        const bool full = s_rows + total > a.row_cap;
        if (row && !full) {
            a.idx[r] = e.idx;
            a.types[r] = (uint8_t)e.type;
            a.conns[r] = (uint16_t)e.clt_id;
            a.req_ids[r] = e.req_id;
            a.lens[r] = (uint16_t)e.len;
            if (e.len <= a.stride) apus_consumer_copy_cmd(v, e, a.payloads + r * a.stride, 0, 1);
        }
        __syncthreads();                       // every read of the examined entries is done before the cursor moves
        if (tid == 0) {
            if (full) {
                s_end = RR_END_FULL;
            } else {
                const apus_consumer_pos_t q = apus_consumer_advance(v, s_pos, s_committed, exam);
                s_rows += total;
                *a.rows_pub = s_rows;
                if (exam && s_logn < a.log_cap) {
                    a.log[3 * s_logn] = q.cursor;
                    a.log[3 * s_logn + 1] = s_rows;
                    a.log[3 * s_logn + 2] = apus_globaltimer_ns();
                    s_logn++;
                }
                if (a.delay_ns) {
                    const uint64_t t = apus_globaltimer_ns();
                    while (apus_globaltimer_ns() - t < a.delay_ns) __nanosleep(1000);
                }
            }
        }
        __syncthreads();
        if (s_end) break;
    }
    if (tid == 0) { a.out[0] = s_end; a.out[1] = s_rows; a.out[2] = s_logn; }
}

extern "C" int rr_launch(const apus_consumer_view_t *v, const rr_args *a, void *stream)
{
    resident_rows_kernel<<<1, RR_THREADS, 0, (cudaStream_t)stream>>>(*v, *a);
    return (int)cudaGetLastError();
}

// loaded before any replica kernel is resident: a lazy load beside them may wait for them
extern "C" int rr_load(void)
{
    cudaFuncAttributes fa;
    return (int)cudaFuncGetAttributes(&fa, resident_rows_kernel);
}

extern "C" unsigned rr_args_size(void) { return (unsigned)sizeof(rr_args); }
