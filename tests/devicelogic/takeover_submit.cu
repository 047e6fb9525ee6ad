/*
 * takeover_submit.cu -- a resident submitter that lives through take-overs, for tests/test_gpu_submit_takeover.py and
 * tools/resident_failover_bench.py, written against the public headers alone.  One persistent kernel per replica,
 * launched once: on a follower its submitter is dormant and every reserve ends APUS_SUBMITTER_NOT_LEADER; the kernel
 * waits that out and writes its requests once its replica leads and the ring has been handed over.
 *
 * Any number of CTAs of TS_THREADS threads take chunks of `batch` requests in turn from a shared counter.  For each
 * chunk thread 0 sums the payload bytes and reserves, every thread puts some of its requests, and thread 0 publishes.
 * The requests lie in device memory in the packed layout (request k's cmd is values[offsets[k], offsets[k + 1])).
 *
 *   - A reserve that ends NOT_LEADER is made again after a back-off, until it ends otherwise, the stop word moves or
 *     timeout_ns has passed since the chunk began; out[3] counts those outcomes.
 *   - The stop word is also polled before every chunk, so that a closed loop faster than the poll interval ends there
 *     (STOPPED, step 1).
 *   - mode TS_WAIT: after each publish, thread 0 waits for the chunk's last ticket to commit; out[4] receives the
 *     %globaltimer ns at which the first chunk's commit was seen.
 *
 * Every wait ends within timeout_ns or on the stop word, so every launch ends by itself.  out[0] is 0, or the first
 * failure: (step << 8) | APUS_SUBMITTER_* with step 1 reserve, 2 publish, 3 commit wait; out[1] counts the requests
 * published; out[2] is the chunk counter; out[5] is what apus_submitter_leading returns as CTA 0 ends.  tickets[k]
 * receives request k's ticket once it is put, terms[chunk] the term of the chunk's reservation.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_submitter.cuh"

#define TS_THREADS 128u
#define TS_MAX_BATCH 1024u
#define TS_WAIT 1u

struct ts_args {
    const uint8_t *types;
    const uint16_t *conns;
    const uint64_t *req_ids;
    const uint64_t *offsets;       /* n + 1 */
    const uint8_t *values;
    uint64_t n;
    uint32_t batch, mode;
    uint64_t timeout_ns;
    uint64_t *tickets;             /* [n] */
    uint64_t *terms;               /* [chunks] */
    unsigned long long *out;       /* {failure, published, chunk counter, NOT_LEADER outcomes, first commit seen,
                                      leading at the end} */
};

__device__ __forceinline__ void ts_fail(const ts_args &a, uint32_t step, uint32_t outcome)
{
    atomicCAS(&a.out[0], 0ull, (unsigned long long)((step << 8) | outcome));
}

__global__ void __launch_bounds__(TS_THREADS) takeover_submit_kernel(const apus_submitter_view_t v, const ts_args a)
{
    __shared__ apus_submitter_res_t s_res;
    __shared__ apus_consumer_poll_t s_stop_poll;           // thread 0's, across chunks
    __shared__ uint64_t s_k0, s_chunk, s_t0;
    __shared__ uint32_t s_m, s_end;
    __shared__ uint32_t s_off[TS_MAX_BATCH];
    const uint32_t tid = threadIdx.x;
    const uint64_t nchunks = (a.n + a.batch - 1) / a.batch;
    if (tid == 0) s_stop_poll = apus_consumer_poll_init();
    for (;;) {
        if (tid == 0) {
            s_end = 0;
            s_chunk = atomicAdd(&a.out[2], 1ull);
            if (s_chunk >= nchunks || *(volatile unsigned long long *)&a.out[0]) {
                s_end = 1;
            } else if (apus_submitter_should_stop(v, s_stop_poll)) {
                ts_fail(a, 1, APUS_SUBMITTER_STOPPED);
                s_end = 1;
            } else {
                s_k0 = s_chunk * a.batch;
                s_m = (uint32_t)(a.n - s_k0 < a.batch ? a.n - s_k0 : a.batch);
                uint64_t xb = 0;
                for (uint32_t j = 0; j < s_m; j++) {
                    const uint64_t k = s_k0 + j;
                    s_off[j] = (uint32_t)xb;
                    xb += apus_submitter_ext_bytes(a.types[k], (uint32_t)(a.offsets[k + 1] - a.offsets[k]));
                }
                s_t0 = apus_globaltimer_ns();
                apus_consumer_poll_t p = apus_consumer_poll_init();
                for (;;) {                         // wait out NOT_LEADER: the replica does not lead yet
                    s_res = apus_submitter_reserve(v, s_m, xb, a.timeout_ns);
                    if (s_res.outcome != APUS_SUBMITTER_NOT_LEADER) break;
                    atomicAdd(&a.out[3], 1ull);
                    if (apus_submitter_should_stop(v, p)) { s_res.outcome = APUS_SUBMITTER_STOPPED; break; }
                    if (apus_globaltimer_ns() - s_t0 >= a.timeout_ns) break;
                    apus_poll_sleep(p.sleep);
                }
                if (s_res.outcome != APUS_SUBMITTER_OK) { ts_fail(a, 1, s_res.outcome); s_end = 1; }
                else a.terms[s_chunk] = s_res.term;
            }
        }
        __syncthreads();                       // hands the reservation to every thread
        if (s_end) break;
        for (uint32_t j = tid; j < s_m; j += TS_THREADS) {
            const uint64_t k = s_k0 + j;
            apus_submitter_put(v, s_res, j, s_off[j], a.types[k], a.conns[k], a.req_ids[k], a.values + a.offsets[k],
                               (uint32_t)(a.offsets[k + 1] - a.offsets[k]));
            a.tickets[k] = s_res.first_ticket + j;
        }
        __syncthreads();                       // every put of the reservation is done before the publish
        if (tid == 0) {
            const uint32_t o = apus_submitter_publish(v, s_res, a.timeout_ns);
            if (o != APUS_SUBMITTER_OK) {
                ts_fail(a, 2, o);
            } else {
                atomicAdd(&a.out[1], (unsigned long long)s_m);
                if (a.mode & TS_WAIT) {
                    const uint32_t w = apus_submitter_wait_committed(v, s_res.first_ticket + s_m - 1, a.timeout_ns);
                    if (w != APUS_SUBMITTER_OK) ts_fail(a, 3, w);
                    else if (s_chunk == 0) a.out[4] = apus_globaltimer_ns();
                }
            }
        }
        __syncthreads();                       // before thread 0 overwrites the shared words of this chunk
    }
    if (tid == 0 && blockIdx.x == 0) a.out[5] = apus_submitter_leading(v);
}

extern "C" int ts_launch(const apus_submitter_view_t *v, const ts_args *a, unsigned ctas, void *stream)
{
    takeover_submit_kernel<<<ctas, TS_THREADS, 0, (cudaStream_t)stream>>>(*v, *a);
    return (int)cudaGetLastError();
}

// loaded before any replica kernel is resident: a lazy load beside them may wait for them
extern "C" int ts_load(void)
{
    cudaFuncAttributes fa;
    return (int)cudaFuncGetAttributes(&fa, takeover_submit_kernel);
}

extern "C" unsigned ts_args_size(void) { return (unsigned)sizeof(ts_args); }
extern "C" unsigned ts_view_size(void) { return (unsigned)sizeof(apus_submitter_view_t); }
