/*
 * resident_submit.cu -- a resident submitter for the tests and tools/resident_submitter_bench.py, written against the
 * public headers alone: any number of CTAs of RS_THREADS threads take chunks of `batch` requests in turn from a shared
 * counter.  For each chunk thread 0 sums the payload bytes and reserves, every thread puts some of its requests, and
 * thread 0 publishes, so that several CTAs reserve, put and publish concurrently and the tickets interleave by chunk.
 * The requests lie in device memory in the packed layout (request k's cmd is values[offsets[k], offsets[k + 1])).
 *
 * mode RS_WAIT: after each publish, thread 0 waits for the chunk's last ticket to commit and records the device time
 * from before its reserve to the commit seen (lat_ns[chunk]).  mode RS_DROP_LAST: the last chunk is reserved and put but
 * never published (a single-CTA launch only: the chunks after it could never publish).
 * Every reserve, publish and commit wait ends within timeout_ns, so every launch ends by itself.  out[0] is 0, or the
 * first failure: (step << 8) | APUS_SUBMITTER_* with step 1 reserve, 2 publish, 3 commit wait; out[1] counts the
 * requests published; out[2] is the chunk counter; out[3..6] sum, over the CTAs, thread 0's %globaltimer ns in each
 * phase of a chunk: the size sum, the reserve, the puts (from the reserve to the barrier after them) and the publish.
 * tickets[k] receives request k's ticket once it is put.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_submitter.cuh"

#define RS_THREADS 128u
#define RS_MAX_BATCH 1024u
#define RS_WAIT      1u
#define RS_DROP_LAST 2u

struct rs_args {
    const uint8_t *types;
    const uint16_t *conns;
    const uint64_t *req_ids;
    const uint64_t *offsets;       /* n + 1 */
    const uint8_t *values;
    uint64_t n;
    uint32_t batch, mode;
    uint64_t timeout_ns;
    uint64_t *tickets;             /* [n] */
    uint64_t *lat_ns;              /* [chunks] (RS_WAIT) */
    unsigned long long *out;       /* {failure, published, chunk counter, ns: size sum, reserve, puts, publish} */
};

__device__ __forceinline__ void rs_fail(const rs_args &a, uint32_t step, uint32_t outcome)
{
    atomicCAS(&a.out[0], 0ull, (unsigned long long)((step << 8) | outcome));
}

__global__ void __launch_bounds__(RS_THREADS) resident_submit_kernel(const apus_submitter_view_t v, const rs_args a)
{
    __shared__ apus_submitter_res_t s_res;
    __shared__ uint64_t s_k0, s_t0, s_chunk;
    __shared__ uint32_t s_m, s_end;
    __shared__ uint32_t s_off[RS_MAX_BATCH];
    const uint32_t tid = threadIdx.x;
    const uint64_t nchunks = (a.n + a.batch - 1) / a.batch;
    uint64_t t_sum = 0, t_res = 0, t_put = 0, t_pub = 0, t_mark = 0;   // thread 0's phase clocks
    for (;;) {
        if (tid == 0) {
            t_mark = apus_globaltimer_ns();
            s_end = 0;
            s_chunk = atomicAdd(&a.out[2], 1ull);
            if (s_chunk >= nchunks || *(volatile unsigned long long *)&a.out[0]) {
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
                t_sum += s_t0 - t_mark;
                s_res = apus_submitter_reserve(v, s_m, xb, a.timeout_ns);
                t_mark = apus_globaltimer_ns();
                t_res += t_mark - s_t0;
                if (s_res.outcome != APUS_SUBMITTER_OK) { rs_fail(a, 1, s_res.outcome); s_end = 1; }
            }
        }
        __syncthreads();                       // hands the reservation to every thread
        if (s_end) break;
        for (uint32_t j = tid; j < s_m; j += RS_THREADS) {
            const uint64_t k = s_k0 + j;
            apus_submitter_put(v, s_res, j, s_off[j], a.types[k], a.conns[k], a.req_ids[k], a.values + a.offsets[k],
                               (uint32_t)(a.offsets[k + 1] - a.offsets[k]));
            a.tickets[k] = s_res.first_ticket + j;
        }
        __syncthreads();                       // every put of the reservation is done before the publish
        if (tid == 0) {
            const uint64_t t = apus_globaltimer_ns();
            t_put += t - t_mark;
            t_mark = t;
        }
        if (tid == 0 && !((a.mode & RS_DROP_LAST) && s_chunk + 1 == nchunks)) {
            const uint32_t o = apus_submitter_publish(v, s_res, a.timeout_ns);
            t_pub += apus_globaltimer_ns() - t_mark;
            if (o != APUS_SUBMITTER_OK) {
                rs_fail(a, 2, o);
            } else {
                atomicAdd(&a.out[1], (unsigned long long)s_m);
                if (a.mode & RS_WAIT) {
                    const uint32_t w = apus_submitter_wait_committed(v, s_res.first_ticket + s_m - 1, a.timeout_ns);
                    if (w != APUS_SUBMITTER_OK) rs_fail(a, 3, w);
                    else a.lat_ns[s_chunk] = apus_globaltimer_ns() - s_t0;
                }
            }
        }
        __syncthreads();                       // before thread 0 overwrites the shared words of this chunk
    }
    if (tid == 0) {
        atomicAdd(&a.out[3], (unsigned long long)t_sum);
        atomicAdd(&a.out[4], (unsigned long long)t_res);
        atomicAdd(&a.out[5], (unsigned long long)t_put);
        atomicAdd(&a.out[6], (unsigned long long)t_pub);
    }
}

extern "C" int rs_launch(const apus_submitter_view_t *v, const rs_args *a, unsigned ctas, void *stream)
{
    resident_submit_kernel<<<ctas, RS_THREADS, 0, (cudaStream_t)stream>>>(*v, *a);
    return (int)cudaGetLastError();
}

// loaded before any replica kernel is resident: a lazy load beside them may wait for them
extern "C" int rs_load(void)
{
    cudaFuncAttributes fa;
    return (int)cudaFuncGetAttributes(&fa, resident_submit_kernel);
}

extern "C" unsigned rs_args_size(void) { return (unsigned)sizeof(rs_args); }
extern "C" unsigned rs_view_size(void) { return (unsigned)sizeof(apus_submitter_view_t); }
