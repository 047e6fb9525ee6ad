/*
 * header_probe.cu -- the primitives of the public device headers (include/apus_consumer.cuh, include/apus_submitter.cuh)
 * driven one by one on views whose words all lie in plain device buffers that the test fills: no replica kernel runs,
 * and nothing depends on timing.  tests/test_gpu_header_primitives.py compares every output with a reference that shares
 * no code with the headers.  Every loop here is bounded, and every submitter call that waits is given a timeout, so
 * every launch ends by itself.
 *
 *   hp_copy      one CTA per case: the `groups` groups of `nthr` threads each copy `len` bytes with apus_copy_cmd (or
 *                apus_consumer_copy_cmd), group g from src + g * len to dst + g * len (adjacent destinations).
 *   hp_loads     apus_ld_u8_any, apus_ld_u16_any and apus_ld_u64_any at every offset 0 .. 63 of a buffer.
 *   hp_consumer  one pass of the documented consumer loop in one CTA: thread 0 takes the position and what is
 *                available, entry k is examined by thread k % blockDim (and its cmd copied by it), thread 0 advances past
 *                the examined prefix -- the entries before the first one whose status is not APUS_CONS_OK -- and calls
 *                apus_consumer_available once more.
 *   hp_submit    scripted reservations: CTA b runs steps [cta_first[b], cta_first[b + 1]); a reserve (its requests put by
 *                every thread of the CTA, request k by thread k % blockDim), a publish of the CTA's latest reservation,
 *                or a commit wait.  Several CTAs run their scripts at once.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_submitter.cuh"

#define HP_COPY_THREADS 512u
#define HP_MAX_BATCH 1024u

// ---------------------------------------------------------------------------------
// copy and loads
// ---------------------------------------------------------------------------------
struct hp_copy_case {
    uint64_t src, dst;            /* byte offsets into the source and destination buffers */
    uint32_t len, nthr, groups, via;   /* via 1: apus_consumer_copy_cmd over a view whose entries are the source */
};

__global__ void __launch_bounds__(HP_COPY_THREADS) hp_copy_kernel(const uint8_t *src, uint8_t *dst, const hp_copy_case *cases)
{
    const hp_copy_case cs = cases[blockIdx.x];
    const uint32_t t = threadIdx.x;
    if (t >= cs.nthr * cs.groups) return;
    const uint32_t g = t / cs.nthr, c = t % cs.nthr;
    const uint64_t off = (uint64_t)g * cs.len;
    if (cs.via) {
        apus_consumer_view_t v = {};
        v.entries = src;
        apus_consumer_entry_t e = {};
        e.cmd_off = cs.src + off;
        e.len = cs.len;
        apus_consumer_copy_cmd(v, e, dst + cs.dst + off, c, cs.nthr);
    } else {
        apus_copy_cmd(dst + cs.dst + off, src + cs.src + off, cs.len, c, cs.nthr);
    }
}

extern "C" int hp_copy(const uint8_t *src, uint8_t *dst, const hp_copy_case *cases, uint32_t ncases, void *stream)
{
    hp_copy_kernel<<<ncases, HP_COPY_THREADS, 0, (cudaStream_t)stream>>>(src, dst, cases);
    return (int)cudaGetLastError();
}

__global__ void hp_loads_kernel(const uint8_t *buf, uint32_t *u8, uint32_t *u16, uint64_t *u64)
{
    const uint32_t at = threadIdx.x;
    u8[at] = apus_ld_u8_any(buf, at);
    u16[at] = apus_ld_u16_any(buf, at);
    u64[at] = apus_ld_u64_any(buf, at);
}

extern "C" int hp_loads(const uint8_t *buf, uint32_t *u8, uint32_t *u16, uint64_t *u64, void *stream)
{
    hp_loads_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(buf, u8, u16, u64);
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------
// consumer
// ---------------------------------------------------------------------------------
/* out: {cursor, next_idx, available, committed, examined, new cursor, new next_idx, available after the pass} */
__global__ void hp_consumer_kernel(const apus_consumer_view_t v, apus_consumer_entry_t *ents, uint32_t cap, uint8_t *rows,
                                   uint32_t stride, uint64_t *out)
{
    __shared__ apus_consumer_pos_t s_pos;
    __shared__ uint64_t s_n, s_committed;
    __shared__ unsigned long long s_stop;
    const uint32_t tid = threadIdx.x;
    if (tid == 0) {
        s_pos = apus_consumer_position(v);
        s_n = apus_consumer_available(v, s_pos, (uint64_t *)&s_committed);
        s_stop = s_n < cap ? s_n : cap;
    }
    __syncthreads();
    const uint64_t n = s_n < cap ? s_n : cap;
    for (uint64_t k = tid; k < n; k += blockDim.x) {
        const apus_consumer_entry_t e = apus_consumer_entry(v, s_pos, s_committed, k);
        ents[k] = e;
        if (e.status != APUS_CONS_OK) atomicMin(&s_stop, (unsigned long long)k);
        else if (e.len <= stride) apus_consumer_copy_cmd(v, e, rows + k * stride, 0, 1);
    }
    __syncthreads();
    if (tid == 0) {
        const apus_consumer_pos_t q = apus_consumer_advance(v, s_pos, s_committed, s_stop);
        uint64_t c2 = 0;
        const uint64_t n2 = apus_consumer_available(v, q, &c2);
        out[0] = s_pos.cursor; out[1] = s_pos.next_idx; out[2] = s_n; out[3] = s_committed;
        out[4] = s_stop; out[5] = q.cursor; out[6] = q.next_idx; out[7] = n2;
    }
}

extern "C" int hp_consumer(const apus_consumer_view_t *v, apus_consumer_entry_t *ents, uint32_t cap, uint8_t *rows,
                           uint32_t stride, uint64_t *out, uint32_t threads, void *stream)
{
    hp_consumer_kernel<<<1, threads, 0, (cudaStream_t)stream>>>(*v, ents, cap, rows, stride, out);
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------
// submitter
// ---------------------------------------------------------------------------------
#define HP_RESERVE 1u
#define HP_PUBLISH 2u
#define HP_WAIT    3u
#define HP_PUT     1u                  /* reserve flag: put the requests req0 .. req0 + n - 1 */
#define HP_EXT_OF_REQUESTS (~0ull)     /* reserve ext: the sum of apus_submitter_ext_bytes of the requests */
#define HP_SKIPPED 0xffu               /* a publish with no reservation to publish */

struct hp_req {
    uint32_t type, conn, len, pad;
    uint64_t req_id, cmd_off;          /* the cmd is cmds + cmd_off */
};
struct hp_step {
    uint32_t op, n, req0, flags;
    uint64_t ext, timeout_ns, ticket;  /* ticket: HP_WAIT */
};
struct hp_out {                        /* per step */
    uint64_t outcome, first_ticket, pos, n, wrap, order, pad0, pad1;
};

__global__ void hp_submit_kernel(const apus_submitter_view_t v, const hp_step *steps, const uint32_t *cta_first,
                                 const hp_req *reqs, const uint8_t *cmds, hp_out *out, unsigned long long *order)
{
    __shared__ apus_submitter_res_t s_res;
    __shared__ hp_step s_step;
    __shared__ uint32_t s_have;
    __shared__ uint32_t s_off[HP_MAX_BATCH];
    const uint32_t tid = threadIdx.x;
    if (tid == 0) s_have = 0;
    for (uint32_t i = cta_first[blockIdx.x]; i < cta_first[blockIdx.x + 1]; i++) {
        if (tid == 0) {
            s_step = steps[i];
            hp_out o = {};
            if (s_step.op == HP_RESERVE) {
                uint64_t xb = s_step.ext;
                if (xb == HP_EXT_OF_REQUESTS) {
                    xb = 0;
                    for (uint32_t j = 0; j < s_step.n && j < HP_MAX_BATCH; j++) {
                        const hp_req r = reqs[s_step.req0 + j];
                        s_off[j] = (uint32_t)xb;
                        xb += apus_submitter_ext_bytes(r.type, r.len);
                    }
                }
                s_res = apus_submitter_reserve(v, s_step.n, xb, s_step.timeout_ns);
                s_have = s_res.outcome == APUS_SUBMITTER_OK;
                o.outcome = s_res.outcome; o.first_ticket = s_res.first_ticket; o.pos = s_res.pos; o.n = s_res.n;
                o.wrap = s_res.wrap;
            } else if (s_step.op == HP_PUBLISH) {
                if (s_have) {
                    o.outcome = apus_submitter_publish(v, s_res, s_step.timeout_ns);
                    o.first_ticket = s_res.first_ticket;
                    o.n = s_res.n;
                    if (o.outcome == APUS_SUBMITTER_OK) o.order = atomicAdd(order, 1ull);
                } else {
                    o.outcome = HP_SKIPPED;
                }
            } else if (s_step.op == HP_WAIT) {
                o.outcome = apus_submitter_wait_committed(v, s_step.ticket, s_step.timeout_ns);
            }
            out[i] = o;
        }
        __syncthreads();                       // hands the reservation to every thread
        if (s_step.op == HP_RESERVE && (s_step.flags & HP_PUT) && s_have) {
            for (uint32_t k = tid; k < s_res.n; k += blockDim.x) {
                const hp_req r = reqs[s_step.req0 + k];
                apus_submitter_put(v, s_res, k, s_off[k], r.type, r.conn, r.req_id, cmds + r.cmd_off, r.len);
            }
        }
        __syncthreads();                       // every put is done before thread 0 takes the next step
    }
}

extern "C" int hp_submit(const apus_submitter_view_t *v, const hp_step *steps, const uint32_t *cta_first, const hp_req *reqs,
                         const uint8_t *cmds, hp_out *out, unsigned long long *order, uint32_t ctas, uint32_t threads,
                         void *stream)
{
    hp_submit_kernel<<<ctas, threads, 0, (cudaStream_t)stream>>>(*v, steps, cta_first, reqs, cmds, out, order);
    return (int)cudaGetLastError();
}

extern "C" unsigned hp_sizes(unsigned which)
{
    switch (which) {
    case 0: return (unsigned)sizeof(hp_copy_case);
    case 1: return (unsigned)sizeof(apus_consumer_entry_t);
    case 2: return (unsigned)sizeof(hp_req);
    case 3: return (unsigned)sizeof(hp_step);
    case 4: return (unsigned)sizeof(hp_out);
    case 5: return (unsigned)sizeof(apus_consumer_view_t);
    case 6: return (unsigned)sizeof(apus_submitter_view_t);
    default: return 0;
    }
}
