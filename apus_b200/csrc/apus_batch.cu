/*
 * apus_batch.cu -- the stream-ordered batch kernels: short launches on a replica's side streams that run beside the
 * resident replica kernel (apus_kernels.cu) and exchange requests and committed entries with buffers in device memory.
 *
 *   synth    apus_submit_synth: device-generated requests written into the HBM submission ring
 *   pack     apus_submit_device / apus_submit_device_packed: sizes, scan and pack passes, then the doorbell (bell)
 *   consume  apus_consume_device / apus_consume_device_packed: head, count, scan, copy and tail
 *   wait     apus_consume_wait: one warp between consume calls, until enough entries are committed past the cursor
 *   mark     apus_consume_mark: one thread writes the consumer position, for a snapshot of the application's state
 *   fence    apus_read_fence: one warp until this replica's state can answer a linearizable read (apus_reader.cuh)
 *
 * apus_engine.cu checks the arguments, accounts ring space, and brackets each enqueue below in the caller's stream
 * order.  The batch layouts are apus_layout.h; the slot format is apus_slot.h; the device helpers shared with the
 * replica kernel are apus_dev.h.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_gpu.h"
#include "apus_layout.h"
#include "apus_slot.h"
#include "apus_dev.h"
#include "apus_fence.h"
#include "apus_reader.cuh"

// ---------------------------------------------------------------------------------
// block scans: the packing and the consume kernels run blocks of the same size
// ---------------------------------------------------------------------------------
static_assert(APUS_PACK_THREADS == APUS_CONS_THREADS, "the packing and the consume kernels share one block scan");

// inclusive sum over the block (APUS_PACK_THREADS == APUS_CONS_THREADS threads) of v; *total = the block's sum
__device__ __forceinline__ uint64_t block_incl_sum(uint64_t v, uint64_t *total)
{
    __shared__ uint64_t warp_sum[APUS_CONS_THREADS / 32];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const uint64_t o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += o;
    }
    if (lane == 31) warp_sum[w] = v;
    __syncthreads();
    uint64_t before = 0, all = 0;
    for (uint32_t i = 0; i < APUS_CONS_THREADS / 32; i++) {
        if (i < w) before += warp_sum[i];
        all += warp_sum[i];
    }
    __syncthreads();
    *total = all;
    return before + v;
}

// exclusive prefix count of `flag` over the block (APUS_CONS_THREADS threads); *total = the block's count
__device__ __forceinline__ uint32_t cons_block_excl(bool flag, uint32_t *total)
{
    __shared__ uint32_t warp_n[APUS_CONS_THREADS / 32];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint32_t b = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) warp_n[w] = __popc(b);
    __syncthreads();
    uint32_t before = 0, all = 0;
    for (uint32_t i = 0; i < APUS_CONS_THREADS / 32; i++) {
        if (i < w) before += warp_n[i];
        all += warp_n[i];
    }
    __syncthreads();
    *total = all;
    return before + __popc(b & ((1u << lane) - 1u));
}

// ---------------------------------------------------------------------------------
// device-generated requests (apus_submit_synth)
// ---------------------------------------------------------------------------------
__global__ void apus_synth_kernel(apus_slot_t *ring, uint32_t mask, uint8_t *pay, uint64_t first_slot, uint32_t n,
                                  uint32_t type, uint32_t conn, uint64_t first_req, uint32_t len, uint32_t seed,
                                  uint64_t pay_pos0, uint32_t need, uint32_t first_flags)
{
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const uint64_t s = first_slot + k, req = first_req + k;
        apus_slot_t *d = &ring[s & mask];
        const uint32_t nb = slot_image_bytes(type, len);
        uint32_t type_off;
        if (need) {
            const uint64_t pos = pay_pos0 + (uint64_t)k * need;
            type_off = slot_type_off(type, APUS_SLOT_EXT | (k == 0 ? first_flags : 0u), pos);
            uint8_t *p = pay + pos;
            p[0] = (uint8_t)len; p[1] = (uint8_t)(len >> 8);
            for (uint32_t q = 0; q < len; q++) p[2 + q] = synth_byte(seed, req, q);
        } else {
            type_off = slot_type_off(type, 0, 0);
            uint8_t *sb = reinterpret_cast<uint8_t *>(d);
            for (uint32_t q = 0; q < nb; q++)
                sb[slot_inline_off(q)] = q == 0 ? (uint8_t)len : q == 1 ? (uint8_t)(len >> 8) : synth_byte(seed, req, q - 2);
        }
        d->rsv0 = 0; d->rsv1 = 0;
        slot_finish(d, s + 1, type_off, (uint16_t)conn, req, (uint16_t)len);
    }
}

// ---------------------------------------------------------------------------------
// device batches (apus_submit_device, apus_submit_device_packed): requests in device memory, packed into the HBM ring
// in stream order
// ---------------------------------------------------------------------------------
/* what request k becomes -- its own type and length, or the NOOP that apus_submit(APUS_NOOP, conn, req_id, NULL, 0)
 * writes when the type is not a request type, the length is above the limit (stride, or 65535 packed) or the packed
 * batch is `bad` -- and where its cmd starts in payloads, in either layout */
__device__ __forceinline__ bool pack_request(const apus_pack_args_t &a, uint32_t k, bool bad, uint32_t *type, uint32_t *len,
                                             uint64_t *src)
{
    const uint32_t ty = a.types[k];
    uint64_t ln, at;
    if (a.offsets) { at = a.offsets[k]; ln = a.offsets[k + 1] - at; }
    else { at = (uint64_t)k * a.stride; ln = a.lens[k]; }
    const bool ok = (ty == APUS_CSM || ty == APUS_CONNECT || ty == APUS_SEND || ty == APUS_CLOSE) && !bad &&
                    ln <= (a.offsets ? 0xffffull : a.stride);
    *type = ok ? ty : (uint32_t)APUS_NOOP;
    *len = ok ? (uint32_t)ln : 0u;
    *src = at;
    return ok;
}

/* the packed layout's per-request share of the batch verdict: offsets[k] <= offsets[k + 1] <= values_bytes for every
 * k is exactly "nondecreasing, and inside values"; valid lengths of such a batch stay inside its reservation */
__device__ __forceinline__ bool pack_offsets_bad(const apus_pack_args_t &a, uint32_t k)
{
    return a.offsets && (a.offsets[k + 1] < a.offsets[k] || a.offsets[k + 1] > a.values_bytes);
}

/* pass 1: per block, the payload-ring bytes of its external images and its rejected requests */
__global__ void __launch_bounds__(APUS_PACK_THREADS) apus_pack_sizes_kernel(apus_pack_args_t a)
{
    __shared__ unsigned long long first_rej;
    const uint32_t k = blockIdx.x * APUS_PACK_THREADS + threadIdx.x;
    if (threadIdx.x == 0) first_rej = ~0ull;
    __syncthreads();
    uint32_t ty = 0, len = 0;
    bool rej = false, bad = false;
    uint64_t xb = 0, src;
    if (k < a.n) {
        rej = !pack_request(a, k, false, &ty, &len, &src);
        bad = pack_offsets_bad(a, k);
        xb = slot_ext_bytes(slot_image_bytes(ty, len));
        if (rej) atomicMin(&first_rej, (unsigned long long)k);
    }
    const uint32_t nrej = __syncthreads_count(rej);
    const uint32_t nbad = __syncthreads_count(bad);
    uint64_t total;
    block_incl_sum(xb, &total);
    if (threadIdx.x == 0) {
        a.blk[APUS_PACK_BLK_WORDS * blockIdx.x] = total;
        a.blk[APUS_PACK_BLK_WORDS * blockIdx.x + 1] = nrej;
        a.blk[APUS_PACK_BLK_WORDS * blockIdx.x + 2] = first_rej;
        a.blk[APUS_PACK_BLK_WORDS * blockIdx.x + 3] = nbad != 0;
    }
}

/* pass 2 (one block): the batch verdict of the packed layout (a bad batch is all NOOPs: no external bytes, every
 * request rejected), handed to every block; exclusive scan of the blocks' external bytes, in place; the batch's
 * rejections into the host words.  The verdict is final before pass 3 writes any slot. */
__global__ void __launch_bounds__(APUS_PACK_THREADS) apus_pack_scan_kernel(apus_pack_args_t a, uint32_t nblk, apus_hostwords_t *hw)
{
    __shared__ unsigned long long first_rej;
    __shared__ unsigned int nrej;
    uint64_t *blk = a.blk;
    bool mine = false;
    if (a.offsets)
        for (uint32_t b = threadIdx.x; b < nblk; b += APUS_PACK_THREADS) mine |= blk[APUS_PACK_BLK_WORDS * b + 3] != 0;
    const bool bad = __syncthreads_or(mine) != 0;
    if (threadIdx.x == 0) { first_rej = bad ? 0ull : ~0ull; nrej = bad ? a.n : 0u; }
    __syncthreads();
    uint64_t carry = 0;
    for (uint32_t b0 = 0; b0 < nblk; b0 += APUS_PACK_THREADS) {
        const uint32_t b = b0 + threadIdx.x;
        const uint64_t v = b < nblk && !bad ? blk[APUS_PACK_BLK_WORDS * b] : 0;
        if (b < nblk && !bad && blk[APUS_PACK_BLK_WORDS * b + 1]) {
            atomicAdd(&nrej, (unsigned int)blk[APUS_PACK_BLK_WORDS * b + 1]);
            atomicMin(&first_rej, (unsigned long long)blk[APUS_PACK_BLK_WORDS * b + 2]);
        }
        uint64_t total;
        const uint64_t incl = block_incl_sum(v, &total);
        if (b < nblk) {
            blk[APUS_PACK_BLK_WORDS * b] = carry + incl - v;
            blk[APUS_PACK_BLK_WORDS * b + 3] = bad;
        }
        carry += total;
    }
    __syncthreads();
    if (threadIdx.x == 0 && nrej) {
        hw->dev_rejected += nrej;                 /* one writer: the batches run one after another on copy_stream */
        if (!hw->dev_first_rejected) hw->dev_first_rejected = a.first_slot + first_rej + 1;
    }
}

/* bytes [16q, 16q + 16) of the data image {u16 len; cmd[len]} of a request whose command is at src */
__device__ __forceinline__ uint4 image_chunk(const uint8_t *src, uint32_t len, uint32_t nb, uint32_t q)
{
    uint32_t w[4] = {0, 0, 0, 0};
    for (uint32_t i = 0; i < 16; i++) {
        const uint32_t j = 16u * q + i;
        uint32_t v = 0;
        if (j == 0) v = len & 0xffu;
        else if (j == 1) v = len >> 8;
        else if (j < nb) v = __ldg(src + (j - 2));
        w[i >> 2] |= v << (8u * (i & 3u));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

/* pass 3: each block packs its APUS_PACK_THREADS requests.  A thread per request finds its external offset (block scan +
 * the block's offset from pass 2); then eight threads per slot write its 16 B chunks -- descriptor, inline image or
 * external image chunks -- and, last, the two stamp chunks. */
__global__ void __launch_bounds__(APUS_PACK_THREADS) apus_pack_kernel(apus_pack_args_t a)
{
    __shared__ uint32_t s_type_off[APUS_PACK_THREADS], s_len[APUS_PACK_THREADS], s_nb[APUS_PACK_THREADS];
    __shared__ uint64_t s_pos[APUS_PACK_THREADS], s_src[APUS_PACK_THREADS];
    const uint32_t kb = blockIdx.x * APUS_PACK_THREADS;
    {
        const uint32_t k = kb + threadIdx.x;
        uint32_t ty = 0, len = 0, nb = 0;
        uint64_t src = 0;
        if (k < a.n) {
            pack_request(a, k, a.blk[APUS_PACK_BLK_WORDS * blockIdx.x + 3] != 0, &ty, &len, &src);
            nb = slot_image_bytes(ty, len);
        }
        const uint64_t xb = slot_ext_bytes(nb);
        uint64_t total;
        const uint64_t off = a.blk[APUS_PACK_BLK_WORDS * blockIdx.x] + block_incl_sum(xb, &total) - xb;
        const uint64_t pos = a.res_pos + off;
        /* the first external image of the batch starts the reservation: a discontinuity for the leader */
        s_type_off[threadIdx.x] = slot_type_off(ty, xb ? (APUS_SLOT_EXT | (off == 0 ? APUS_SLOT_WRAP : 0u)) : 0u, pos);
        s_len[threadIdx.x] = len;
        s_nb[threadIdx.x] = nb;
        s_pos[threadIdx.x] = pos;
        s_src[threadIdx.x] = src;
    }
    __syncthreads();
    const uint32_t c = threadIdx.x & 7u;
    for (uint32_t i = threadIdx.x >> 3; i < APUS_PACK_THREADS; i += APUS_PACK_THREADS / 8) {
        const uint32_t k = kb + i;
        const bool live = k < a.n;                     /* (every lane runs the same iterations: __syncwarp below) */
        const uint64_t ticket = a.first_slot + k + 1;
        uint4 *d = reinterpret_cast<uint4 *>(&a.ring[(a.first_slot + k) & a.mask]);
        const uint32_t to = s_type_off[i], len = s_len[i], nb = s_nb[i];
        const uint8_t *src = a.payloads + s_src[i];
        if (live && c == 0) {
            uint32_t w[4];
            slot_desc_words(w, a.req_ids[k], to, len, a.conns[k]);
            d[0] = make_uint4(w[0], w[1], w[2], w[3]);
        }
        if (live && (to & APUS_SLOT_EXT)) {
            uint4 *p = reinterpret_cast<uint4 *>(a.pay + s_pos[i]);
            for (uint32_t q = c; 16u * q < nb; q += 8) p[q] = image_chunk(src, len, nb, q);
        } else if (live && c != 0 && c != 3 && c != 7) {
            const uint32_t q = c < 3 ? c - 1 : c - 2;                      /* slot_inline_chunk(q) == c */
            d[c] = image_chunk(src, len, nb, q);
        }
        __syncwarp();
        if (live && (c == 3 || c == 7)) d[c] = make_uint4((uint32_t)ticket, (uint32_t)(ticket >> 32), 0u, 0u);
    }
}

/* the doorbell of a device batch, after its slots and payload in copy_stream order; the value was fixed at enqueue */
__global__ void apus_bell_kernel(uint64_t *bell, uint64_t upto)
{
    __threadfence_system();
    *(volatile uint64_t *)bell = upto;
}

// ---------------------------------------------------------------------------------
// DEVICE CONSUMERS (APUS_F_DEVICE_APPLY): the work of one apus_consume_device or apus_consume_device_packed call, five
// kernels in stream order on the replica's consume stream -- head (snapshot the record and the cursor), count (per
// block: rows, their cmd bytes and the first entry that stops the examination), scan (where the examination stops, row
// and byte offsets, the new cursor), copy (the rows), tail (the row count and the packed byte total, then the cursor
// and the status words).  A strided call stops before a cmd longer than its stride; a packed call stops before the
// first cmd that would end past values_cap, which depends on the running byte sum of the rows before it.  Entries are
// found through the offset index, never by walking bytes; they never wrap (the ghost-header rule places them at 0), so
// each cmd is one contiguous run.
// ---------------------------------------------------------------------------------
#define CONS_OK        APUS_CONS_OK
#define CONS_LATER     APUS_CONS_LATER    // not committed (yet): the examination ends here, quietly
#define CONS_BAD_IDX   APUS_CONS_BAD      // the entry at the index word does not carry the expected idx
#define CONS_TOO_LONG  3u    // CSM-like with a cmd longer than the row stride (strided calls)
#define CONS_NONE      0xffffffffu

struct ConsEntry {
    uint64_t off;
    uint32_t ty, len, status;
};
// entry j of this call: its offset from the index word, then whether it is committed (within [cursor, committed) of
// the one lap the cursor bounds), carries idx next_idx + j, and fits a row (strided calls; a packed call's capacity
// stop is the scan kernel's)
__device__ __forceinline__ ConsEntry cons_classify(const apus_consume_args_t &a, const apus_cons_state_t &s, uint64_t j)
{
    ConsEntry e = {0, 0, 0, CONS_OK};
    e.status = apus_cons_locate(a.region + a.entries_off, reinterpret_cast<const uint32_t *>(a.region + APUS_INDEX_OFF),
                                a.idx_mask, a.log_len, s.cursor, s.committed, s.next_idx + j, &e.off, &e.ty, &e.len);
    if (e.status == CONS_OK && !a.offsets && e.len > a.stride) e.status = CONS_TOO_LONG;   // (len is 0 without a cmd)
    return e;
}

// 1: snapshot the record (acquire: the entry bytes and index words it covers are visible from here on) and the cursor
__global__ void apus_consume_head_kernel(apus_consume_args_t a)
{
    apus_cons_state_t *s = a.st;
    const apus_ctrl_t *ctrl = reinterpret_cast<const apus_ctrl_t *>(a.region);
    uint64_t committed, held;
    apus_cons_read(ctrl->cons_rec, committed, held);
    const uint64_t cursor = apus_ld_relaxed_sys(&ctrl->cons_cur[0]), nidx = apus_ld_relaxed_sys(&ctrl->cons_cur[1]);
    const uint64_t avail = apus_cons_avail(held, nidx);
    s->cursor = cursor; s->next_idx = nidx; s->committed = committed;
    s->m = s->error ? 0 : (avail < a.max_n ? avail : a.max_n);
}

// 2: per block, the CSM-like entries before the block's first stop, that stop {j, reason, len}, and (packed) the cmd
// bytes of those entries
__global__ void __launch_bounds__(APUS_CONS_THREADS) apus_consume_count_kernel(apus_consume_args_t a)
{
    __shared__ uint32_t first;
    const apus_cons_state_t s = *a.st;
    const uint64_t j = (uint64_t)blockIdx.x * APUS_CONS_THREADS + threadIdx.x;
    if (threadIdx.x == 0) first = CONS_NONE;
    __syncthreads();
    ConsEntry e = {0, 0, 0, CONS_LATER};
    if (j < s.m) e = cons_classify(a, s, j);
    if (j < s.m && e.status != CONS_OK) atomicMin(&first, (uint32_t)j);
    __syncthreads();
    const bool row = j < s.m && e.status == CONS_OK && apus_has_cmd(e.ty) && j < first;
    const uint32_t rows = __syncthreads_count(row);
    uint64_t *blk = reinterpret_cast<uint64_t *>(a.st + 1) + APUS_CONS_BLK_WORDS * blockIdx.x;
    if (threadIdx.x == 0) blk[0] = rows;
    if (first == CONS_NONE) {
        if (threadIdx.x == 0) blk[1] = CONS_NONE;
    } else if (j == first) {
        blk[1] = (uint64_t)first | ((uint64_t)e.status << 32) | ((uint64_t)e.len << 40);
    }
    if (a.offsets) {
        uint64_t bytes;
        block_incl_sum(row ? e.len : 0u, &bytes);
        if (threadIdx.x == 0) blk[2] = bytes;
    }
}

// 3 (one block): the first block with a stop ends the examination; exclusive scan of the rows of the blocks up to it,
// in place; the examined count, the row count and the new cursor (end of the last examined entry, E1: L is 0).
// Packed: exclusive scan of the blocks' cmd bytes, in place; a block whose rows end past values_cap ends the
// examination too, if it comes first, and inside it the entries are classified again to find the first cmd that ends
// past values_cap -- the examination stops just before it.
__global__ void __launch_bounds__(APUS_CONS_THREADS) apus_consume_scan_kernel(apus_consume_args_t a)
{
    __shared__ uint32_t bstop, bcap, tcap;
    __shared__ uint64_t s_bytes, s_need;
    apus_cons_state_t *s = a.st;
    uint64_t *blk = reinterpret_cast<uint64_t *>(s + 1);
    const uint32_t nblk = (uint32_t)((s->m + APUS_CONS_THREADS - 1) / APUS_CONS_THREADS);
    if (threadIdx.x == 0) { bstop = CONS_NONE; bcap = CONS_NONE; tcap = CONS_NONE; s_bytes = 0; s_need = 0; }
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < nblk; b += APUS_CONS_THREADS)
        if (blk[APUS_CONS_BLK_WORDS * b + 1] != CONS_NONE) atomicMin(&bstop, b);
    __syncthreads();
    uint32_t last = bstop == CONS_NONE ? nblk : bstop + 1;           // blocks whose rows count
    if (a.offsets) {
        uint64_t carry = 0;
        for (uint32_t b0 = 0; b0 < last; b0 += APUS_CONS_THREADS) {
            const uint32_t b = b0 + threadIdx.x;
            const uint64_t v = b < last ? blk[APUS_CONS_BLK_WORDS * b + 2] : 0;
            uint64_t total;
            const uint64_t incl = block_incl_sum(v, &total);
            if (b < last) {
                blk[APUS_CONS_BLK_WORDS * b + 2] = carry + incl - v;
                if (carry + incl > a.values_cap) atomicMin(&bcap, b);
            }
            carry += total;
        }
        __syncthreads();
        if (bcap == CONS_NONE) {
            if (threadIdx.x == 0) s_bytes = carry;
        } else {
            // every block before bcap ends inside values_cap, and bcap's own stop (if any) comes after its capacity
            // stop: the bytes the count kernel summed end before that own stop
            last = bcap + 1;
            const uint64_t j = (uint64_t)bcap * APUS_CONS_THREADS + threadIdx.x;
            const uint64_t own = blk[APUS_CONS_BLK_WORDS * bcap + 1], base = blk[APUS_CONS_BLK_WORDS * bcap + 2];
            ConsEntry e = {0, 0, 0, CONS_LATER};
            if (j < s->m && j < (uint32_t)own) e = cons_classify(a, *s, j);
            const uint64_t v = e.status == CONS_OK && apus_has_cmd(e.ty) ? e.len : 0u;
            uint64_t total;
            const uint64_t incl = block_incl_sum(v, &total);
            if (base + incl > a.values_cap && v) atomicMin(&tcap, threadIdx.x);
            __syncthreads();
            if (threadIdx.x == tcap) { s_bytes = base + incl - v; s_need = v; }
        }
    }
    uint64_t carry = 0;
    for (uint32_t b0 = 0; b0 < last; b0 += APUS_CONS_THREADS) {
        const uint32_t b = b0 + threadIdx.x;
        const uint64_t v = b < last ? blk[APUS_CONS_BLK_WORDS * b] : 0;
        uint64_t total;
        const uint64_t incl = block_incl_sum(v, &total);
        if (b < last) blk[APUS_CONS_BLK_WORDS * b] = carry + incl - v;
        carry += total;
    }
    // rows of the capacity block before its stop (every thread: the count is block-wide)
    uint32_t cap_rows = 0;
    if (bcap != CONS_NONE) {
        const uint64_t j = (uint64_t)bcap * APUS_CONS_THREADS + threadIdx.x;
        ConsEntry e = {0, 0, 0, CONS_LATER};
        if (threadIdx.x < tcap) e = cons_classify(a, *s, j);
        cap_rows = __syncthreads_count(threadIdx.x < tcap && e.status == CONS_OK && apus_has_cmd(e.ty));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t n_exam = s->m, need = 0, rows = carry;
        if (bcap != CONS_NONE) {
            n_exam = (uint64_t)bcap * APUS_CONS_THREADS + tcap;
            rows = blk[APUS_CONS_BLK_WORDS * bcap] + cap_rows;
            if (rows == 0) need = s_need;                         // the call's first row: report the bytes it needs
        } else if (bstop != CONS_NONE) {
            const uint64_t w = blk[APUS_CONS_BLK_WORDS * bstop + 1];
            const uint32_t why = (uint32_t)(w >> 32) & 0xffu;
            n_exam = (uint32_t)w;
            if (why == CONS_BAD_IDX) s->error = APUS_CONSUME_BAD_IDX;
            if (why == CONS_TOO_LONG) need = (w >> 40) & 0xffffu;
        }
        uint64_t cur = s->cursor;
        if (n_exam) {
            const ConsEntry e = cons_classify(a, *s, n_exam - 1);
            cur = apus_cons_cursor_after(e.off, e.ty, e.len, a.log_len);
        }
        s->rows = rows; s->n_exam = n_exam; s->new_cursor = cur; s->need_stride = need; s->bytes = s_bytes;
    }
}

// 4: each block writes the rows of its entries (j < examined): one thread per entry for the fields, then eight
// threads per entry for the cmd bytes -- at row * stride, or (packed) at the row's byte offset: the block's byte base
// plus the cmd bytes of the rows before it in the block
__global__ void __launch_bounds__(APUS_CONS_THREADS) apus_consume_copy_kernel(apus_consume_args_t a)
{
    __shared__ uint64_t s_off[APUS_CONS_THREADS], s_dst[APUS_CONS_THREADS];
    __shared__ uint32_t s_len[APUS_CONS_THREADS];
    const apus_cons_state_t s = *a.st;
    const uint64_t *blk = reinterpret_cast<const uint64_t *>(a.st + 1) + APUS_CONS_BLK_WORDS * blockIdx.x;
    const uint8_t *entries = a.region + a.entries_off;
    if ((uint64_t)blockIdx.x * APUS_CONS_THREADS >= s.n_exam) return;          // the whole block is past the stop
    const uint64_t j = (uint64_t)blockIdx.x * APUS_CONS_THREADS + threadIdx.x;
    ConsEntry e = {0, 0, 0, CONS_LATER};
    if (j < s.n_exam) e = cons_classify(a, s, j);
    const bool live = j < s.n_exam && apus_has_cmd(e.ty);
    uint32_t tot;
    const uint64_t row = blk[0] + cons_block_excl(live, &tot);
    uint64_t dst = row * a.stride;
    if (a.offsets) {
        const uint64_t v = live ? e.len : 0u;
        uint64_t total;
        dst = blk[2] + block_incl_sum(v, &total) - v;
    }
    if (live) {
        a.idx[row] = s.next_idx + j;
        a.types[row] = (uint8_t)e.ty;
        a.conns[row] = (uint16_t)apus_ld_u16_any(entries, e.off + E_CLTID);
        a.req_ids[row] = apus_ld_u64_any(entries, e.off + E_REQID);
        if (a.offsets) a.offsets[row] = dst;
        else a.lens[row] = (uint16_t)e.len;
    }
    s_off[threadIdx.x] = e.off; s_dst[threadIdx.x] = dst; s_len[threadIdx.x] = live ? e.len : CONS_NONE;
    __syncthreads();
    const uint32_t c = threadIdx.x & 7u;
    for (uint32_t i = threadIdx.x >> 3; i < APUS_CONS_THREADS; i += APUS_CONS_THREADS / 8)
        if (s_len[i] != CONS_NONE)
            apus_copy_cmd(a.payloads + s_dst[i], entries + s_off[i] + E_CMD, s_len[i], c, 8);
}

// 5: the row count and (packed) offsets[rows], then -- every read of the examined entries has completed with the copy kernel -- the cursor the
// follower forwards to the leader's pruning rule, and the status words
__global__ void apus_consume_tail_kernel(apus_consume_args_t a)
{
    const apus_cons_state_t *s = a.st;
    apus_ctrl_t *ctrl = reinterpret_cast<apus_ctrl_t *>(a.region);
    *a.count = (uint32_t)s->rows;
    if (a.offsets) a.offsets[s->rows] = s->bytes;
    const uint64_t nidx = s->next_idx + s->n_exam;
    apus_st_relaxed_sys_2x64(ctrl->cons_cur, s->new_cursor, nidx);
    apus_st_relaxed_sys(&a.hw->cons_cursor, s->new_cursor);
    apus_st_relaxed_sys(&a.hw->cons_next_idx, nidx);
    apus_st_relaxed_sys(&a.hw->cons_need_stride, s->need_stride);
    apus_st_relaxed_sys(&a.hw->cons_error, s->error);
}

// ---------------------------------------------------------------------------------
// CONSUME WAITS (apus_consume_wait): one warp on the consume stream, between consume calls, until at least min_entries
// committed entries lie past the cursor.  The cursor moves only inside the consume calls on this same stream, so the
// host cannot name the absolute count to wait for when it enqueues the wait (a cuStreamWaitValue64 would need it).
// Lane 0 polls the consumer record (the head kernel's acquire) and the cursor, backing off with __nanosleep so that a
// waiting consumer does not load L2 beside the resident replica kernels, and reads the host's release word over PCIe
// only every APUS_WAIT_RELEASE_POLL_NS.  It writes nothing the replica kernels read.
// ---------------------------------------------------------------------------------
// one step between two polls of a stream-ordered wait (consume waits, read fences), started at t0 on %globaltimer: the
// release epoch every APUS_WAIT_RELEASE_POLL_NS (t_rel: when it was read last), the deadline, then a back-off sleep
// (`sleep` doubles up to APUS_WAIT_SLEEP_MAX_NS).  true: the wait ends, with APUS_WAIT_RELEASED or APUS_WAIT_TIMED_OUT
// in `why`.
__device__ __forceinline__ bool wait_backoff(const apus_hostwords_t *hw, uint64_t epoch, uint64_t t0, uint64_t timeout_ns,
                                             uint64_t &t_rel, uint32_t &sleep, uint32_t &why)
{
    const uint64_t now = apus_globaltimer_ns();
    if (apus_poll_word_moved(&hw->cons_wait_epoch, epoch, now, t_rel)) { why = APUS_WAIT_RELEASED; return true; }
    if (now - t0 >= timeout_ns) { why = APUS_WAIT_TIMED_OUT; return true; }
    apus_poll_sleep(sleep);
    return false;
}

__global__ void apus_consume_wait_kernel(const apus_ctrl_t *ctrl, apus_hostwords_t *hw, uint64_t epoch,
                                         uint32_t min_entries, uint64_t timeout_ns, uint32_t *outcome)
{
    if (threadIdx.x != 0) return;
    const uint64_t t0 = apus_globaltimer_ns();
    uint64_t t_rel = t0, avail;
    uint32_t why, sleep = APUS_WAIT_SLEEP_MIN_NS;
    for (;;) {
        uint64_t committed, held;
        apus_cons_read(ctrl->cons_rec, committed, held);
        avail = apus_cons_avail(held, apus_ld_relaxed_sys(&ctrl->cons_cur[1]));
        if (avail >= min_entries) { why = APUS_WAIT_READY; break; }
        if (wait_backoff(hw, epoch, t0, timeout_ns, t_rel, sleep, why)) break;
    }
    if (outcome) *(volatile uint32_t *)outcome = why;
    apus_st_relaxed_sys(&hw->cons_wait_outcome, why);
    apus_st_relaxed_sys(&hw->cons_wait_avail, avail);
}

// ---------------------------------------------------------------------------------
// CONSUME MARKS (apus_consume_mark): one thread on the consume stream writes the consumer position {cursor offset, idx
// of the next entry} as the consume calls before it left it, into a 16 B device word of the caller's.  A copy of the
// application's state enqueued behind the mark in stream order is the state at that position.  A consumer stopped for
// good (APUS_CONSUME_BAD_IDX) marks next idx 0, which no seed accepts.  It writes nothing the replica kernels read.
// ---------------------------------------------------------------------------------
__global__ void apus_consume_mark_kernel(const apus_ctrl_t *ctrl, const apus_cons_state_t *st, uint64_t *mark)
{
    const uint64_t cursor = apus_ld_relaxed_sys(&ctrl->cons_cur[0]), nidx = apus_ld_relaxed_sys(&ctrl->cons_cur[1]);
    *reinterpret_cast<ulonglong2 *>(mark) = make_ulonglong2(cursor, st->error ? 0ull : nidx);
}

// ---------------------------------------------------------------------------------
// READ FENCES (apus_read_fence): one warp on the consume stream; lane 0 takes the three steps of apus_reader.cuh, the
// definitions a resident reader takes too.
//   1. K: the entries-committed word of the leader's consumer record (apus_cons_read's acquire), which its commit warp
//      publishes only under APUS_F_APPLY_ANY_ROLE (cons_on == 2); otherwise, or with the leader not mapped, NOT_LEADER.
//   2. after K (the acquire orders the loads below after it): the SID word of every member this replica maps; fewer
//      than N/2 + 1 at term <= t ends NOT_LEADER (rf_confirmed).
//   3. this replica's own record, polled as a consume wait polls (wait_backoff) until rf_ready: held >= K, and the
//      entry the offset index names for idx `held` carries idx `held` (else it is another lap's: poll again) and a term
//      >= t.
// F = held.  N + 2 loads of other replicas' words (the leader's cons_on and record, the SIDs), one local poll.  It
// writes the caller's index (READY only) and outcome words and two pinned status words, nothing the replica kernels read.
// ---------------------------------------------------------------------------------
__global__ void apus_read_fence_kernel(apus_fence_args_t a)
{
    if (threadIdx.x != 0) return;
    const uint64_t t0 = apus_globaltimer_ns();
    uint64_t F = 0;
    uint32_t why = APUS_WAIT_NOT_LEADER;
    const uint8_t *lead = NULL;
#pragma unroll
    for (uint32_t i = 0; i < APUS_MAX_SERVERS; i++)
        if (i == a.leader) lead = a.member[i];
    uint64_t K;
    uint32_t mask;
    if (apus_fence_take_k(lead, APUS_REGION_CONS_ON, APUS_REGION_CONS_REC, K) &&
        apus_fence_confirm(a.member, a.n, APUS_REGION_SID, a.term, mask)) {
        const apus_ctrl_t *own = reinterpret_cast<const apus_ctrl_t *>(a.region);
        const uint32_t *index = reinterpret_cast<const uint32_t *>(a.region + APUS_INDEX_OFF);
        const uint8_t *entries = a.region + a.entries_off;
        uint64_t t_rel = t0;
        uint32_t sleep = APUS_WAIT_SLEEP_MIN_NS;
        for (;;) {
            uint64_t held;
            if (apus_fence_ready(entries, index, a.idx_mask, a.log_len, own->cons_rec, K, a.term, held)) {
                F = held;
                why = APUS_WAIT_READY;
                break;
            }
            if (wait_backoff(a.hw, a.epoch, t0, a.timeout_ns, t_rel, sleep, why)) break;
        }
    }
    if (why == APUS_WAIT_READY) *(volatile uint64_t *)a.index = F;
    if (a.outcome) *(volatile uint32_t *)a.outcome = why;
    apus_st_relaxed_sys(&a.hw->fence_outcome, why);
    apus_st_relaxed_sys(&a.hw->fence_index, F);
}

// ---------------------------------------------------------------------------------
// host side: loading and enqueueing (apus_engine.cu brackets each enqueue in the caller's stream order)
// ---------------------------------------------------------------------------------
// These kernels run while the replica kernels are resident.  Under lazy module loading (CUDA_MODULE_LOADING=LAZY, the
// default) the first launch of a kernel loads it, and a load may wait for the running kernels: with a resident leader
// that waits for the very requests a fill kernel writes, or a resident follower whose pruning waits for the consume
// kernels' cursor, that never returns.  So every kernel of this file is loaded before any launch.
extern "C" cudaError_t apus_batch_load(void)
{
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, apus_synth_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_pack_sizes_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_pack_scan_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_pack_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_bell_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_consume_head_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_consume_count_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_consume_scan_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_consume_copy_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_consume_tail_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_consume_wait_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_consume_mark_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, apus_read_fence_kernel);
    return e;
}

// n synthetic requests from slot first_slot on, 256 threads per block and at most eight blocks per SM (`sms`)
extern "C" cudaError_t apus_synth_enqueue(apus_slot_t *ring, uint32_t mask, uint8_t *pay, uint64_t first_slot, uint32_t n,
                                          uint32_t type, uint32_t conn, uint64_t first_req, uint32_t len, uint32_t seed,
                                          uint64_t pay_pos0, uint32_t need, uint32_t first_flags, int sms,
                                          cudaStream_t stream)
{
    const int threads = 256;
    int blocks = (int)((n + threads - 1) / threads);
    if (blocks > sms * 8) blocks = sms * 8;
    apus_synth_kernel<<<blocks, threads, 0, stream>>>(ring, mask, pay, first_slot, n, type, conn, first_req, len, seed,
                                                      pay_pos0, need, first_flags);
    return cudaGetLastError();
}

// the three packing passes of a device batch, then (bell set) its doorbell `upto`
extern "C" cudaError_t apus_pack_enqueue(const apus_pack_args_t *a, apus_hostwords_t *hw, uint64_t *bell, uint64_t upto,
                                         cudaStream_t stream)
{
    const uint32_t nblk = apus_pack_blocks(a->n);
    apus_pack_sizes_kernel<<<nblk, APUS_PACK_THREADS, 0, stream>>>(*a);
    apus_pack_scan_kernel<<<1, APUS_PACK_THREADS, 0, stream>>>(*a, nblk, hw);
    apus_pack_kernel<<<nblk, APUS_PACK_THREADS, 0, stream>>>(*a);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && bell) {
        apus_bell_kernel<<<1, 1, 0, stream>>>(bell, upto);
        e = cudaGetLastError();
    }
    return e;
}

extern "C" cudaError_t apus_consume_enqueue(const apus_consume_args_t *a, cudaStream_t stream)
{
    apus_consume_head_kernel<<<1, 1, 0, stream>>>(*a);
    apus_consume_count_kernel<<<a->nblk, APUS_CONS_THREADS, 0, stream>>>(*a);
    apus_consume_scan_kernel<<<1, APUS_CONS_THREADS, 0, stream>>>(*a);
    apus_consume_copy_kernel<<<a->nblk, APUS_CONS_THREADS, 0, stream>>>(*a);
    apus_consume_tail_kernel<<<1, 1, 0, stream>>>(*a);
    return cudaGetLastError();
}

extern "C" cudaError_t apus_consume_wait_enqueue(const uint8_t *region, apus_hostwords_t *hw, uint64_t epoch,
                                                 uint32_t min_entries, uint64_t timeout_ns, uint32_t *outcome,
                                                 cudaStream_t stream)
{
    apus_consume_wait_kernel<<<1, 32, 0, stream>>>(reinterpret_cast<const apus_ctrl_t *>(region), hw, epoch, min_entries,
                                                   timeout_ns, outcome);
    return cudaGetLastError();
}

extern "C" cudaError_t apus_consume_mark_enqueue(const uint8_t *region, const apus_cons_state_t *st, uint64_t *mark,
                                                 cudaStream_t stream)
{
    apus_consume_mark_kernel<<<1, 1, 0, stream>>>(reinterpret_cast<const apus_ctrl_t *>(region), st, mark);
    return cudaGetLastError();
}

extern "C" cudaError_t apus_read_fence_enqueue(const apus_fence_args_t *a, cudaStream_t stream)
{
    apus_read_fence_kernel<<<1, 32, 0, stream>>>(*a);
    return cudaGetLastError();
}
