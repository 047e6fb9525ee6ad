/*
 * apus_kernels.cu -- the persistent sm_90a kernels of the replication engine.
 *
 * One kernel, `apus_replica_kernel`, launched with one CTA per replica ROLE that
 * lives on the launching GPU (apus_role_t table).  Two roles:
 *
 *   LEADER   the hot loop of the reference's leader, fused:
 *            get_tailq_message (dare_ibv_ud.c:780-790) + log_append_entry
 *            (dare_log.h:466-558) + persist_new_entries' sender stamp
 *            (dare_server.c:1803-1804) + update_remote_logs step I/II
 *            (dare_ibv_rc.c:1526-1573: byte range then tail) + the commit rule
 *            (dare_ibv_rc.c:1725-1758) + the commit publish (:1760-1822) +
 *            log pruning (dare_server.c:1996-2122).
 *            15 producer warps build a TILE of entries in shared memory and push
 *            it with 16 B vector stores into the local log and into every
 *            follower's log over NVLink; warp 15 is the commit warp: lane i
 *            polls follower i's ack word and a shuffle ranking of the acks finds
 *            the count a majority holds.
 *   FOLLOWER persist_new_entries' follower branch (dare_server.c:1792-1810) +
 *            rc_send_entries_reply (dare_ibv_rc.c:1828-1863): poll the tail
 *            publish, walk the new entries, set reply[me] locally and in the
 *            leader's copy, publish the ack word, follow `commit`, adopt `head`
 *            from committed HEAD entries (dare_server.c:2163-2186).
 *
 * Ordering (invariant I1, "data before tail"): all data stores of a tile ->
 * bar.sync -> fence.sc.sys -> 16 B st.relaxed.sys of {end, count}.  The
 * follower reads the pair with ld.acquire.sys (or, for a self-certifying publish,
 * verifies its checksum over the bytes) and then reads the entry bytes with
 * ld.relaxed.sys (never through a stale L1 line).  Acks mirror this in the other
 * direction.
 *
 * Pure integer / byte work: no tensor cores, bound by NVLink store bandwidth and
 * by launch-free round-trip latency.
 *
 * The short stream-ordered kernels of device submission and consumption are
 * apus_batch.cu; the device helpers both files use are apus_dev.h.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "apus_gpu.h"
#include "apus_layout.h"
#include "apus_cert.h"
#include "apus_dev.h"

// ---------------------------------------------------------------------------------
// helpers only the replica kernel uses (the shared ones are apus_dev.h)
// ---------------------------------------------------------------------------------
// NVSwitch multicast stores: ONE store, every replica of the group (the issuing GPU's own copy included) receives it
__device__ __forceinline__ void mst_v4(void *p, uint4 v)
{
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(__uint_as_float(v.x)),
                 "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w))
                 : "memory");
}
__device__ __forceinline__ void mst_u32(void *p, uint32_t v)
{
    asm volatile("multimem.st.relaxed.sys.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t globaltimer_ns()
{
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// named barrier for a subset of the CTA's warps
__device__ __forceinline__ void bar_sync(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// {count | term16}: a tail publish's entry count or a heartbeat's beat, stamped with the low 16 bits of the term so that
// a follower can drop what a deposed leader still stores
__device__ __forceinline__ uint64_t term_word(uint64_t count, uint64_t term)
{
    return (count & APUS_PUB_CUM_MASK) | ((term & 0xffffull) << APUS_PUB_TERM_SHIFT);
}
__device__ __forceinline__ bool term_word_is(uint64_t w, uint64_t term)
{
    return (w >> APUS_PUB_TERM_SHIFT) == (term & 0xffffull);
}

// A host control plane moves the head the way the reference's log_pruning does (dare_server.c:2041-2046): it appends a
// HEAD entry that CARRIES the new head offset.  The leader adopts the offset when it places that entry -- never by
// re-reading the log header: a ring offset read "a while ago" cannot be told from a new one (the reader may have waited
// for its turn while almost a whole ring was appended), and a stale head taken for an advance unprotects entries the
// followers' applications have not replayed yet.
__device__ __forceinline__ uint64_t adopt_head(uint64_t head, uint64_t carried, uint64_t new_end, uint64_t L)
{
    if (carried >= L) return head;
    const uint64_t ne = (new_end == L) ? 0 : new_end;
    return (apus_ring_dist(head, carried, L) <= apus_ring_dist(head, ne, L)) ? carried : head;     // only forward, only inside the used region
}
// the little-endian u64 of the 8 bytes at p, any alignment: the head offset a HEAD entry carries
__device__ __forceinline__ uint64_t le_u64(const uint8_t *p)
{
    uint64_t v = 0;
#pragma unroll
    for (int q = 7; q >= 0; q--) v = (v << 8) | p[q];
    return v;
}

#define WATCHDOG_NS (20ull * 1000ull * 1000ull * 1000ull)

// error codes reported through hostwords.error
#define APUS_KERR_WATCHDOG_LEADER   1
#define APUS_KERR_WATCHDOG_FOLLOWER 2
#define APUS_KERR_WATCHDOG_COMMIT   3
#define APUS_KERR_BAD_ENTRY         4
#define APUS_KERR_COUNT_MISMATCH    5

// ---------------------------------------------------------------------------------
// shared memory
// ---------------------------------------------------------------------------------
#define N_PRODUCER_WARPS 15
#define NT (N_PRODUCER_WARPS * 32)      // producer threads
#define MAXB APUS_MAX_TILE_ENTRIES
#define PUBMASK (APUS_PUBRING_RECORDS - 1)

// Placement state handed from claim to claim (the four stamped rec_* pairs of apus_seq_t), decoded
struct PlaceRec {
    uint64_t placed;     // entries placed so far
    uint64_t end;        // end offset after the last placed entry (len = empty log)
    uint64_t tail;       // offset of the last placed entry
    uint64_t head;       // head offset (only the turn holder moves it)
    bool wrapped;        // the ring has wrapped at least once (no fresh bytes left)
    bool prev_head;      // the last placed entry is a HEAD entry of the pruning rule
};

struct LeaderShared {
    // per fetched slot (filled while fetching: no strided re-reads of the 128 B slots)
    uint32_t es[MAXB];         // log stride of the entry (64 + len, or 64)
    uint32_t xb[MAXB];         // payload-ring bytes to stage for it (0 when inline)
    uint32_t cum_es[MAXB];     // inclusive prefix sum of es over the fetched batch (state independent)
    uint32_t cum_xb[MAXB];     // inclusive prefix sum of xb
    uint32_t rel[MAXB];        // entry start - sub-tile start (bytes)
    uint32_t xoff[MAXB];       // offset of the entry's image in the ext staging
    uint64_t ap[32];           // apply offsets of the replicas, read ahead of the place turn
    uint32_t ap_valid;         // ap[] was read while holding the place turn of this claim (never earlier)
    uint32_t static_cut;       // first k > 0 whose payload image restarted the payload ring (else n_fetch)
    uint32_t first_ext_all;    // first entry with an external payload image (else 0xffffffff)
    uint32_t host_head_k;      // last HEAD entry submitted by the host in this batch (else 0xffffffff): it carries the new head
    // the batch's descriptors, reduced while they are fetched (t1_fetch) and turned into the words above by t1_scan
    uint32_t r_es_min, r_es_max, r_xb_min, r_xb_max, r_cut, r_fext, r_hh1;
    uint32_t part_es[MAXB / 32], part_xb[MAXB / 32];   // per-32-entry totals of the CTA-wide scan (non-uniform batches)
    uint64_t idx_base;         // idx of an entry = idx_base + its 1-based position in the placement order
    uint8_t  ty[MAXB];
    uint8_t  flg[MAXB];        // bit0 EXT, bit1 WRAP
    // claim: slots [slot0, slot0 + n_fetch); slot0 is also the stamp of this claim's place and publish turns
    uint32_t n_fetch, finish, abort, was_blocked;
    uint64_t slot0, t_dequeue, t_place_acq, pub_h, pub_tail_seen;
    // placement state while this CTA holds the place turn (what the rec_* pairs of apus_seq_t carry), and the
    // high-water mark of bytes ever written (fresh beyond)
    PlaceRec st;
    uint64_t st_hwm;
    // current sub-tile
    uint32_t kbase, m, gap, ghost, fresh, auto_head, ext_bytes, last, blocked, hbytes;
    uint32_t base_es, base_xb, fast, after_gap;   // after_gap: the last placement was a wrap gap (leader_place)
    uint64_t ext_base, auto_head_val, a, b, idx0, cum_after, new_end, tail_after, hwm_after;
    uint8_t  *peer_entries[APUS_MAX_SERVERS];
    uint32_t *peer_index[APUS_MAX_SERVERS];
    uint64_t prof_ph[8], prof_tn[8];  // worker 0's profile (LeaderProf), thread 0 alone
};

#define LS_BYTES ((sizeof(LeaderShared) + 127u) & ~127u)
#define L_SLOTS_OFF LS_BYTES
#define L_EXT_OFF   (L_SLOTS_OFF + MAXB * APUS_CSLOT_BYTES)
#define L_IMG_OFF   (L_EXT_OFF + APUS_LEADER_EXT_BYTES)
#define L_TOTAL     (L_IMG_OFF + APUS_LEADER_IMG_BYTES + 16)
static_assert(L_TOTAL <= 232448u, "leader shared memory exceeds the sm_90 opt-in limit per CTA (227 KiB)");

struct FollowerShared {
    uint32_t off[APUS_FOLLOWER_WIN_BYTES / 64 + 8];   // entry offsets found in the window (relative to win_lo)
    uint32_t n;
    uint32_t done;
    uint64_t win_lo, win_hi, next;           // window bounds in the log, next walk offset
    uint64_t head_val, head_end;             // last HEAD entry of the window (head_end == len: none)
    uint64_t end_seen, cum_seen, commit_seen;
    uint32_t head_j;                         // index mode: 1 + position of the last HEAD entry of the batch
    uint32_t cert;                           // the publish being processed was self-certifying: ONE entry at cert_start
    uint64_t cert_start;
};
#define FS_BYTES ((sizeof(FollowerShared) + 127u) & ~127u)
#define F_TOTAL (FS_BYTES + APUS_FOLLOWER_WIN_BYTES + 16)

extern __shared__ __align__(16) uint8_t smem_raw[];

// gpu-scope handoffs between the leader's worker CTAs
__device__ __forceinline__ uint64_t ld_acquire_gpu(const volatile void *p)
{
    uint64_t v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void ld_acquire_gpu_2x64(const volatile void *p, uint64_t &a, uint64_t &b)
{
    asm volatile("ld.acquire.gpu.global.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_release_gpu(volatile void *p, uint64_t v)
{
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// ---------------------------------------------------------------------------------
// Self-certifying publishes: the checksum (cs_weight / cs_mask / cs_chunk_words / cs_key) lives in apus_cert.h, which
// the CPU property test compiles too.
// ---------------------------------------------------------------------------------
// contribution of the 16 B chunk at log offset lo (16 B aligned), restricted to the bytes inside [a, b)
__device__ __forceinline__ uint64_t cs_chunk(const uint4 v, uint64_t lo, uint64_t a, uint64_t b)
{
    return cs_chunk_words((uint64_t)v.x | ((uint64_t)v.y << 32), (uint64_t)v.z | ((uint64_t)v.w << 32), lo, a, b);
}
// first n bytes of a 16 B chunk from `nw`, the rest from `old`
__device__ __forceinline__ uint4 chunk_select(const uint4 nw, const uint4 old, int n)
{
    uint32_t a[4] = {nw.x, nw.y, nw.z, nw.w}, o[4] = {old.x, old.y, old.z, old.w}, r[4];
#pragma unroll
    for (int w = 0; w < 4; w++) {
        const int k = n - 4 * w;                      // bytes of this word that come from `nw`
        const uint32_t m = k >= 4 ? 0xffffffffu : (k <= 0 ? 0u : ((1u << (8 * k)) - 1u));
        r[w] = (a[w] & m) | (o[w] & ~m);
    }
    return make_uint4(r[0], r[1], r[2], r[3]);
}


// ---------------------------------------------------------------------------------
// LEADER
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t hdr_byte(uint32_t j, uint64_t idx, uint64_t term, uint64_t req_id,
                                             uint32_t clt, uint32_t type, uint32_t sender)
{
    // dare_log_entry_t bytes 0..40 (dare_log.h:33-48)
    if (j < 8) return (uint32_t)(idx >> (8 * j)) & 0xFF;
    if (j < 16) return (uint32_t)(term >> (8 * (j - 8))) & 0xFF;
    if (j < 24) return (uint32_t)(req_id >> (8 * (j - 16))) & 0xFF;
    if (j == 24) return clt & 0xFF;
    if (j == 25) return (clt >> 8) & 0xFF;
    if (j == 26) return type;
    if (j == 27) return sender;
    return 0;   // reply[13]
}

// bytes 0..40 of an entry header into shared memory at any alignment, by `gl` lanes (sub = lane in group)
__device__ __noinline__ void group_write_header(uint8_t *e, int sub, int gl, uint64_t idx, uint64_t term, uint64_t req_id,
                                                   uint32_t clt, uint32_t type, uint32_t sender, bool skip_sender)
{
    if ((((uint32_t)(uintptr_t)e) & 15u) == 0 && !skip_sender) {
        // 16 B aligned entry: two 16 B stores, one 8 B store, one byte; bytes 41..47 stay (hole)
        if (sub == 0) *reinterpret_cast<uint4 *>(e + 0) = make_uint4((uint32_t)idx, (uint32_t)(idx >> 32), (uint32_t)term, (uint32_t)(term >> 32));
        else if (sub == 1) *reinterpret_cast<uint4 *>(e + 16) = make_uint4((uint32_t)req_id, (uint32_t)(req_id >> 32),
                                                                         (clt & 0xffffu) | (type << 16) | (sender << 24), 0u);
        else if (sub == 2) *reinterpret_cast<uint64_t *>(e + 32) = 0;
        else if (sub == 3) e[40] = 0;
    } else if ((((uint32_t)(uintptr_t)e) & 7u) == 0) {
        // aligned entry: 8-byte stores for bytes 0..39, byte 40 separately; bytes 41..47 stay (hole)
        if (sub == 0) *reinterpret_cast<uint64_t *>(e + 0) = idx;
        else if (sub == 1) *reinterpret_cast<uint64_t *>(e + 8) = term;
        else if (sub == 2) *reinterpret_cast<uint64_t *>(e + 16) = req_id;
        else if (sub == 3) {
            if (skip_sender) {
                e[24] = (uint8_t)clt; e[25] = (uint8_t)(clt >> 8); e[26] = (uint8_t)type;
                e[28] = 0; e[29] = 0; e[30] = 0; e[31] = 0;
            } else {
                *reinterpret_cast<uint64_t *>(e + 24) =
                    (uint64_t)(clt & 0xffffu) | ((uint64_t)type << 16) | ((uint64_t)sender << 24);
            }
        } else if (sub == 4) *reinterpret_cast<uint64_t *>(e + 32) = 0;
        else if (sub == 5) e[40] = 0;
    } else {
        for (uint32_t j = sub; j < 41; j += gl)
            if (!(skip_sender && j == E_SENDER)) e[j] = (uint8_t)hdr_byte(j, idx, term, req_id, clt, type, sender);
    }
}

// copy nbytes from a 16 B-aligned shared source to an arbitrarily aligned shared destination
__device__ __noinline__ void group_copy_smem(uint8_t *dst, const uint8_t *src, uint32_t nbytes, int sub, int gl)
{
    const uint32_t nchunks = (nbytes + 15u) >> 4;
    const uint32_t dalign = (uint32_t)(uintptr_t)dst & 15u;
    for (uint32_t c = sub; c < nchunks; c += gl) {
        const uint4 v = *reinterpret_cast<const uint4 *>(src + 16u * c);
        uint8_t *d = dst + 16u * c;
        const uint32_t left = nbytes - 16u * c;
        if (dalign == 0 && left >= 16) {
            *reinterpret_cast<uint4 *>(d) = v;
        } else if ((dalign & 3u) == 0 && left >= 16) {
            uint32_t *d4 = reinterpret_cast<uint32_t *>(d);
            d4[0] = v.x; d4[1] = v.y; d4[2] = v.z; d4[3] = v.w;
        } else if ((dalign & 1u) == 0 && left >= 16) {
            uint16_t *d2 = reinterpret_cast<uint16_t *>(d);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 8; k++) d2[k] = (uint16_t)(w[k >> 1] >> (16 * (k & 1)));
        } else {
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
            const uint32_t nb = left < 16 ? left : 16;
#pragma unroll
            for (uint32_t k = 0; k < 16; k++)
                if (k < nb) d[k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
        }
    }
}

// global (16 B aligned) -> shared, nchunks 16 B chunks, by `nthr` threads (tid = 0..nthr-1), 4 loads in flight each
__device__ __noinline__ void cta_fetch_chunks(uint8_t *dst, const uint8_t *src, uint32_t nchunks, uint32_t tid, uint32_t nthr)
{
    uint32_t c = tid;
    for (; c + 3u * nthr < nchunks; c += 4u * nthr) {
        const uint4 v0 = apus_ld_relaxed_sys_v4(src + 16ull * c);
        const uint4 v1 = apus_ld_relaxed_sys_v4(src + 16ull * (c + nthr));
        const uint4 v2 = apus_ld_relaxed_sys_v4(src + 16ull * (c + 2u * nthr));
        const uint4 v3 = apus_ld_relaxed_sys_v4(src + 16ull * (c + 3u * nthr));
        reinterpret_cast<uint4 *>(dst)[c] = v0;
        reinterpret_cast<uint4 *>(dst)[c + nthr] = v1;
        reinterpret_cast<uint4 *>(dst)[c + 2u * nthr] = v2;
        reinterpret_cast<uint4 *>(dst)[c + 3u * nthr] = v3;
    }
    for (; c < nchunks; c += nthr) reinterpret_cast<uint4 *>(dst)[c] = apus_ld_relaxed_sys_v4(src + 16ull * c);
}

// What T2 needs to know about the whole fetched batch, reduced by every producer thread over the descriptors it
// fetched (t1_fetch) and then over the CTA: whether every entry has the same stride and staged size (then the prefix
// sums are closed-form), the first payload-ring restart, the first external image and the last host HEAD entry.
struct DescReduce {
    uint32_t es_min, es_max, xb_min, xb_max, cut, fext, hh1;
    __device__ __forceinline__ void init()
    {
        es_min = xb_min = cut = fext = 0xffffffffu;
        es_max = xb_max = hh1 = 0;
    }
};

// the descriptor chunk of entry k -> compact per-entry arrays, and into the thread's reduction
__device__ __forceinline__ void note_desc(LeaderShared *S, DescReduce &R, uint32_t k, const uint4 v)
{
    const uint32_t to = v.z, ty = (to >> APUS_SLOT_TYPE_SHIFT) & APUS_SLOT_TYPE_MASK, len = v.w & 0xffffu;
    const uint32_t es = apus_entry_stride(ty, len), xb = (to & APUS_SLOT_EXT) ? ((data_bytes(ty, len) + 15u) & ~15u) : 0u;
    S->ty[k] = (uint8_t)ty;
    S->flg[k] = (uint8_t)(((to & APUS_SLOT_EXT) ? 1u : 0u) | ((to & APUS_SLOT_WRAP) ? 2u : 0u));
    S->es[k] = es;
    S->xb[k] = xb;
    R.es_min = min(R.es_min, es); R.es_max = max(R.es_max, es);
    R.xb_min = min(R.xb_min, xb); R.xb_max = max(R.xb_max, xb);
    if (k > 0 && (to & APUS_SLOT_WRAP)) R.cut = min(R.cut, k);
    if (to & APUS_SLOT_EXT) R.fext = min(R.fext, k);
    if (ty == T_HEAD) R.hh1 = max(R.hh1, k + 1u);
}

// fetch `cnt` slots starting at ring slot `s` into shared slot `k0` onward.  A 128 B ring slot is kept as a
// 96 B compact slot: its two stamp chunks (3 and 7) are neither loaded nor stored, so that the inline image
// is contiguous in shared memory (and a quarter of the PCIe / HBM read traffic is saved).  8 loads in flight per
// thread: a 512-slot claim is 3072 chunks, one round for every producer thread and a second for a few.
__device__ __noinline__ void cta_fetch_slots(LeaderShared *S, uint8_t *slots, const apus_slot_t *ring, uint64_t s, uint32_t k0,
                                                uint32_t cnt, int tid)
{
    DescReduce R;
    R.init();
    const uint8_t *src = reinterpret_cast<const uint8_t *>(ring + s);
    uint8_t *dst = slots + (size_t)k0 * APUS_CSLOT_BYTES;
    const uint32_t nq = cnt * 6u;                                  // compact chunks
    // warp 1 takes the first chunks (warp 0 is busy with the turns).  NT is a multiple of 6: a thread's chunks are
    // all the same chunk of their slots, so only the threads of the descriptor chunks decode descriptors.
    const uint32_t q0 = (tid >= 32) ? tid - 32 : tid + NT - 32;
    const bool desc = (q0 % 6u) == 0;
    for (uint32_t q = q0; q < nq; q += 8u * NT) {
        uint4 v[8];
#pragma unroll
        for (uint32_t i = 0; i < 8; i++) {
            // zeroed first: a register that a predicated load leaves undefined on the other path makes ptxas keep the
            // eight values in local memory, one load after the other (issuing the surplus loads at a clamped address
            // instead costs real reads -- over PCIe, hundreds of them at one host address)
            const uint32_t qi = q + i * NT, k = qi / 6u, r = qi - 6u * k;
            v[i] = make_uint4(0, 0, 0, 0);
            if (qi < nq) v[i] = apus_ld_relaxed_sys_v4(src + (size_t)k * APUS_SLOT_BYTES + 16u * (r < 3u ? r : r + 1u));
        }
#pragma unroll
        for (uint32_t i = 0; i < 8; i++) {
            const uint32_t qi = q + i * NT;
            if (qi < nq) {
                reinterpret_cast<uint4 *>(dst)[qi] = v[i];
                if (desc) note_desc(S, R, k0 + qi / 6u, v[i]);
            }
        }
    }
    // each warp folds its lanes', lane 0 folds the warp's into the r_* words (which t0_claim reset)
    R.es_min = __reduce_min_sync(0xffffffffu, R.es_min); R.es_max = __reduce_max_sync(0xffffffffu, R.es_max);
    R.xb_min = __reduce_min_sync(0xffffffffu, R.xb_min); R.xb_max = __reduce_max_sync(0xffffffffu, R.xb_max);
    R.cut = __reduce_min_sync(0xffffffffu, R.cut); R.fext = __reduce_min_sync(0xffffffffu, R.fext);
    R.hh1 = __reduce_max_sync(0xffffffffu, R.hh1);
    if ((tid & 31) == 0 && R.es_max) {       // (a warp that decoded no descriptor has nothing to add)
        atomicMin(&S->r_es_min, R.es_min); atomicMax(&S->r_es_max, R.es_max);
        atomicMin(&S->r_xb_min, R.xb_min); atomicMax(&S->r_xb_max, R.xb_max);
        if (R.cut != 0xffffffffu) atomicMin(&S->r_cut, R.cut);
        if (R.fext != 0xffffffffu) atomicMin(&S->r_fext, R.fext);
        if (R.hh1) atomicMax(&S->r_hh1, R.hh1);
    }
}

// After T1 (all producer threads, between the T1 barrier and T2): the state-independent part of the placement --
// inclusive prefix sums of the log strides and of the staged payload bytes of the fetched batch, closed-form when every
// entry has the same shape (the benchmark's, and most applications' bursts), else a CTA-wide scan -- and the batch
// words T2 reads.  Ends with a barrier of the producer warps.
__device__ __noinline__ void t1_scan(LeaderShared *S, int tid)
{
    const int lane = tid & 31, warp = tid >> 5;
    const uint32_t nf = S->n_fetch;
    if (S->r_es_min == S->r_es_max && S->r_xb_min == S->r_xb_max) {
        const uint32_t es0 = S->r_es_min, xb0 = S->r_xb_min;
        for (uint32_t k = tid; k < nf; k += NT) { S->cum_es[k] = (k + 1u) * es0; S->cum_xb[k] = (k + 1u) * xb0; }
    } else {
        // warp w scans the 32-entry parts w, w + 15, ...; then every entry adds the totals of the parts before its own
        for (uint32_t c = warp; 32u * c < nf; c += N_PRODUCER_WARPS) {
            const uint32_t k = 32u * c + lane;
            uint32_t inc = k < nf ? S->es[k] : 0u, xinc = k < nf ? S->xb[k] : 0u;
#pragma unroll
            for (int sft = 1; sft < 32; sft <<= 1) {
                const uint32_t o = __shfl_up_sync(0xffffffffu, inc, sft);
                const uint32_t xo = __shfl_up_sync(0xffffffffu, xinc, sft);
                if (lane >= sft) { inc += o; xinc += xo; }
            }
            if (k < nf) { S->cum_es[k] = inc; S->cum_xb[k] = xinc; }
            if (lane == 31) { S->part_es[c] = inc; S->part_xb[c] = xinc; }
        }
        bar_sync(1, NT);
        for (uint32_t k = 32u + tid; k < nf; k += NT) {
            uint32_t ce = 0, cx = 0;
            for (uint32_t c = 0; c < (k >> 5); c++) { ce += S->part_es[c]; cx += S->part_xb[c]; }
            S->cum_es[k] += ce; S->cum_xb[k] += cx;
        }
    }
    if (tid == 0) {
        S->static_cut = S->r_cut < nf ? S->r_cut : nf;
        S->first_ext_all = S->r_fext;
        S->host_head_k = S->r_hh1 ? S->r_hh1 - 1u : 0xffffffffu;
        S->ap_valid = 0;          // apply offsets are read inside the place turn, only if the pruning rule could be due
    }
    bar_sync(1, NT);
}

// the apply offset of replica i that the pruning rule reads: mine from my header, a follower's as it reported it, and
// for a replica I am not connected to (removed, or the leader I took over from) my own: the reference sets the apply
// offset of a server that is off to the leader's (log_pruning, dare_server.c:2028-2031), so it never holds the head back
__device__ __forceinline__ uint64_t ld_apply(const apus_devctx_t *__restrict__ cx, const apus_ctrl_t *ctrl,
                                             const apus_loghdr_t *hdr, int i)
{
    return (i == cx->idx || !cx->peer[i]) ? apus_ld_relaxed_sys(&hdr->apply) : apus_ld_relaxed_sys(&ctrl->apply_off[i]);
}

// T2b (inside the place turn): place the next sub-tile of the fetched batch (entries kbase..nf) --
// log_append_entry's offset rules, free-space rule E2 and the pruning rule, on the placement
// state this CTA holds.  Kept short: everything state independent was done by t1_scan.
__device__ __noinline__ void leader_place(const apus_devctx_t *__restrict__ cx, LeaderShared *S, const apus_cslot_t *sl, int lane)
{
    const int N = cx->group_size;
    apus_loghdr_t *hdr = reinterpret_cast<apus_loghdr_t *>(cx->region + APUS_HDR_OFF);
    const uint64_t L = cx->log_len;
    const bool autoprune = (cx->flags & APUS_FLAG_AUTOPRUNE) != 0;
    const uint32_t kbase = S->kbase, nf = S->n_fetch;
    const uint64_t end = S->st.end;

    uint64_t head = S->st.head;                                // refreshed by the caller while blocked
    const uint64_t pos0 = (end == L) ? 0 : end;               // empty log starts at 0 (dare_log.h:216-219)
    uint64_t used = (end == L) ? 0 : apus_ring_dist(head, end, L);
    // ---- device-side log pruning (log_pruning / force_log_pruning, dare_server.c:1996-2122):
    //      head := the smallest apply offset in the group, published through a HEAD entry
    uint32_t autoh = 0;
    uint64_t new_head = 0;
    // "never two HEAD entries in a row" (prev_log_entry_head, dare_server.c:2042) keeps an idle log from filling with HEAD
    // entries; a placement that is BLOCKED on space right behind a HEAD entry must still be able to prune again once the
    // followers' applications have caught up -- else a slow follower host deadlocks the leader (back-pressure, rule E2).
    // Never right after a gap: the gap and the entry at 0 are one append of the reference (log_append_entry), and
    // log_pruning saw the end before the gap, where this rule was already evaluated.  Here `used` would count the
    // skipped stretch [old end, L) and could put a HEAD between the ghost and its entry.  That placement cannot block:
    // the gap was taken only because the entry fits at 0.  A gap placement is never a tile's last (S->last stays 0),
    // so its state never reaches the next claim's place_fast: the placement after it is always this CTA's leader_place.
    if (autoprune && !S->after_gap && end != L && used >= (L >> 2) && (!S->st.prev_head || S->was_blocked) &&
        L - pos0 >= APUS_HDR_BYTES) {
        uint64_t d = 0;                                   // distance apply -> end, per replica
        if (lane < N) {
            d = apus_ring_dist(S->ap[lane], end, L);
            if (d > used) d = used;                       // never behind the current head (or stale read-ahead)
        }
#pragma unroll
        for (int sft = 16; sft > 0; sft >>= 1) {
            const uint64_t o = __shfl_xor_sync(0xffffffffu, d, sft);
            d = o > d ? o : d;
        }
        if (d == 0) d = apus_ring_dist(S->st.tail, end, L);    // leave one entry (dare_server.c:2031-2034)
        if (d <= used && used - d >= (L >> 3)) {
            autoh = 1;
            new_head = (end >= d) ? end - d : L - (d - end);
            used = d;                                     // the head moves before the append (:2041)
            head = new_head;
        }
    }
    const uint32_t hbytes = autoh ? APUS_HDR_BYTES : 0;
    // limits for a contiguous sub-tile starting at pos0
    uint64_t lim = L - pos0;                                   // no entry may cross len
    const uint64_t imgcap = APUS_LEADER_IMG_BYTES - 16u - (pos0 & 15u);
    if (lim > imgcap) lim = imgcap;
    // rule E2: stay strictly before head (keep room for one HEAD entry when pruning on the device)
    const uint64_t reserve = autoprune ? APUS_HDR_BYTES : 0;
    const uint64_t lim_space = (L - used > 1 + reserve) ? (L - used - 1 - reserve) : 0;
    const uint64_t limit = lim < lim_space ? lim : lim_space;
    const uint32_t base_es = kbase ? S->cum_es[kbase - 1] : 0u, base_xb = kbase ? S->cum_xb[kbase - 1] : 0u;

    // how many entries from kbase fit: the prefix sums are monotone, one compare + ballot per 32 entries
    uint32_t m = nf - kbase, first_ext = 0xffffffffu;
    for (uint32_t r = kbase; r < nf; r += 32) {
        const uint32_t k = r + lane;
        const bool in = k < nf;
        const bool bad = in && ((uint64_t)hbytes + (S->cum_es[k] - base_es) > limit ||
                                S->cum_xb[k] - base_xb > APUS_LEADER_EXT_BYTES || (k > kbase && (S->flg[k] & 2u)));
        const uint32_t badmask = __ballot_sync(0xffffffffu, bad);
        const uint32_t good = badmask ? (uint32_t)(__ffs(badmask) - 1) : 32u;
        if (first_ext == 0xffffffffu) {
            const uint32_t extmask = __ballot_sync(0xffffffffu, in && (uint32_t)lane < good && (S->flg[k] & 1u));
            if (extmask) first_ext = r + (uint32_t)(__ffs(extmask) - 1);
        }
        if (badmask) { m = r + good - kbase; break; }
    }
    if (lane == 0) {
        const uint32_t carry = hbytes + (m ? S->cum_es[kbase + m - 1] - base_es : 0u);      // log bytes of the sub-tile
        const uint32_t xcarry = m ? S->cum_xb[kbase + m - 1] - base_xb : 0u;               // staged payload bytes
        S->gap = 0; S->ghost = 0; S->blocked = 0; S->last = 0;
        uint64_t a = pos0, b = pos0;
        if (m == 0 && !autoh) {
            // entry kbase does not fit at pos0: wrap (dare_log.h:502-504, 526-538) or no space
            const uint32_t es0 = S->es[kbase];
            const uint64_t left = L - pos0;
            if (es0 > left && used + left + es0 + reserve < L) {
                S->gap = 1;
                S->ghost = (left >= APUS_HDR_BYTES && apus_has_cmd(S->ty[kbase])) ? 1u : 0u;   // header fits: ghost stays behind
                b = L;
            } else {
                S->blocked = 1;        // back-pressure: wait for head to advance
            }
        } else {
            b = pos0 + carry;
        }
        S->a = a; S->b = b; S->m = m;
        S->hbytes = hbytes; S->base_es = base_es; S->base_xb = base_xb;
        S->ext_bytes = (m && first_ext != 0xffffffffu) ? xcarry : 0u;
        S->ext_base = (first_ext != 0xffffffffu) ? (uint64_t)(sl[first_ext].type_off & APUS_SLOT_OFF_MASK) * 16ull : 0ull;
        S->auto_head = autoh; S->auto_head_val = new_head;
        S->idx0 = S->idx_base + S->st.placed + 1;
        S->fresh = (a >= S->st_hwm) ? 1u : 0u;
        if (S->blocked) S->was_blocked = 1;
        if (!S->blocked) {
            S->was_blocked = 0;
            S->after_gap = S->gap;
            // commit the placement to the state this CTA carries
            if (autoh) apus_st_relaxed_sys(&hdr->head, new_head);
            if (autoh) S->st.head = new_head;
            if (S->host_head_k != 0xffffffffu && S->host_head_k >= kbase && S->host_head_k < kbase + m) {
                const uint64_t nh = adopt_head(S->st.head, le_u64(sl[S->host_head_k].inl), b, L);
                if (nh != S->st.head) { S->st.head = nh; apus_st_relaxed_sys(&hdr->head, nh); }
            }
            if (S->gap) {
                S->st.end = 0; S->st_hwm = L;
            } else {
                uint64_t ne = b; if (ne == L) ne = 0;                   // rule E1
                S->new_end = ne;
                S->st.end = ne;
                S->st.tail = m ? a + hbytes + (S->cum_es[kbase + m - 1] - base_es) - S->es[kbase + m - 1] : a;
                S->tail_after = S->st.tail;
                S->st.placed += m + autoh;
                S->cum_after = S->st.placed;
                if (autoh) atomicAdd(reinterpret_cast<unsigned long long *>(&reinterpret_cast<apus_ctrl_t *>(cx->region)->auto_heads), 1ull);
                S->st.prev_head = autoh && m == 0;         // never two HEAD entries in a row (dare_log.h:477-480)
                if (b > S->st_hwm) S->st_hwm = b;
                S->last = (kbase + m == nf) ? 1u : 0u;
            }
            S->hwm_after = S->st_hwm;
        }
    }
}


// ---------------------------------------------------------------------------------
// Turn protocols between the leader's worker CTAs (and the commit warp, which reads the publish records)
// ---------------------------------------------------------------------------------
// lane 0: wait until the four rec_* pairs carry `stamp` (the place turn is mine) and decode them.  false: the launch is
// being aborted and the turn never came -- nothing may be placed.
__device__ __forceinline__ bool place_acquire(apus_seq_t *seq, uint64_t stamp, PlaceRec &r)
{
    uint64_t s0, s1, s2, s3, tf;
    uint32_t spins = 0;
    for (;;) {
        ld_relaxed_sys_2x64(seq->rec_placed, s0, r.placed);
        ld_relaxed_sys_2x64(seq->rec_end, s1, r.end);
        ld_relaxed_sys_2x64(seq->rec_tail, s2, tf);
        ld_relaxed_sys_2x64(seq->rec_head, s3, r.head);
        if (s0 == stamp && s1 == stamp && s2 == stamp && s3 == stamp) break;
        if ((++spins & 0x3ffu) == 0 && apus_ld_relaxed_sys(&seq->abort_flag)) return false;
    }
    r.wrapped = (tf & APUS_REC_WRAPPED) != 0;
    r.prev_head = (tf & APUS_REC_PREV_HEAD) != 0;
    r.tail = tf & ~(APUS_REC_WRAPPED | APUS_REC_PREV_HEAD);
    return true;
}
// one thread: hand the place turn to the claim that starts at slot `stamp`
__device__ __forceinline__ void place_handoff(apus_seq_t *seq, uint64_t stamp, const PlaceRec &r)
{
    apus_st_relaxed_sys_2x64(seq->rec_placed, stamp, r.placed);
    apus_st_relaxed_sys_2x64(seq->rec_end, stamp, r.end);
    apus_st_relaxed_sys_2x64(seq->rec_tail, stamp,
                        r.tail | (r.wrapped ? APUS_REC_WRAPPED : 0ull) | (r.prev_head ? APUS_REC_PREV_HEAD : 0ull));
    apus_st_relaxed_sys_2x64(seq->rec_head, stamp, r.head);
}

// lane 0 of the tile path: wait for publish turn `stamp` (unless it is mine already: `h` then holds its record number), then for room in
// the publish ring (the commit warp drains it; the tail is re-read only when the last value seen would not leave room).
// `h` returns the record number to write; with `timed`, `wait_ns` gains the ns spent waiting for the turn.  false: the
// launch is being aborted -- nothing may be published.
__device__ __forceinline__ bool pub_acquire(apus_seq_t *seq, uint64_t stamp, bool have_turn, uint64_t &h,
                                            uint64_t &tail_seen, bool timed, uint64_t &wait_ns)
{
    bool ok = true;
    if (!have_turn) {
        const uint64_t t0 = timed ? globaltimer_ns() : 0;
        uint32_t spins = 0;
        uint64_t sq;
        for (;;) {
            // acquire: a predecessor that published self-certified data fenced it before this hand-over
            ld_acquire_gpu_2x64(seq->pub_turn, sq, h);
            if (sq == stamp) break;
            if ((++spins & 0x3ffu) == 0 && apus_ld_relaxed_sys(&seq->abort_flag)) { ok = false; break; }
        }
        if (timed) wait_ns += globaltimer_ns() - t0;
    }
    uint32_t spins = 0;
    while (ok && h - tail_seen >= APUS_PUBRING_RECORDS - 2) {
        tail_seen = apus_ld_relaxed_sys(&seq->pub_tail);
        if ((++spins & 0x3ffu) == 0 && apus_ld_relaxed_sys(&seq->abort_flag)) ok = false;
    }
    return ok;
}
// one thread: hand the publish turn to the claim that starts at slot `stamp`; `h` is the record it will write
__device__ __forceinline__ void pub_handoff(apus_seq_t *seq, uint64_t stamp, uint64_t h)
{
    apus_st_relaxed_sys_2x64(seq->pub_turn, stamp, h);
}
// lanes 16..23: publish record h, one 16 B {h + 1, value} pair per lane (the PR_* fields of apus_layout.h)
__device__ __forceinline__ void pub_record(apus_pubrec_t *ring, uint64_t h, int lane, uint64_t cum, uint64_t end,
                                           uint64_t tickets, uint64_t t0, uint64_t tail, uint64_t hwm, uint64_t next_idx,
                                           uint64_t bytes)
{
    if (lane < 16 || lane >= 24) return;
    const int q = lane - 16;
    const uint64_t val = q == PR_CUM ? cum : q == PR_END ? end : q == PR_TICKETS ? tickets : q == PR_T0 ? t0
                       : q == PR_TAIL ? tail : q == PR_HWM ? hwm : q == PR_NEXTIDX ? next_idx : bytes;
    apus_st_relaxed_sys_2x64(&ring[h & PUBMASK].w[2 * q], h + 1, val);
}
// warp: lane l looks at pair l & 7 of record rn0 + l / 8, for the first `nrec` (<= 4) records; v is the lane's value.
// Returns how many of them, in order from rn0, are valid (all eight pairs stamped with their record number + 1).
// `known_valid`: the records were found valid before and not committed since, so no writer has reused them (a writer
// waits for pub_tail, which the commit warp moves only past committed records): nrec, and only the values are loaded.
__device__ __forceinline__ uint32_t pubrec_probe(const apus_pubrec_t *ring, uint64_t rn0, uint32_t nrec, int lane, uint64_t &v,
                                                 bool known_valid = false)
{
    const uint64_t rn = rn0 + (uint64_t)(lane >> 3);
    uint64_t st = 0;
    v = 0;
    if ((uint32_t)(lane >> 3) < nrec) ld_relaxed_sys_2x64(&ring[rn & PUBMASK].w[2 * (lane & 7)], st, v);
    if (known_valid) return nrec;
    const uint32_t okm = __ballot_sync(0xffffffffu, st == rn + 1);
    uint32_t n = 0;
    while (n < nrec && ((okm >> (8 * n)) & 0xffu) == 0xffu) n++;
    return n;
}
// field f (PR_*) of record q of a probe, from lane 8q + f, in every lane
__device__ __forceinline__ uint64_t pubrec_field(uint64_t v, uint32_t q, int f)
{
    return __shfl_sync(0xffffffffu, v, 8 * (int)q + f);
}
// what the commit warp's bookkeeping takes from the newest committed record
struct PubRec {
    uint64_t cum, end, tickets, tail, hwm, next_idx;
};
__device__ __forceinline__ PubRec pubrec_decode(uint64_t v, uint32_t q)
{
    PubRec r;
    r.cum = pubrec_field(v, q, PR_CUM);
    r.end = pubrec_field(v, q, PR_END);
    r.tickets = pubrec_field(v, q, PR_TICKETS);
    r.tail = pubrec_field(v, q, PR_TAIL);
    r.hwm = pubrec_field(v, q, PR_HWM);
    r.next_idx = pubrec_field(v, q, PR_NEXTIDX);
    return r;
}

// the 16 B chunk v of the image at log offset lo (16 B aligned), restricted to [a, b), into the local log and every
// follower's.  A whole chunk is one 16 B store per replica -- in fabric mode ONE multicast store that the switch fans
// out (leader egress 1x instead of (N-1)x); a chunk at an edge of the range is stored byte by byte.
__device__ __forceinline__ void push_chunk(uint8_t *entries, uint8_t *mc_entries, uint8_t *const *peer_entries, int N,
                                           uint64_t lo, const uint4 v, uint64_t a, uint64_t b)
{
    if (lo >= a && lo + 16 <= b) {
        if (mc_entries) {
            mst_v4(mc_entries + lo, v);
        } else {
            apus_st_v4(entries + lo, v);
#pragma unroll 1
            for (int f = 0; f < N; f++)
                if (peer_entries[f]) apus_st_v4(peer_entries[f] + lo, v);
        }
    } else {
#pragma unroll 1
        for (uint32_t j = 0; j < 16; j++) {
            const uint64_t o = lo + j;
            if (o < a || o >= b) continue;
            const uint32_t w = (j < 4) ? v.x : (j < 8) ? v.y : (j < 12) ? v.z : v.w;
            const uint32_t byte = (w >> (8 * (j & 3))) & 0xff;
            apus_st_u8(entries + o, byte);
#pragma unroll 1
            for (int f = 0; f < N; f++)
                if (peer_entries[f]) apus_st_u8(peer_entries[f] + o, byte);
        }
    }
}


// ---------------------------------------------------------------------------------
// Express path: ONE request, handled by warp 0 alone while the rest of the CTA stays parked at its barrier.
// This is the closed-loop commit-latency path (proxy.c:108-161: an application thread enqueues one request and
// spins until it is committed): slot already in registers (worker 0 polls the slot itself), placement state
// cached from the previous request, the 64+len bytes composed in a 256 B scratch, pushed with one 16 B store per
// chunk and follower, and published with a SELF-CERTIFYING record -- no system fence anywhere on the way.
// The publish turn is then HELD (nobody is waiting for it) and handed on, after a fence, when somebody else claims.
// Anything unusual (wrap, pruning due, payload in the byte ring, no room) returns 1: the tile machine takes the claim.
// ---------------------------------------------------------------------------------
struct Express {
    uint64_t next_seq;                 // slot number right after my latest claim
    PlaceRec rec;                      // placement state I handed on under stamp next_seq
    uint64_t pub_h;                    // publish-ring record number that goes with publish turn next_seq
    uint32_t have_place;               // `rec` is what the sequencer records hold
    uint32_t hold;                     // I still hold publish turn next_seq (self-certified data, not fenced yet)
    uint64_t dt[5];                    // ns of the latest request: place, compose, push, publish turn, publish (profiling)
};

__device__ __forceinline__ void express_release(apus_seq_t *seq, Express &X, int lane)
{
    // the data of my self-certified publishes becomes ordinary fenced data before anybody else may publish behind it
    __syncwarp();
    if (lane == 0) {
        __threadfence_system();
        pub_handoff(seq, X.next_seq, X.pub_h);
    }
    X.hold = 0;
    __syncwarp();
}

// 0: placed, pushed and published; 1: the tile machine takes the claim; 2: the launch is being aborted
__device__ __noinline__ int leader_express(const apus_devctx_t *__restrict__ cx, LeaderShared *S, Express &X,
                                              const uint64_t claimed, uint4 sv, const bool have_slot, uint8_t *scratch,
                                              const int lane, const uint4 pf, const uint64_t pf_pos)
{
    const int N = cx->group_size, me = cx->idx;
    const uint64_t L = cx->log_len;
    apus_ctrl_t *ctrl = reinterpret_cast<apus_ctrl_t *>(cx->region);
    apus_seq_t *seq = reinterpret_cast<apus_seq_t *>(cx->region + APUS_SEQ_OFF);
    apus_pubrec_t *pubring = reinterpret_cast<apus_pubrec_t *>(cx->region + APUS_PUBRING_OFF);
    uint8_t *entries = cx->region + cx->entries_off;
    uint32_t *lindex = reinterpret_cast<uint32_t *>(cx->region + APUS_INDEX_OFF);
    const uint64_t t_deq = (cx->flags & (APUS_FLAG_STATS | APUS_FLAG_PROFILE)) ? globaltimer_ns() : 0;

    if (!have_slot && lane < 8)
        sv = apus_ld_relaxed_sys_v4(reinterpret_cast<const uint8_t *>(cx->sub_slots + (claimed & cx->sub_mask)) + 16u * lane);
    const uint32_t to = __shfl_sync(0xffffffffu, sv.z, 0), lw = __shfl_sync(0xffffffffu, sv.w, 0);
    const uint32_t ty = (to >> APUS_SLOT_TYPE_SHIFT) & APUS_SLOT_TYPE_MASK, len = lw & 0xffffu, clt = lw >> 16;
    const uint64_t req_id = (uint64_t)__shfl_sync(0xffffffffu, sv.x, 0) | ((uint64_t)__shfl_sync(0xffffffffu, sv.y, 0) << 32);
    if (!apus_has_cmd(ty) || (to & APUS_SLOT_EXT)) return 1;
    const uint32_t es = APUS_HDR_BYTES + len, nb = 2u + len;

    // the followers' ack counts (is everybody caught up?) are needed only when the entry is published: in flight meanwhile
    const bool isf = lane < N && lane != me && cx->peer[lane];
    uint64_t ackv = 0;
    if (isf) ackv = apus_ld_relaxed_sys(&ctrl->ack[lane]);

    // ---- place turn (tail and prev_head are not needed here: the entry goes behind `end`, and I hand on my own) ----
    PlaceRec r = X.rec;
    if (!(X.have_place && X.next_seq == claimed)) {
        uint32_t ok = 1;
        if (lane == 0) ok = place_acquire(seq, claimed, r) ? 1u : 0u;
        if (!__shfl_sync(0xffffffffu, ok, 0)) return 2;
        r.placed = __shfl_sync(0xffffffffu, r.placed, 0); r.end = __shfl_sync(0xffffffffu, r.end, 0);
        r.head = __shfl_sync(0xffffffffu, r.head, 0);
        r.wrapped = __shfl_sync(0xffffffffu, r.wrapped ? 1u : 0u, 0) != 0;
        X.rec = r; X.have_place = 1; X.next_seq = claimed;
    }
    const bool wrapped = r.wrapped;
    const uint64_t placed = r.placed;
    const uint64_t pos0 = (r.end == L) ? 0 : r.end;
    const uint64_t used = (r.end == L) ? 0 : apus_ring_dist(r.head, r.end, L);
    const bool autoprune = (cx->flags & APUS_FLAG_AUTOPRUNE) != 0;
    const uint64_t reserve = autoprune ? APUS_HDR_BYTES : 0;
    // Pruning is the tile machine's business (it appends the HEAD entry): once the ring is half used every request is
    // handed over until a HEAD entry has made room.  Below that the express path does not even look at the apply offsets.
    if (autoprune && used >= (L >> 1)) return 1;
    if (pos0 + es > L || used + es + reserve >= L) return 1;          // wrap / no room: general placement

    const uint64_t a = pos0, b = pos0 + es;
    const uint64_t ne = (b == L) ? 0 : b;                             // rule E1
    const bool nw = wrapped || b == L;
    const uint64_t cum = placed + 1;
    // hand the place turn on at once (stamp = next slot number) and remember what I wrote
    const PlaceRec nr = {cum, ne, a, r.head, nw, false};
    if (lane == 0) place_handoff(seq, claimed + 1, nr);
    X.rec = nr; X.have_place = 1;
    const uint64_t idx = S->idx_base + placed + 1;
    const bool xprof = (cx->flags & APUS_FLAG_PROFILE) != 0;
    const uint64_t t_place = xprof ? globaltimer_ns() : 0;

    // ---- compose: lane c builds the 16 B chunk c of the entry.  Everything except two HOLES (bytes 41..47 and the
    //      slack behind the data image) is new; the holes keep what the log held (dare_log.h:507-529 never writes them) --
    //      those bytes were PREFETCHED while this warp was idle (pf, taken at the offset the next entry was going to get) ----
    const uint64_t a16 = a & ~15ull;
    const uint32_t nch = (uint32_t)(((b + 15ull) & ~15ull) - a16) >> 4;          // <= 11
    const uint64_t lo = a16 + 16ull * lane;
    uint4 v = make_uint4(0, 0, 0, 0);
    if ((a & 15ull) == 0) {
        uint4 oldv = make_uint4(0, 0, 0, 0);
        if (wrapped) {
            if (pf_pos == a) oldv = pf;
            else if (lane < (int)nch) oldv = apus_ld_relaxed_sys_v4(entries + lo);
        }
        const int j = lane - 3;                                       // data image chunk of this lane
        const int srcl = (j < 0) ? 0 : ((j < 2) ? j + 1 : ((j + 2) & 31));   // slot chunk holding image bytes [16j, 16j+16)
        uint4 dv;
        dv.x = __shfl_sync(0xffffffffu, sv.x, srcl); dv.y = __shfl_sync(0xffffffffu, sv.y, srcl);
        dv.z = __shfl_sync(0xffffffffu, sv.z, srcl); dv.w = __shfl_sync(0xffffffffu, sv.w, srcl);
        if (lane == 0) v = make_uint4((uint32_t)idx, (uint32_t)(idx >> 32), (uint32_t)cx->term, (uint32_t)(cx->term >> 32));
        else if (lane == 1) v = make_uint4((uint32_t)req_id, (uint32_t)(req_id >> 32), (clt & 0xffffu) | (ty << 16) | ((uint32_t)me << 24), 0u);
        else if (lane == 2) v = make_uint4(0u, 0u, oldv.z & 0xffffff00u, oldv.w);           // reply[4..12] = 0, bytes 41..47 stay
        else v = chunk_select(dv, oldv, (int)nb - 16 * j);
    } else {
        // entry at an odd offset (ragged payloads): byte-granular composition in shared memory
        uint8_t *img = scratch, *xsl = scratch + 256;
        if (lane < (int)nch)
            reinterpret_cast<uint4 *>(img)[lane] = wrapped ? apus_ld_relaxed_sys_v4(entries + lo) : make_uint4(0, 0, 0, 0);
        if (lane == 1 || lane == 2) reinterpret_cast<uint4 *>(xsl)[lane - 1] = sv;   // inline image bytes 0..31
        if (lane >= 4 && lane <= 6) reinterpret_cast<uint4 *>(xsl)[lane - 2] = sv;   // ... 32..79
        __syncwarp();
        uint8_t *e = img + (a - a16);
        group_write_header(e, lane, 32, idx, cx->term, req_id, clt, ty, me, false);
        group_copy_smem(e + E_DATA, xsl, nb, lane, 32);
        __syncwarp();
        if (lane < (int)nch) v = reinterpret_cast<const uint4 *>(img)[lane];
    }
    const uint64_t t_compose = xprof ? globaltimer_ns() : 0;

    // ---- push: local log first, then every follower; checksum of exactly the bytes [a, b) ----
    uint64_t cs = 0;
    if (lane < (int)nch) {
        cs = cs_chunk(v, lo, a, b);
        push_chunk(entries, cx->mc_region ? cx->mc_region + cx->entries_off : nullptr, S->peer_entries, N, lo, v, a, b);
    }
    {   // offset index: lane f writes replica f's word (lane `me` the local one)
        const uint32_t at = (uint32_t)cum & cx->idx_mask;
        uint32_t *ip = (lane == me) ? lindex : (lane < N ? S->peer_index[lane] : nullptr);
        if (ip) ip[at] = (uint32_t)a;
    }
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) cs += __shfl_xor_sync(0xffffffffu, cs, sft);
    // self-certify only when every follower has acked everything before this entry: each of them is then at
    // exactly `a` and can verify the one entry; a follower that lags is served by a fenced publish (it may skip records)
    const bool caught = __ballot_sync(0xffffffffu, isf && ackv != placed) == 0;

    const uint64_t t_push = xprof ? globaltimer_ns() : 0;
    // ---- publish turn (mine already when I held it) and room in the publish ring; an abort publishes nothing.  The
    //      same waits as pub_acquire, written out: through the helper this window took ~260 ns more per request (H100) ----
    uint64_t h = X.pub_h;
    uint32_t ab = 0;
    if (!X.hold) {
        if (lane == 0) {
            uint64_t sq;
            uint32_t spins = 0;
            for (;;) {
                ld_acquire_gpu_2x64(seq->pub_turn, sq, h);
                if (sq == claimed) break;
                if ((++spins & 0x3ffu) == 0 && apus_ld_relaxed_sys(&seq->abort_flag)) { ab = 1; break; }
            }
        }
        ab = __shfl_sync(0xffffffffu, ab, 0);
        if (ab) return 2;
        h = __shfl_sync(0xffffffffu, h, 0);
    }
    if (lane == 0) {
        uint32_t spins = 0;
        while (h - S->pub_tail_seen >= APUS_PUBRING_RECORDS - 2) {
            S->pub_tail_seen = apus_ld_relaxed_sys(&seq->pub_tail);
            if ((++spins & 0x3ffu) == 0 && apus_ld_relaxed_sys(&seq->abort_flag)) { ab = 1; break; }
        }
    }
    if (__shfl_sync(0xffffffffu, ab, 0)) return 2;
    const uint64_t t_turn = xprof ? globaltimer_ns() : 0;
    const uint64_t cumt = term_word(cum, cx->term);
    const bool cert = caught && !(cx->flags & APUS_FLAG_NO_EXPRESS);
    if (cx->flags & APUS_FLAG_APPLY_ANY_ROLE) {
        // my own consumers read this entry once the commit warp has acquired the record's PR_END pair (apus_dev.h):
        // the warp's local entry and index stores go before that pair
        __syncwarp();
        if (lane == 16 + PR_END) asm volatile("fence.acq_rel.gpu;" ::: "memory");
    }
    if (isf) {
        apus_ctrl_t *pc = reinterpret_cast<apus_ctrl_t *>(cx->peer[lane]);
        if (cert) {
            apus_st_relaxed_sys_2x64(&pc->pub_csum, cs + cs_key(cumt), a);
            apus_st_relaxed_sys_2x64(&pc->pub_end, ne | APUS_PUB_CERT, cumt);
        } else {
            __threadfence_system();                                  // data before tail (I1), the classic way
            apus_st_relaxed_sys_2x64(&pc->pub_end, ne, cumt);
        }
    }
    pub_record(pubring, h, lane, cum, ne, claimed + 1, t_deq, a, nw ? L : b, idx + 1, (uint64_t)es * (uint64_t)(N - 1));
    X.next_seq = claimed + 1; X.pub_h = h + 1;
    if (xprof) {
        const uint64_t t_end = globaltimer_ns();
        X.dt[0] = t_place - t_deq; X.dt[1] = t_compose - t_place; X.dt[2] = t_push - t_compose; X.dt[3] = t_turn - t_push; X.dt[4] = t_end - t_turn;
    }
    if (cert) {
        X.hold = 1;                    // nobody is waiting: keep the turn, skip the fence
    } else {
        X.hold = 0;
        __syncwarp();
        if (lane == 0) pub_handoff(seq, claimed + 1, h + 1);
    }
    return 0;
}

// ---------------------------------------------------------------------------------
// The self-certifying tail publish, read (the writers: t6_publish and leader_express)
// ---------------------------------------------------------------------------------
// {end | APUS_PUB_CERT, count|term} and the certificate half {checksum, start}, decoded.  Term fence: a publish stamped
// with another term (a deposed leader still storing) counts no entries.
struct TailPub {
    uint64_t end, cum, csum, start;
    uint32_t cert;             // self-certifying: ONE entry at `start`, no writer fence before it
};
__device__ __forceinline__ TailPub tail_pub_decode(uint64_t end_w, uint64_t cum_w, uint64_t csum, uint64_t start, uint64_t term)
{
    TailPub p;
    p.cum = term_word_is(cum_w, term) ? cum_w & APUS_PUB_CUM_MASK : 0;
    p.cert = (end_w & APUS_PUB_CERT) ? 1u : 0u;
    p.end = end_w & ~APUS_PUB_CERT;
    p.csum = csum;
    p.start = start;
    return p;
}
// warp, on a self-certifying publish p: is it exactly the next entry (ONE entry, at the walk position old_end, at most
// 496 B), and do the bytes there add up to its checksum?  An entry of up to 12 chunks is taken from the speculative read
// of lanes 4..15 (lane 4 + c holds chunk c, at spec_lo); a longer one is read again.  The key is the publish's
// count|term: p.cum > acked here, so the term fence passed and term_word rebuilds the word that was stored.
__device__ __forceinline__ bool tail_pub_verify(const TailPub &p, uint64_t old_end, uint64_t acked, uint64_t L, uint64_t term,
                                                const uint8_t *entries, const uint4 spec, uint64_t spec_lo, int lane)
{
    const uint64_t a = p.start, b = (p.end == 0) ? L : p.end;
    if (!(p.cum == acked + 1 && a == ((old_end == L) ? 0 : old_end) && b > a && b - a <= 32u * 16u - 16u)) return false;
    const uint64_t a16 = a & ~15ull;
    const uint32_t nch = (uint32_t)(((b + 15ull) & ~15ull) - a16) >> 4;
    uint64_t cs = 0;
    if (nch <= 12) {
        if (lane >= 4 && lane < 4 + (int)nch) cs = cs_chunk(spec, spec_lo, a, b);
    } else if (lane < (int)nch) cs = cs_chunk(apus_ld_relaxed_sys_v4(entries + a16 + 16ull * lane), a16 + 16ull * lane, a, b);
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) cs += __shfl_xor_sync(0xffffffffu, cs, sft);
    return (cs + cs_key(term_word(p.cum, term))) == p.csum;
}

// ---------------------------------------------------------------------------------
// Commit warp (worker 0, warp 15): one function per phase (DESIGN.md §3c) -- probe, quorum rank, commit walk, commit
// stores, heartbeat, exit decision, fin publish -- called in order by leader_commit_warp
// ---------------------------------------------------------------------------------
struct CommitWarp {            // addresses derived from cx once, then the state; the same in every lane but `peer`
    apus_ctrl_t *ctrl; apus_seq_t *seq; const apus_pubrec_t *ring; apus_loghdr_t *hdr; apus_hostwords_t *hw;
    apus_ctrl_t *peer;         // lane i: follower i's control block (null: not a follower of mine)
    int N, me, quorum;
    uint64_t committed, committed_tickets, lat_count, bytes_rep, batches;
    uint64_t tail;             // next record to commit
    uint64_t seen;             // records [tail, seen) are valid and not committed yet
    uint64_t published;        // entries published = cum of the newest valid record
    uint64_t last_progress;
    uint32_t spins, hb_spins;
    uint64_t last_hb, hb_beat; // beats keep growing across launches
};

// The commit publish {offset, term} in a follower's control block: one 16 B store by cw_commit.  The follower keeps its
// header `commit` itself (clamped to what it holds, I4); a deposed leader's offsets are dropped by the term fence.
__device__ __forceinline__ uint64_t commit_pub_offset(uint64_t off, uint64_t term_w, uint64_t term, uint64_t fallback)
{
    return term_w == term ? off : fallback;
}

// End of a bounded launch, into a follower's control block: how many entries exist, a fence, then which launch (its
// ticket target) that count belongs to -- so that the follower can leave once it has acked and applied all of them
__device__ __forceinline__ void fin_publish(apus_ctrl_t *pc, uint64_t entries, uint64_t target)
{
    apus_st_relaxed_sys(&pc->fin_entries, entries);
    __threadfence_system();
    apus_st_relaxed_sys(&pc->fin_target, target);
}
// follower warp: has the leader ended the launch `target`?  `entries` is then its count of entries (every lane)
__device__ __forceinline__ bool fin_read(const apus_ctrl_t *ctrl, uint64_t target, int lane, uint64_t &entries)
{
    uint64_t ft = 0;
    if (lane == 0) ft = ld_acquire_sys(&ctrl->fin_target);
    if (__shfl_sync(0xffffffffu, ft, 0) != target) return false;
    entries = apus_ld_relaxed_sys(&ctrl->fin_entries);
    return true;
}

// probe: every lane looks at one pair of the next four publish records; lane 0 reports what has been published.
// Returns the number of new valid records, rv the lane's pair.
__device__ __forceinline__ uint32_t cw_probe(CommitWarp &C, int lane, uint64_t &rv)
{
    const uint32_t nvalid = pubrec_probe(C.ring, C.seen, 4, lane, rv);
    if (nvalid) {
        C.published = pubrec_field(rv, nvalid - 1, PR_CUM);
        C.seen += nvalid;
        if (lane == 0) apus_st_relaxed_sys(&C.ctrl->pub_seen, C.published);
    }
    return nvalid;
}

// quorum rank: lane i holds what replica i has acked (entries, monotone), the leader's own vote is everything it has
// published (dare_ibv_rc.c:1736 "i == idx"); returns the largest count a majority (size/2+1, dare_ibv_rc.c:1741) holds
__device__ __forceinline__ uint64_t cw_quorum(const CommitWarp &C, int lane)
{
    uint64_t v = 0;
    if (lane < C.N && lane != C.me) v = apus_ld_relaxed_sys(&C.ctrl->ack[lane]);
    if (lane == C.me) v = C.published;
    // rank: how many replicas hold at least what I hold
    int cnt = 0;
    for (int j = 0; j < C.N; j++) {
        uint64_t vj = __shfl_sync(0xffffffffu, v, j);
        cnt += (vj >= v) ? 1 : 0;
    }
    uint64_t cand = (lane < C.N && cnt >= C.quorum) ? v : 0;
    for (int s = 16; s > 0; s >>= 1) {
        uint64_t o = __shfl_xor_sync(0xffffffffu, cand, s);
        cand = o > cand ? o : cand;
    }
    return cand;
}

// commit walk: map the quorum count Q to the log offset recorded at publish time -- the commit is a prefix and an entry
// boundary (invariant I3) -- over the records in [tail, seen), four per step.  The first step reuses the probe's pairs
// (rv, nvalid records) when they are exactly the pending records.  false: Q covers no record; else `last` is the newest
// covered record.
__device__ __forceinline__ bool cw_walk(const apus_devctx_t *__restrict__ cx, CommitWarp &C,
                                        uint64_t Q, uint64_t rv, uint32_t nvalid, int lane, PubRec &last)
{
    bool any = false;
    bool reuse = (C.tail + nvalid == C.seen);
    while (C.tail != C.seen) {
        uint64_t val = rv;
        uint32_t nv = nvalid;
        if (!reuse) nv = pubrec_probe(C.ring, C.tail, C.seen - C.tail < 4 ? (uint32_t)(C.seen - C.tail) : 4u, lane, val, true);
        reuse = false;
        // how many of these (up to four, in order) are covered by the quorum count
        const uint32_t cm = __ballot_sync(0xffffffffu, (lane & 7) == PR_CUM && (uint32_t)(lane >> 3) < nv && val <= Q);
        uint32_t nc = 0;
        while (nc < 4 && ((cm >> (8 * nc)) & 1u)) nc++;
        if (nc == 0) break;
        last = pubrec_decode(val, nc - 1);
        C.committed = last.cum;
        for (uint32_t q = 0; q < nc; q++) {
            C.bytes_rep += pubrec_field(val, q, PR_BYTES);
            const uint64_t t0 = pubrec_field(val, q, PR_T0);
            if ((cx->flags & APUS_FLAG_STATS) && cx->lat_ns && lane == 0) {
                const uint64_t d = globaltimer_ns() - t0;
                cx->lat_ns[(C.lat_count + q) & (APUS_LAT_RING - 1)] = d > 0xffffffffull ? 0xffffffffu : (uint32_t)d;
            }
        }
        C.lat_count += nc; C.batches += nc;
        C.tail += nc;
        any = true;
        if (nc < 4) break;
    }
    return any;
}

// commit stores: {commit offset, term} into every follower (dare_ibv_rc.c:1810), {commit offset, tickets} to the host,
// and the leader's bookkeeping, in publish order (single writer).  Records [t0, C.tail) are the ones this advance commits.
__device__ __forceinline__ void cw_commit(const apus_devctx_t *__restrict__ cx, CommitWarp &C, const PubRec &r, int lane,
                                          uint64_t t0)
{
    apus_ctrl_t *ctrl = C.ctrl;
    apus_loghdr_t *hdr = C.hdr;
    const uint64_t off = r.end, tickets = r.tickets;
    if (C.peer) apus_st_relaxed_sys_2x64(C.peer->pub_commit, off, cx->term);
    if (lane == 0) {
        // {commit offset, committed tickets}: ONE 16 B store into pinned host memory -- this is what
        // releases the proxy.c:160 spinners; a 16 B host load sees a consistent pair
        apus_st_relaxed_sys_2x64(&C.hw->commit_off, off, tickets);
        apus_st_relaxed_sys(&C.hw->consumed, tickets);                 // submission-ring space
        apus_st_relaxed_sys(&C.hw->last_commit_ns, globaltimer_ns());
        if (cx->flags & APUS_FLAG_APPLY_ANY_ROLE) {
            // my own device consumers: acquire the PR_END pair of every record this advance commits (each stored
            // behind its own writer's fence), then release the consumer record over them (apus_dev.h).  Before
            // pub_tail: none of the records is reused meanwhile
            uint64_t st_, end_;
            for (uint64_t h = t0; h != C.tail; h++) ld_acquire_gpu_2x64(&C.ring[h & PUBMASK].w[2 * PR_END], st_, end_);
            cons_publish_gpu(ctrl, off, C.committed);
        }
        apus_st_relaxed_sys(&C.seq->pub_tail, C.tail);                 // publish-ring space
        hdr->commit = off;
        // leader applies = update_state; with device consumers my apply offset is their cursor (cw_forward_apply)
        if (!(cx->flags & APUS_FLAG_APPLY_ANY_ROLE)) apus_st_relaxed_sys(&hdr->apply, off);
        hdr->end = off; hdr->tail = r.tail; hdr->old_end = off;
        ctrl->committed = C.committed; ctrl->committed_tickets = tickets; ctrl->lat_count = C.lat_count;
        ctrl->published = C.committed; ctrl->consumed = tickets; ctrl->next_idx = r.next_idx; ctrl->hwm = r.hwm;
        ctrl->bytes_replicated = C.bytes_rep; ctrl->batches = C.batches;
    }
    C.committed_tickets = tickets;
    C.last_progress = globaltimer_ns();
    __syncwarp();
}

// heartbeat (dare_ibv_rc.c:868-958: the leader writes its SID into every follower's ctrl_data.hb[]): the commit warp
// is the leader's liveness -- when the hosting process dies the context goes with it and the beats stop
__device__ __forceinline__ void cw_heartbeat(const apus_devctx_t *__restrict__ cx, CommitWarp &C, int lane)
{
    if (cx->hb_period_ns && (++C.hb_spins & 0x1fu) == 0) {
        const uint64_t now = globaltimer_ns();
        if (now - C.last_hb >= cx->hb_period_ns) {
            C.last_hb = now; C.hb_beat++;
            if (C.peer) apus_st_relaxed_sys(&C.peer->hb, term_word(C.hb_beat, cx->term));
        }
    }
}

// APUS_F_APPLY_ANY_ROLE, lane 0, every 64th pass (C.spins counts them in cw_exit) and on the way out: my device
// consumers' cursor becomes my apply offset, the one ld_apply gives the pruning rule for me -- what f_housekeeping
// forwards on a follower
__device__ __forceinline__ void cw_forward_apply(const apus_devctx_t *__restrict__ cx, const CommitWarp &C, int lane, bool last)
{
    if ((cx->flags & APUS_FLAG_APPLY_ANY_ROLE) && lane == 0 && (last || (C.spins & 0x3fu) == 0))
        apus_st_relaxed_sys(&C.hdr->apply, apus_ld_relaxed_sys(&C.ctrl->cons_cur[0]));
}

// exit decision: 1 every worker finished and nothing is in flight, 2 abort (or the watchdog), 0 go on
__device__ __forceinline__ int cw_exit(const apus_devctx_t *__restrict__ cx, CommitWarp &C, bool new_records, int lane)
{
    apus_seq_t *seq = C.seq;
    int ex = 0;
    if (lane == 0) {
        if (!new_records && C.tail == C.seen && C.committed == C.published && ld_acquire_gpu(&seq->workers_done) == cx->n_workers) {
            ex = 3;
        } else if ((++C.spins & 0x3ffu) == 0) {
            if (apus_ld_relaxed_sys(&seq->abort_flag)) ex = 2;
            else if (globaltimer_ns() - C.last_progress > WATCHDOG_NS && (C.tail != C.seen || C.committed != C.published) &&
                     (cx->target != ~0ull || apus_ld_relaxed_sys_u32(&C.hw->stop))) {
                apus_st_relaxed_sys(&C.hw->error, APUS_KERR_WATCHDOG_COMMIT);
                apus_st_relaxed_sys(&seq->abort_flag, 1);
                ex = 2;
            }
        }
    }
    ex = __shfl_sync(0xffffffffu, ex, 0);
    if (ex == 3) {
        // workers are done (acquire above): any record they wrote is visible now; one more look at the ring
        uint64_t v;
        ex = pubrec_probe(C.ring, C.seen, 1, lane, v) ? 0 : 1;
    }
    return ex;
}

__device__ void leader_commit_warp(const apus_devctx_t *__restrict__ cx)
{
    const int lane = threadIdx.x & 31;
    const int N = cx->group_size, me = cx->idx;
    apus_ctrl_t *ctrl = reinterpret_cast<apus_ctrl_t *>(cx->region);
    CommitWarp C = {ctrl, reinterpret_cast<apus_seq_t *>(cx->region + APUS_SEQ_OFF),
                    reinterpret_cast<const apus_pubrec_t *>(cx->region + APUS_PUBRING_OFF),
                    reinterpret_cast<apus_loghdr_t *>(cx->region + APUS_HDR_OFF), cx->hw,
                    (lane < N && lane != me && cx->peer[lane]) ? reinterpret_cast<apus_ctrl_t *>(cx->peer[lane]) : nullptr,
                    N, me, cx->quorum,
                    ctrl->committed, ctrl->committed_tickets, ctrl->lat_count, ctrl->bytes_replicated, ctrl->batches,
                    0, 0, ctrl->published, globaltimer_ns(), 0, 0, 0, globaltimer_ns() >> 10};
    for (;;) {
        uint64_t rv;
        const uint32_t nvalid = cw_probe(C, lane, rv);
        const uint64_t Q = cw_quorum(C, lane);
        if (Q > C.committed && C.tail != C.seen) {
            PubRec r;
            const uint64_t t0 = C.tail;
            if (cw_walk(cx, C, Q, rv, nvalid, lane, r)) cw_commit(cx, C, r, lane, t0);
        }
        cw_heartbeat(cx, C, lane);
        const int ex = cw_exit(cx, C, nvalid != 0, lane);
        cw_forward_apply(cx, C, lane, ex != 0);
        if (ex) {
            if (ex == 1 && cx->target != ~0ull && C.peer) fin_publish(C.peer, C.committed, cx->target);
            break;
        }
    }
}

// ---------------------------------------------------------------------------------
// The tile loop of a worker CTA, one function per phase (DESIGN.md §3a): T0 claim, T1 fetch, T2 place, T3 prefill,
// T4 compose, T5 store, T6 publish.  leader_main runs them in order with a CTA barrier of the producer warps between.
// ---------------------------------------------------------------------------------
// Worker 0's profile (APUS_FLAG_STATS, thread 0 alone): the phase_ns / turn_ns slots of apus_ctrl_t, kept in shared memory
// and written out after every tile and while waiting for requests.
struct LeaderProf {
    bool on;
    uint64_t *ph, *tn, tprev;      // ph / tn: LeaderShared::prof_ph / prof_tn -- only thread 0 uses them; in registers
                                    // they would take 32 from every producer thread (and the kernel spills)
    // the time since the previous mark goes to phase i
    __device__ __forceinline__ void phase(int i) { if (on) { const uint64_t t = globaltimer_ns(); ph[i] += t - tprev; tprev = t; } }
    __device__ __forceinline__ void flush(apus_ctrl_t *ctrl) const
    {
        if (on) for (int i = 0; i < 8; i++) { ctrl->phase_ns[i] = ph[i]; ctrl->turn_ns[i] = tn[i]; }
    }
};

// T0 claim (warp 0): take the next slots of the submission ring -- lock-free, one compare-and-swap on the
// claimed-slots counter.  The claimed range [slot0, slot0+n) is also the worker's place in the order: the place and
// publish turns are stamped with slot numbers.  A lone request is taken by the express path right here; a claim for the
// tile machine leaves with S->n_fetch > 0, a stop or an abort with S->finish.
//
// Every worker contends for the counter, so a claim costs as few dependent round trips as possible (DESIGN.md §3a): a
// pass issues its loads together (counter, doorbell, claim-sizing averages, w0_idle, every 64th pass the abort flag),
// then, only when there is something to claim, the compare-and-swap with an acquire re-read of the doorbell beside it.
// A failed compare-and-swap returns the current counter: lane 0 decides the claim again from that value and the
// doorbell already read, and retries at once.  That retry loop reads the abort flag; a stop and the watchdog are
// checked by the passes around it, and the loop ends because every lost attempt moves the counter towards `t`.
__device__ __forceinline__ void t0_claim(const apus_devctx_t *__restrict__ cx, LeaderShared *S, Express &X,
                                         uint64_t &xguess, uint4 &pf, uint64_t &pf_pos, uint64_t &last_progress,
                                         LeaderProf &P, const uint32_t wid, const int lane)
{
    apus_ctrl_t *ctrl = reinterpret_cast<apus_ctrl_t *>(cx->region);
    apus_seq_t *seq = reinterpret_cast<apus_seq_t *>(cx->region + APUS_SEQ_OFF);
    apus_hostwords_t *hw = cx->hw;
    uint8_t *entries = cx->region + cx->entries_off;
    uint32_t n = 0, fin = 0, spins = 0, lone_waits = 0;
    const uint64_t tw0 = P.on ? globaltimer_ns() : 0;
    uint64_t claimed = 0;
    const bool poll_slot = cx->slot_poll != 0 && wid == 0;
    const bool express_on = (cx->flags & APUS_FLAG_NO_EXPRESS) == 0;
    if (wid == 0 && lane == 0) apus_st_relaxed_sys(&seq->w0_idle, 1);
    for (;;) {
        // worker 0 polls the NEXT SLOT itself (lanes 0..7, one 128 B read over PCIe) while lane 0 looks at the
        // claim counter and the doorbell: a lone request is in registers one PCIe round trip after the host wrote it
        uint4 sv = make_uint4(0, 0, 0, 0);
        const uint64_t sv_for = xguess;
        if (poll_slot && lane < 8)
            sv = apus_ld_relaxed_sys_v4(reinterpret_cast<const uint8_t *>(cx->sub_slots + (xguess & cx->sub_mask)) + 16u * lane);
        // (a second poll in flight does not help: two loads of one line from one SM are merged, the younger one
        //  returns the older one's sample, and the extra load only lengthens the loop)
        // idle-time prefetch: the bytes the log holds where the NEXT entry will go (its holes keep them); the offset
        // is known as long as this warp placed the latest entry
        if (express_on && X.have_place && X.rec.end != cx->log_len && X.rec.wrapped && pf_pos != X.rec.end &&
            (X.rec.end & 15ull) == 0 && X.rec.end + 16ull * 12 <= cx->log_len) {
            if (lane < 12) pf = apus_ld_relaxed_sys_v4(entries + X.rec.end + 16ull * lane);
            pf_pos = X.rec.end;
        }
        // lane 0: one round trip of independent loads (the averages are small: their low 32 bits hold them); the
        // doorbell is read relaxed here and with acquire next to the compare-and-swap
        uint32_t ctl = 0, aes = 0, axb = 0;
        uint64_t t = 0, w0i = 0, ab = 0;
        if (lane == 0) {
            if ((spins & 0x3fu) == 0) ab = apus_ld_relaxed_sys(&seq->abort_flag);
            t = cx->doorbell_relay ? apus_ld_relaxed_sys(&seq->doorbell) : apus_ld_relaxed_sys(cx->sub_tail);
            claimed = apus_ld_relaxed_sys(&seq->claimed_slots);
            if (wid != 0) w0i = apus_ld_relaxed_sys(&seq->w0_idle);
            aes = apus_ld_relaxed_sys_u32(&seq->avg_es); axb = apus_ld_relaxed_sys_u32(&seq->avg_xb);
            // worker 0 waits for its slot poll (a PCIe round trip) in every pass anyway: there, a doorbell that shows
            // requests is re-read with acquire at once, under the poll, and not beside the compare-and-swap
            if (poll_slot && t > claimed) t = cx->doorbell_relay ? ld_acquire_gpu(&seq->doorbell) : ld_acquire_sys(cx->sub_tail);
            if (ab || claimed >= cx->target) ctl = 1;
        }
        ctl = __shfl_sync(0xffffffffu, ctl, 0);
        claimed = __shfl_sync(0xffffffffu, claimed, 0);
        t = __shfl_sync(0xffffffffu, t, 0);
        w0i = __shfl_sync(0xffffffffu, w0i, 0);
        // a held publish turn is passed on as soon as anybody else has claimed slots (or I am leaving)
        if (X.hold && (ctl || claimed != X.next_seq)) express_release(seq, X, lane);
        if (ctl) { fin = 1; break; }
        bool slot_ok = false;
        if (poll_slot) {
            const uint64_t stamp = (uint64_t)sv.x | ((uint64_t)sv.y << 32);
            slot_ok = (__ballot_sync(0xffffffffu, (lane == 3 || lane == 7) && stamp == sv_for + 1) == 0x88u) && sv_for == claimed;
            xguess = claimed;
        }
        uint64_t avail = t > claimed ? t - claimed : 0;
        if (slot_ok && avail == 0) avail = 1;
        // the doorbell may show a lone request before the slot poll in flight does: wait for the poll (next
        // iteration) instead of claiming now and fetching the slot with one more PCIe round trip
        if (poll_slot && express_on && avail == 1 && !slot_ok && ++lone_waits < 8) avail = 0; else lone_waits = 0;
        // lone requests belong to worker 0 while it is polling (express path)
        if (avail == 1 && wid != 0 && w0i) avail = 0;
        if (avail) {
            uint32_t nn = 0, won = 0;
            if (lane == 0) {
                // a claim should fit ONE tile image / staging buffer (else it is placed in pieces while holding the
                // place turn, which serializes the workers)
                if (aes < 64) aes = 128;
                uint32_t fit = (APUS_LEADER_IMG_BYTES - 256u) / aes;
                if (axb) { const uint32_t xf = APUS_LEADER_EXT_BYTES / axb; if (xf < fit) fit = xf; }
                if (fit < 1) fit = 1;
                const uint32_t cap = fit > MAXB ? MAXB : fit;
                // claim; a lost compare-and-swap returns the counter: decide again from it and the doorbell already
                // read.  This loop ends: every lost attempt moved the counter towards `t`.  It reads the abort flag
                // every 64 attempts; a stop and the watchdog are looked at by the passes around it.  (`lost`, not
                // `spins`: the pass counter must stay the same in every lane, the stop check below is warp-wide.)
                for (uint32_t lost = 0;; lost++) {
                    const uint64_t room = cx->target - claimed;
                    if (avail > room) avail = room;
                    // share a shallow queue between the workers instead of one big tile
                    uint64_t want = (avail + cx->n_workers - 1) / cx->n_workers;
                    if (want < 32) want = avail < 32 ? avail : 32;
                    nn = want > cap ? cap : (uint32_t)want;
                    const uint64_t was = atomicCAS(reinterpret_cast<unsigned long long *>(&seq->claimed_slots),
                                                   (unsigned long long)claimed, (unsigned long long)(claimed + nn));
                    // the doorbell again, with acquire, in flight with the compare-and-swap: it shows at least `t` and
                    // orders the fetch of the claimed slots after it (not for a lone request that only the slot poll
                    // has shown: its stamp is what publishes it; not for worker 0, which has read `t` with acquire)
                    if (t > claimed && !poll_slot) (void)(cx->doorbell_relay ? ld_acquire_gpu(&seq->doorbell) : ld_acquire_sys(cx->sub_tail));
                    if (was == claimed) { won = 1; break; }
                    claimed = was;
                    if (claimed >= cx->target) break;
                    if ((lost & 0x3fu) == 0x3fu && apus_ld_relaxed_sys(&seq->abort_flag)) break;
                    avail = t > claimed ? t - claimed : 0;
                    // a lone request: worker 0 waits for its slot poll (the next pass), the others leave it to worker 0
                    if (avail == 1 && ((poll_slot && express_on) || (wid != 0 && w0i))) avail = 0;
                    if (!avail) break;
                }
            }
            won = __shfl_sync(0xffffffffu, won, 0);
            claimed = __shfl_sync(0xffffffffu, claimed, 0);
            if (won) {
                nn = __shfl_sync(0xffffffffu, nn, 0);
                if (X.hold && claimed != X.next_seq) express_release(seq, X, lane);   // won after a lost attempt
                if (nn == 1 && express_on) {
                    const int rc = leader_express(cx, S, X, claimed, sv, slot_ok && claimed == sv_for, smem_raw + L_IMG_OFF,
                                                  lane, pf, pf_pos);
                    if (rc == 0) {
                        xguess = claimed + 1; last_progress = globaltimer_ns();
                        if (P.on) { P.tn[5]++; P.ph[7]++; for (int q = 0; q < 5; q++) P.ph[1 + q] += X.dt[q]; }
                        continue;
                    }
                    if (rc == 2) { fin = 1; break; }
                    // rc == 1: the tile machine places this claim; the cached placement state is still what the records hold
                }
                n = nn;
                break;
            }
        }
        if ((++spins & 0x1ffu) == 0) {
            // stop / watchdog (the abort flag is not raised on a stop: this worker holds no turn)
            uint32_t stopf = 0;
            if (lane == 0) {
                if (apus_ld_relaxed_sys_u32(&hw->stop)) stopf = 1;
                else if (cx->target != ~0ull && globaltimer_ns() - last_progress > WATCHDOG_NS) {
                    apus_st_relaxed_sys(&hw->error, APUS_KERR_WATCHDOG_LEADER);
                    apus_st_relaxed_sys(&seq->abort_flag, 1); stopf = 1;
                }
                P.flush(ctrl);
            }
            stopf = __shfl_sync(0xffffffffu, stopf, 0);
            if (stopf) { fin = 1; break; }
        }
    }
    if (X.hold) express_release(seq, X, lane);
    X.have_place = 0; pf_pos = ~0ull;                  // other workers may place in between
    if (lane == 0) {
        if (wid == 0) apus_st_relaxed_sys(&seq->w0_idle, 0);
        if (P.on) { P.tn[0] += globaltimer_ns() - tw0; P.tn[6]++; }
        if (n) S->slot0 = claimed;
        S->n_fetch = n; S->finish = fin;
        DescReduce R0;
        R0.init();
        S->r_es_min = R0.es_min; S->r_es_max = R0.es_max; S->r_xb_min = R0.xb_min; S->r_xb_max = R0.xb_max;
        S->r_cut = R0.cut; S->r_fext = R0.fext; S->r_hh1 = R0.hh1;
        S->t_dequeue = globaltimer_ns();
    }
}

// T1 fetch (all producer threads): the claimed slots (descriptor + inline payload), coalesced 16 B loads; the
// descriptors are reduced on the way (DescReduce)
__device__ __forceinline__ void t1_fetch(const apus_devctx_t *__restrict__ cx, LeaderShared *S, int tid)
{
    uint8_t *slots = smem_raw + L_SLOTS_OFF;
    const uint32_t nf = S->n_fetch;
    const uint64_t s0 = S->slot0 & cx->sub_mask;
    const uint64_t nslots = (uint64_t)cx->sub_mask + 1;
    const uint32_t first = (s0 + nf <= nslots) ? nf : (uint32_t)(nslots - s0);   // ring wrap: two runs
    cta_fetch_slots(S, slots, cx->sub_slots, s0, 0, first, tid);
    if (first < nf) cta_fetch_slots(S, slots, cx->sub_slots, 0, first, nf - first, tid);
    if (tid == 0) S->kbase = 0;
}

// lane 0 of T2, first sub-tile of a claim: take the place turn.  When the whole claim fits contiguously and no pruning
// is due (the common case: the turn is held for a dozen integer operations) place it at once and hand the turn on
// (S->fast); else leave the state in S->st for leader_place.
__device__ __forceinline__ void place_fast(const apus_devctx_t *__restrict__ cx, LeaderShared *S, LeaderProf &P)
{
    apus_ctrl_t *ctrl = reinterpret_cast<apus_ctrl_t *>(cx->region);
    apus_seq_t *seq = reinterpret_cast<apus_seq_t *>(cx->region + APUS_SEQ_OFF);
    apus_loghdr_t *hdr = reinterpret_cast<apus_loghdr_t *>(cx->region + APUS_HDR_OFF);
    const apus_cslot_t *sl = reinterpret_cast<const apus_cslot_t *>(smem_raw + L_SLOTS_OFF);
    const uint64_t L = cx->log_len;
    const uint32_t nf = S->n_fetch;
    const uint64_t tw0 = P.on ? globaltimer_ns() : 0;
    PlaceRec r;
    const bool got = place_acquire(seq, S->slot0, r);
    if (P.on) { P.tn[1] += globaltimer_ns() - tw0; S->t_place_acq = globaltimer_ns(); }
    if (!got) { S->abort = 1; S->fast = 1; S->blocked = 0; return; }   // no stamp: nothing may be placed

    const uint64_t pos0 = (r.end == L) ? 0 : r.end;
    const uint64_t used = (r.end == L) ? 0 : apus_ring_dist(r.head, r.end, L);
    const uint64_t total = S->cum_es[nf - 1];
    const bool autoprune = (cx->flags & APUS_FLAG_AUTOPRUNE) != 0;
    const uint64_t reserve = autoprune ? APUS_HDR_BYTES : 0;
    // is the pruning rule due?  (scalar version of the test in leader_place)
    bool prune_due = false;
    if (autoprune && r.end != L && used >= (L >> 2) && !r.prev_head && L - pos0 >= APUS_HDR_BYTES) {
        if (!S->ap_valid) {
            for (int i = 0; i < cx->group_size; i++) S->ap[i] = ld_apply(cx, ctrl, hdr, i);
            S->ap_valid = 1;
        }
        uint64_t d = 0;
        for (int i = 0; i < cx->group_size; i++) {
            uint64_t di = apus_ring_dist(S->ap[i], r.end, L);
            if (di > used) di = used;
            d = di > d ? di : d;
        }
        if (d == 0) d = apus_ring_dist(r.tail, r.end, L);
        prune_due = (d <= used && used - d >= (L >> 3));
    }
    const bool fits = !prune_due && pos0 + total <= L && total <= APUS_LEADER_IMG_BYTES - 16u - (pos0 & 15u) &&
                      used + total + reserve < L && S->cum_xb[nf - 1] <= APUS_LEADER_EXT_BYTES && S->static_cut == nf;
    if (!fits) {
        S->st = r;
        S->st_hwm = r.wrapped ? L : pos0;
        S->fast = 0;
        if (P.on) P.tn[4]++;
        return;
    }
    const uint64_t b = pos0 + total;
    const uint64_t ne = (b == L) ? 0 : b;
    const uint64_t nt = b - S->es[nf - 1];
    const bool nw = r.wrapped || b == L;
    uint64_t headv = r.head;
    if (S->host_head_k != 0xffffffffu) {          // a HEAD entry submitted by the host carries the new head
        const uint64_t nh = adopt_head(headv, le_u64(sl[S->host_head_k].inl), ne, L);
        if (nh != headv) { headv = nh; apus_st_relaxed_sys(&hdr->head, nh); }
    }
    // hand the turn on at once ...
    const PlaceRec nr = {r.placed + nf, ne, nt, headv, nw, false};
    place_handoff(seq, S->slot0 + nf, nr);
    if (P.on) { P.tn[7] += globaltimer_ns() - S->t_place_acq; P.tn[3]++; }
    // ... and only then write down the tile for the other warps
    S->gap = 0; S->ghost = 0; S->blocked = 0; S->last = 1;
    S->a = pos0; S->b = b; S->m = nf;
    S->hbytes = 0; S->base_es = 0; S->base_xb = 0;
    S->ext_bytes = (S->first_ext_all != 0xffffffffu) ? S->cum_xb[nf - 1] : 0u;
    S->ext_base = (S->first_ext_all != 0xffffffffu)
                      ? (uint64_t)(sl[S->first_ext_all].type_off & APUS_SLOT_OFF_MASK) * 16ull : 0ull;
    S->auto_head = 0; S->auto_head_val = 0;
    S->idx0 = S->idx_base + r.placed + 1;
    S->fresh = r.wrapped ? 0u : 1u;
    S->new_end = ne; S->tail_after = nt; S->cum_after = r.placed + nf;
    S->hwm_after = nw ? L : b;
    S->fast = 1;
}

// T2 place (warp 0): the next sub-tile of the fetched batch.  For the first one the turn and the fast path (the
// state-independent part was done by all producer threads in t1_scan); what the fast path does not place is placed by
// leader_place while the turn is held, and the state is handed on with the last sub-tile.
__device__ __forceinline__ void t2_place(const apus_devctx_t *__restrict__ cx, LeaderShared *S, bool have_place_turn,
                                         LeaderProf &P, int lane)
{
    const int N = cx->group_size;
    apus_ctrl_t *ctrl = reinterpret_cast<apus_ctrl_t *>(cx->region);
    apus_seq_t *seq = reinterpret_cast<apus_seq_t *>(cx->region + APUS_SEQ_OFF);
    apus_loghdr_t *hdr = reinterpret_cast<apus_loghdr_t *>(cx->region + APUS_HDR_OFF);
    if (!have_place_turn) {
        if (lane == 0) place_fast(cx, S, P);
        __syncwarp();
        if (S->fast) return;
    }
    if (!S->ap_valid) {
        if (lane < N) S->ap[lane] = ld_apply(cx, ctrl, hdr, lane);
        __syncwarp();
        if (lane == 0) S->ap_valid = 1;
        __syncwarp();
    }
    leader_place(cx, S, reinterpret_cast<const apus_cslot_t *>(smem_raw + L_SLOTS_OFF), lane);
    if (lane == 0 && S->last) {
        // all my slots are placed: hand the placement state to the next claim
        S->st.wrapped = S->st_hwm == cx->log_len;
        place_handoff(seq, S->slot0 + S->n_fetch, S->st);
        if (P.on) P.tn[7] += globaltimer_ns() - S->t_place_acq;
    }
}

// T3 prefill (all producer threads): the image gets zeros when the range is fresh, else the bytes the local log holds
// (holes of an entry keep what was there, like the reference), and the payload-ring range of the sub-tile is staged;
// all loads in flight together.
// A composed entry overwrites all of its bytes except two HOLES -- bytes 41..47 of the header and the slack behind the
// data image ([48 + nb, stride): 14 bytes for a request) -- which keep what the log held (dare_log.h:507-529 never
// writes them).  For tiles of large entries only the chunks that overlap a hole are brought in; small entries are
// mostly holes' neighbours, the whole range is read in one coalesced sweep.
__device__ __forceinline__ void hole_chunks(const LeaderShared *S, const apus_cslot_t *sl, uint32_t j, uint64_t lo[4])
{
    uint32_t rel, es_, nb_;
    if (S->auto_head && j == 0) { rel = 0; es_ = APUS_HDR_BYTES; nb_ = 8; }
    else {
        const uint32_t k = S->kbase + j - S->auto_head;
        rel = S->hbytes + (S->cum_es[k] - S->base_es) - S->es[k];
        es_ = S->es[k]; nb_ = data_bytes(S->ty[k], sl[k].len);
    }
    const uint64_t eo = S->a + rel;
    const uint64_t h0 = eo + 41, h1 = eo + 47, g0 = eo + 48 + nb_, g1 = eo + es_ - 1;   // hole byte ranges (inclusive)
    const uint64_t cs[4] = { h0 >> 4, h1 >> 4, g0 >> 4, g1 >> 4 };
#pragma unroll
    for (int q = 0; q < 4; q++) {
        lo[q] = cs[q] << 4;
        if (q >= 2 && g1 < g0) lo[q] = ~0ull;                     // no slack
        else if (q > 0 && cs[q] == cs[q - 1]) lo[q] = ~0ull;      // same chunk as the previous hole
    }
}

__device__ __noinline__ void t3_prefill(const apus_devctx_t *__restrict__ cx, LeaderShared *S, int tid)
{
    const apus_cslot_t *sl = reinterpret_cast<const apus_cslot_t *>(smem_raw + L_SLOTS_OFF);
    uint8_t *ext = smem_raw + L_EXT_OFF;
    uint8_t *img = smem_raw + L_IMG_OFF;
    const uint8_t *entries = cx->region + cx->entries_off;
    const uint32_t kbase = S->kbase, m = S->m, gap = S->gap, autoh = S->auto_head;
    const uint64_t a = S->a, b = S->b;
    const uint64_t a16 = a & ~15ull;
    const uint32_t nchunks = (uint32_t)(((b + 15ull) & ~15ull) - a16) >> 4;
    const bool holes_only = !gap && (b - a) >= (uint64_t)(m + autoh) * 512ull;
    if (holes_only) {
        // the (up to four) hole chunks of an entry are loaded together (zeroed first, see cta_fetch_slots)
        const uint64_t hi16 = a16 + 16ull * nchunks;
        const bool fresh = S->fresh != 0;
        for (uint32_t j = tid; j < m + autoh; j += NT) {
            uint64_t lo[4];
            hole_chunks(S, sl, j, lo);
            uint4 v[4];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                v[q] = make_uint4(0, 0, 0, 0);
                if (!fresh && lo[q] >= a16 && lo[q] < hi16) v[q] = apus_ld_relaxed_sys_v4(entries + lo[q]);
            }
#pragma unroll
            for (int q = 0; q < 4; q++)
                if (lo[q] >= a16 && lo[q] < hi16) reinterpret_cast<uint4 *>(img)[(lo[q] - a16) >> 4] = v[q];
        }
    } else if (S->fresh) {
        for (uint32_t c = tid; c < nchunks; c += NT) reinterpret_cast<uint4 *>(img)[c] = make_uint4(0, 0, 0, 0);
    } else {
        cta_fetch_chunks(img, entries + a16, nchunks, tid, NT);
    }
    if (!gap && S->ext_bytes) cta_fetch_chunks(ext, cx->sub_pay + S->ext_base, S->ext_bytes >> 4, tid, NT);
    for (uint32_t j = tid; j < m; j += NT) {
        const uint32_t k = kbase + j;
        S->rel[k] = S->hbytes + (S->cum_es[k] - S->base_es) - S->es[k];
        S->xoff[k] = (S->cum_xb[k] - S->base_xb) - S->xb[k];
    }
}

// T4 compose (all producer warps): the entries of the sub-tile into the image
__device__ __noinline__ void t4_compose(const apus_devctx_t *__restrict__ cx, const LeaderShared *S, int warp, int lane)
{
    const apus_cslot_t *sl = reinterpret_cast<const apus_cslot_t *>(smem_raw + L_SLOTS_OFF);
    const uint8_t *ext = smem_raw + L_EXT_OFF;
    uint8_t *img = smem_raw + L_IMG_OFF;
    const int me = cx->idx;
    const uint32_t kbase = S->kbase, m = S->m, autoh = S->auto_head;
    const uint64_t a = S->a, b = S->b;
    uint8_t *e0 = img + (a & 15ull);                  // the entry at offset a
    if (S->gap) {
        if (S->ghost && warp == 0) {
            // header of the wrapping entry without payload, sender untouched (dare_log.h:496-503, 521)
            group_write_header(e0, lane, 32, S->idx0, cx->term, sl[kbase].req_id, sl[kbase].clt_id, S->ty[kbase], 0, true);
            if (lane == 8) { e0[E_DATA] = (uint8_t)(sl[kbase].len & 0xff); e0[E_DATA + 1] = (uint8_t)(sl[kbase].len >> 8); }
        }
        return;
    }
    if (autoh && warp == N_PRODUCER_WARPS - 1) {
        // <HEAD, head_offset> entry (dare_log.h:29-32, dare_server.c:2043-2046)
        group_write_header(e0, lane, 32, S->idx0, cx->term, 0, 0, T_HEAD, me, false);
        if (lane >= 8 && lane < 16) e0[E_DATA + lane - 8] = (uint8_t)(S->auto_head_val >> (8 * (lane - 8)));
    }
    // small entries: 8 lanes per entry (4 entries per warp step); large ones: the whole warp
    const bool small = (b - a) <= (uint64_t)(m + autoh) * 256ull;
    const int gl = small ? 8 : 32;
    const int grp = small ? (lane >> 3) : 0, sub = small ? (lane & 7) : lane;
    const uint32_t per_step = small ? 4u * N_PRODUCER_WARPS : N_PRODUCER_WARPS;
    for (uint32_t j = (small ? warp * 4u + grp : warp); j < m; j += per_step) {
        const uint32_t k = kbase + j;
        uint8_t *e = e0 + S->rel[k];
        const uint32_t ty = S->ty[k];
        const uint32_t nb = data_bytes(ty, sl[k].len);
        const uint32_t es_k = S->es[k];
        if (((uint32_t)(uintptr_t)e & 15u) == 0 && (es_k & 15u) == 0) {
            // the entry occupies whole 16 B chunks of the image: lane `sub` builds chunks sub, sub+gl, ... in
            // registers (header fields; the data image straight from the slot / the staged payload) and
            // writes each with ONE 16 B store; the two holes keep what the prefill put there
            const uint64_t idx = S->idx0 + autoh + j, rq = sl[k].req_id;
            const uint8_t *src = (S->flg[k] & 1u) ? ext + S->xoff[k] : sl[k].inl;
            const uint32_t nch_e = es_k >> 4;
            for (uint32_t c = (uint32_t)sub; c < nch_e; c += (uint32_t)gl) {
                uint4 *dst = reinterpret_cast<uint4 *>(e) + c;
                if (c == 0) *dst = make_uint4((uint32_t)idx, (uint32_t)(idx >> 32), (uint32_t)cx->term, (uint32_t)(cx->term >> 32));
                else if (c == 1) *dst = make_uint4((uint32_t)rq, (uint32_t)(rq >> 32),
                                                   ((uint32_t)sl[k].clt_id) | (ty << 16) | ((uint32_t)me << 24), 0u);
                else if (c == 2) { const uint4 o = *dst; *dst = make_uint4(0u, 0u, o.z & 0xffffff00u, o.w); }
                else {
                    const int nbv = (int)nb - 16 * (int)(c - 3);
                    if (nbv >= 16) *dst = *reinterpret_cast<const uint4 *>(src + 16u * (c - 3));
                    else if (nbv > 0) *dst = chunk_select(*reinterpret_cast<const uint4 *>(src + 16u * (c - 3)), *dst, nbv);
                }
            }
        } else {
            group_write_header(e, sub, gl, S->idx0 + autoh + j, cx->term, sl[k].req_id, sl[k].clt_id, ty, me, false);
            if (nb) group_copy_smem(e + E_DATA, (S->flg[k] & 1u) ? ext + S->xoff[k] : sl[k].inl, nb, sub, gl);
        }
    }
}

// T5 store (all producer threads): the byte range [a,b) to the local log and to every follower, then the offset index
__device__ __noinline__ void t5_store(const apus_devctx_t *__restrict__ cx, const LeaderShared *S, int tid)
{
    const int N = cx->group_size;
    const uint8_t *img = smem_raw + L_IMG_OFF;
    uint8_t *entries = cx->region + cx->entries_off;
    uint32_t *lindex = reinterpret_cast<uint32_t *>(cx->region + APUS_INDEX_OFF);
    uint8_t *mc_entries = cx->mc_region ? cx->mc_region + cx->entries_off : nullptr;
    const uint32_t kbase = S->kbase, m = S->m, autoh = S->auto_head;
    const uint64_t a = S->a, b = S->b;
    const uint64_t a16 = a & ~15ull;
    const uint32_t nchunks = (uint32_t)(((b + 15ull) & ~15ull) - a16) >> 4;
    for (uint32_t c = tid; c < nchunks; c += NT)
        push_chunk(entries, mc_entries, S->peer_entries, N, a16 + 16ull * c, reinterpret_cast<const uint4 *>(img)[c], a, b);
    if (S->gap) return;
    // entry-offset index: the c-th entry ever appended sits at index[c & idx_mask]
    const uint64_t cum0 = S->cum_after - (m + autoh);
    for (uint32_t j = tid; j < m + autoh; j += NT) {
        uint32_t w;
        if (autoh && j == 0) w = (uint32_t)a | APUS_IDX_HEAD_FLAG;
        else {
            const uint32_t k = kbase + j - autoh;
            w = (uint32_t)(a + S->rel[k]) | (S->ty[k] == T_HEAD ? APUS_IDX_HEAD_FLAG : 0u);
        }
        const uint32_t at = (uint32_t)(cum0 + 1 + j) & cx->idx_mask;
        if (cx->mc_region) {
            mst_u32(reinterpret_cast<uint32_t *>(cx->mc_region + APUS_INDEX_OFF) + at, w);
        } else {
            lindex[at] = w;
#pragma unroll 1
            for (int f = 0; f < N; f++)
                if (S->peer_index[f]) S->peer_index[f][at] = w;
        }
    }
}

// T6 publish (warp 0): the tail in claim order (data before tail, invariant I1)
__device__ __forceinline__ void t6_publish(const apus_devctx_t *__restrict__ cx, LeaderShared *S, bool have_pub_turn,
                                           uint64_t gap_bytes, LeaderProf &P, int lane)
{
    const int N = cx->group_size, me = cx->idx;
    apus_seq_t *seq = reinterpret_cast<apus_seq_t *>(cx->region + APUS_SEQ_OFF);
    apus_pubrec_t *pubring = reinterpret_cast<apus_pubrec_t *>(cx->region + APUS_PUBRING_OFF);
    const bool pubs = lane < N && lane != me && cx->peer[lane];
    // data before tail (invariant I1): all data stores of the tile -> bar.sync (before this phase) -> one system
    // fence per publishing lane (cumulative over the barrier) -> the tail.  A system fence costs microseconds;
    // fencing in every warp serializes 15 of them.  With device consumers on this leader (APUS_F_APPLY_ANY_ROLE) the
    // lane that stores the record's PR_END pair fences too, in the same instruction: the commit warp acquires that pair
    // before it publishes the consumer record (apus_dev.h).
    if (pubs || ((cx->flags & APUS_FLAG_APPLY_ANY_ROLE) && lane == 16 + PR_END)) __threadfence_system();
    // the publish turn: {slot number, record number} in one 16 B word.  Held for the N-1 tail stores
    // and the eight 16 B stores of the publish record -- no fence inside the turn
    if (lane == 0) {
        uint64_t h = S->pub_h;
        if (!pub_acquire(seq, S->slot0, have_pub_turn, h, S->pub_tail_seen, P.on, P.tn[2])) S->abort = 1;
        S->pub_h = h;
    }
    __syncwarp();
    if (S->abort) return;
    if (pubs) {
        apus_ctrl_t *pc = reinterpret_cast<apus_ctrl_t *>(cx->peer[lane]);
        apus_st_relaxed_sys_2x64(&pc->pub_end, S->new_end, term_word(S->cum_after, cx->term));
    }
    pub_record(pubring, S->pub_h, lane, S->cum_after, S->new_end, S->slot0 + S->kbase + S->m, S->t_dequeue,
               S->tail_after, S->hwm_after, S->idx0 + S->m + S->auto_head, (S->b - S->a + gap_bytes) * (uint64_t)(N - 1));
    __syncwarp();
    if (lane == 0) {
        S->pub_h += 1;
        if (S->last) pub_handoff(seq, S->slot0 + S->n_fetch, S->pub_h);
        S->kbase += S->m;
    }
}

__device__ void leader_main(const apus_devctx_t *__restrict__ cx, const uint32_t wid)
{
    LeaderShared *S = reinterpret_cast<LeaderShared *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = cx->group_size, me = cx->idx;
    apus_ctrl_t *ctrl = reinterpret_cast<apus_ctrl_t *>(cx->region);
    apus_seq_t *seq = reinterpret_cast<apus_seq_t *>(cx->region + APUS_SEQ_OFF);
    apus_pubrec_t *pubring = reinterpret_cast<apus_pubrec_t *>(cx->region + APUS_PUBRING_OFF);
    apus_loghdr_t *hdr = reinterpret_cast<apus_loghdr_t *>(cx->region + APUS_HDR_OFF);
    apus_hostwords_t *hw = cx->hw;

    // ---- sequencer reset handshake: worker 0 prepares the shared words of this launch ----
    if (tid == 0) {
        if (wid == 0) {
            seq->claimed_slots = ctrl->consumed;
            seq->doorbell = ctrl->consumed;
            seq->workers_done = 0; seq->abort_flag = 0; seq->w0_idle = 0;
            for (uint32_t i = 0; i < APUS_PUBRING_RECORDS; i++)
                for (int q = 0; q < 8; q++) pubring[i].w[2 * q] = 0;          // no valid record
            // the turns are stamped with slot numbers: the first claim of this launch starts at ctrl->consumed
            const PlaceRec r0 = {ctrl->published, hdr->end, hdr->tail, hdr->head, ctrl->hwm == cx->log_len, false};
            place_handoff(seq, ctrl->consumed, r0);
            seq->pub_tail = 0;
            pub_handoff(seq, ctrl->consumed, 0);
            // (the commit warp keeps ctrl/hdr in step with what is COMMITTED; a clean launch ends with
            //  everything committed, so there is nothing published-but-uncommitted to carry over)
            __threadfence();
            st_release_gpu(&seq->ready_epoch, cx->epoch);
        } else {
            while (ld_acquire_gpu(&seq->ready_epoch) != cx->epoch) { }
        }
        S->finish = 0; S->abort = 0; S->was_blocked = 0; S->after_gap = 0; S->pub_tail_seen = 0; S->ap_valid = 0;
        S->idx_base = ctrl->next_idx - 1 - ctrl->published;
        for (int i = 0; i < APUS_MAX_SERVERS; i++) {
            S->peer_entries[i] = (i < N && i != me && cx->peer[i]) ? cx->peer[i] + cx->entries_off : nullptr;
            S->peer_index[i] = (i < N && i != me && cx->peer[i]) ? reinterpret_cast<uint32_t *>(cx->peer[i] + APUS_INDEX_OFF) : nullptr;
        }
    }
    __syncthreads();

    if (warp == N_PRODUCER_WARPS) {   // warp 15: the commit warp lives in worker 0
        if (wid == 0) leader_commit_warp(cx);
        else if (wid == 1 && cx->doorbell_relay && lane == 0) {
            // doorbell relay: the only poller of the host-mapped doorbell (one PCIe read in flight instead
            // of one per idle worker -- those reads also slow every system fence down); workers poll the mirror
            uint64_t last = apus_ld_relaxed_sys(&seq->doorbell);
            uint32_t spins = 0;
            for (;;) {
                const uint64_t t = ld_acquire_sys(cx->sub_tail);
                if (t != last) { st_release_gpu(&seq->doorbell, t); last = t; }   // slots were written before the doorbell
                if ((++spins & 0x3fu) == 0 &&
                    (apus_ld_relaxed_sys(&seq->abort_flag) || apus_ld_relaxed_sys(&seq->workers_done) >= cx->n_workers)) break;
            }
        }
        return;
    }

    // ---- producer warps 0..14 ------------------------------------------------------
    uint64_t last_progress = globaltimer_ns();
    LeaderProf P;
    P.on = (cx->flags & APUS_FLAG_STATS) != 0 && tid == 0 && wid == 0;
    P.ph = S->prof_ph; P.tn = S->prof_tn;
    if (tid == 0) for (int i = 0; i < 8; i++) { P.ph[i] = ctrl->phase_ns[i]; P.tn[i] = ctrl->turn_ns[i]; }
    P.tprev = globaltimer_ns();
    Express X = {};
    uint64_t xguess = ctrl->consumed;          // worker 0: the slot it expects to be claimed next
    uint4 pf = make_uint4(0, 0, 0, 0);         // express: prefetched log bytes at offset pf_pos (lane c: chunk c)
    uint64_t pf_pos = ~0ull;

    for (;;) {
        if (warp == 0) t0_claim(cx, S, X, xguess, pf, pf_pos, last_progress, P, wid, lane);
        bar_sync(1, NT);
        if (S->finish) break;
        const uint32_t nf = S->n_fetch;
        P.phase(0);
        t1_fetch(cx, S, tid);
        bar_sync(1, NT);
        t1_scan(S, tid);
        P.phase(1);
        if (tid == 32) {
            // entry-size statistics of this claim (sizes the next one)
            apus_st_relaxed_sys(&seq->avg_es, (S->cum_es[nf - 1] + nf - 1) / nf);
            apus_st_relaxed_sys(&seq->avg_xb, (S->cum_xb[nf - 1] + nf - 1) / nf);
        }
        bool have_pub_turn = false, have_place_turn = false, aborted = false;
        uint64_t gap_bytes = 0;      // bytes of a wrap gap replicated ahead of the next publish

        while (S->kbase < nf) {
            if (warp == 0) t2_place(cx, S, have_place_turn, P, lane);
            have_place_turn = true;
            bar_sync(1, NT);
            P.phase(2);
            // stop / watchdog while waiting for a turn: this worker holds no valid placement -- it must not hand a turn
            // on, store a byte or publish (a stale placement would overwrite entries that are already acked)
            if (S->abort) { aborted = true; break; }
            if (S->blocked) {   // no space before head: poll again
                if (tid == 0) {
                    // (a stop raises the abort flag here: this worker holds the place turn, the others wait for it)
                    if (apus_ld_relaxed_sys_u32(&hw->stop) || apus_ld_relaxed_sys(&seq->abort_flag)) { apus_st_relaxed_sys(&seq->abort_flag, 1); S->finish = 1; }
                    else if (cx->target != ~0ull && globaltimer_ns() - last_progress > WATCHDOG_NS) {
                        apus_st_relaxed_sys(&hw->error, APUS_KERR_WATCHDOG_LEADER);
                        apus_st_relaxed_sys(&seq->abort_flag, 1); S->finish = 1;
                    }
                }
                if (tid < N) S->ap[tid] = ld_apply(cx, ctrl, hdr, tid);
                bar_sync(1, NT);
                if (S->finish) { aborted = true; break; }
                continue;
            }
            t3_prefill(cx, S, tid);
            bar_sync(1, NT);
            P.phase(3);
            t4_compose(cx, S, warp, lane);
            bar_sync(1, NT);
            P.phase(4);
            t5_store(cx, S, tid);
            bar_sync(1, NT);
            P.phase(5);
            if (S->gap) {
                // nothing is published after a gap: the next sub-tile (at offset 0) carries it
                gap_bytes += S->b - S->a;
                bar_sync(1, NT);
                continue;
            }
            if (warp == 0) t6_publish(cx, S, have_pub_turn, gap_bytes, P, lane);
            have_pub_turn = true;
            gap_bytes = 0;
            last_progress = globaltimer_ns();
            bar_sync(1, NT);
            if (S->abort) { aborted = true; break; }
            if (P.on) { P.phase(6); P.ph[7]++; P.flush(ctrl); }
        }
        if (aborted) break;
    }
    P.flush(ctrl);
    if (tid == 0) { __threadfence(); atomicAdd(reinterpret_cast<unsigned long long *>(&seq->workers_done), 1ull); }
}

// ---------------------------------------------------------------------------------
// FOLLOWER: one function per phase (DESIGN.md §3c), called in order by follower_main
// ---------------------------------------------------------------------------------
struct FollowerAt {           // what the phases address, derived from cx once
    apus_ctrl_t *ctrl, *lctrl;     // my control block, the leader's
    apus_loghdr_t *hdr;
    uint8_t *entries, *lentries;   // my log, the leader's copy of it
    const uint32_t *index;         // the offset index the leader writes next to my log
    apus_hostwords_t *hw;
    uint64_t L;
    uint32_t flags;
    int me;
};
struct FollowerRep {           // the same in every thread: each updates it from the same shared words
    uint64_t old_end;          // walk position (dare_server.c:1795)
    uint64_t acked;            // entries walked (reply byte set) so far
    uint64_t applied;          // apply offset (== commit as far as I hold the entries)
    uint64_t pend_val, pend_end;   // head carried by the last HEAD entry held, and the offset right after it (L: none)
    uint64_t last_progress;
};
struct FollowerPoll {          // warp 0's own
    uint32_t spins;
    bool suspected;
    uint64_t host_applied;     // HOST_APPLY / DEVICE_APPLY: the offset the application has replayed or the device
                               // consumers have read (what the leader may prune behind), as last forwarded
    uint64_t last_hb, last_hb_t;   // the heartbeat word last seen, and when it changed
    uint64_t fbeat;            // my liveness counter in the leader's HBM
    // APUS_FLAG_PROFILE: phase_ns[0] certificates verified, [1] ns from first sight to verified, [2] verify retries
    uint64_t cert_first_cum, cert_first_t;
};

// warp 0, every 256 spins of the poll: stop, watchdog, failure detector, host-apply report, liveness beat.  true: leave
__device__ __forceinline__ bool f_housekeeping(const apus_devctx_t *__restrict__ cx, const FollowerAt &A, const FollowerRep &R, FollowerPoll &W, int lane)
{
    uint32_t stopf = 0;
    uint64_t ha = W.host_applied;
    if (lane == 0) {
        if (apus_ld_relaxed_sys_u32(&A.hw->stop)) stopf = 1;
        else if (cx->target != ~0ull && globaltimer_ns() - R.last_progress > WATCHDOG_NS) {
            apus_st_relaxed_sys(&A.hw->error, APUS_KERR_WATCHDOG_FOLLOWER);
            stopf = 1;
        }
        // failure detector (hb_receive_cb, dare_server.c:866-993): the leader's beats stopped
        if (cx->hb_timeout_ns && !W.suspected && globaltimer_ns() - W.last_hb_t > cx->hb_timeout_ns)
            apus_st_relaxed_sys(&A.hw->leader_suspect, 1 + cx->term);
        if (A.flags & APUS_FLAG_HOST_APPLY) ha = apus_ld_relaxed_sys(&A.hw->host_apply);
        else if (A.flags & APUS_FLAG_DEVICE_APPLY) ha = apus_ld_relaxed_sys(&A.ctrl->cons_cur[0]);
    }
    if (cx->hb_timeout_ns && globaltimer_ns() - W.last_hb_t > cx->hb_timeout_ns) W.suspected = true;
    if (lane == 0) apus_st_relaxed_sys(&A.lctrl->fbeat[A.me], ++W.fbeat);          // I am alive (leader's failure detector)
    stopf = __shfl_sync(0xffffffffu, stopf, 0);
    ha = __shfl_sync(0xffffffffu, ha, 0);
    if ((A.flags & (APUS_FLAG_HOST_APPLY | APUS_FLAG_DEVICE_APPLY)) && ha != W.host_applied) {
        // apply_committed_entries advances `apply` only after do_action (dare_server.c:1939-1962): what this
        // replica reports to the leader's pruning rule is what the HOST has replayed, or what the device consumers
        // have finished reading (the consume work moves its cursor only after its last read of those entries)
        W.host_applied = ha;
        if (lane == 0) { A.hdr->apply = ha; apus_st_relaxed_sys(&A.lctrl->apply_off[A.me], ha); }
    }
    return stopf != 0;
}

// warp 0: poll until there is news -- lane 0 the tail publish {end, entries|term} (one 16 B acquire load), lane 1 its
// certificate half, lane 2 the commit publish {offset, term}, lane 3 the heartbeat word -- then the early ack, and the
// news into S for the whole CTA
__device__ __forceinline__ void f_poll(const apus_devctx_t *__restrict__ cx, const FollowerAt &A, FollowerShared *S, const FollowerRep &R,
                                       FollowerPoll &W, int lane)
{
    TailPub p;
    uint64_t c = 0, cum_seen = 0;
    uint32_t done = 0;
    for (;;) {
        uint64_t x0 = 0, x1 = 0;
        // lanes 4..15 read, SPECULATIVELY and in the same breath, the bytes where the next entry must land (a
        // self-certifying publish names exactly that offset): when its certificate shows up the bytes are already
        // in registers -- verification costs no second trip to memory
        const uint64_t spec_a = (R.old_end == A.L) ? 0 : R.old_end;
        const uint64_t spec_lo = (spec_a & ~15ull) + 16ull * (uint64_t)(lane - 4);
        uint4 spec = make_uint4(0, 0, 0, 0);
        if (lane == 0) apus_ld_acquire_sys_2x64(&A.ctrl->pub_end, x0, x1);
        else if (lane == 1) ld_relaxed_sys_2x64(&A.ctrl->pub_csum, x0, x1);
        else if (lane == 2) ld_relaxed_sys_2x64(A.ctrl->pub_commit, x0, x1);
        else if (lane == 3) x0 = apus_ld_relaxed_sys(&A.ctrl->hb);
        else if (lane < 16 && spec_lo + 16 <= A.L) spec = apus_ld_relaxed_sys_v4(A.entries + spec_lo);
        const uint64_t e = __shfl_sync(0xffffffffu, x0, 0), cumt = __shfl_sync(0xffffffffu, x1, 0);
        const uint64_t csum = __shfl_sync(0xffffffffu, x0, 1), start = __shfl_sync(0xffffffffu, x1, 1);
        p = tail_pub_decode(e, cumt, csum, start, cx->term);
        const uint64_t coff = __shfl_sync(0xffffffffu, x0, 2), cterm = __shfl_sync(0xffffffffu, x1, 2);
        c = commit_pub_offset(coff, cterm, cx->term, R.applied);
        const uint64_t hbw = __shfl_sync(0xffffffffu, x0, 3);
        uint64_t cum = p.cum;
        bool new_entries = cum > R.acked;
        if (new_entries && p.cert && (A.flags & APUS_FLAG_PROFILE) && cum != W.cert_first_cum) { W.cert_first_cum = cum; W.cert_first_t = globaltimer_ns(); }
        if (new_entries && p.cert) {
            // self-certifying publish: the bytes may still be in flight -- read them back from my own HBM until they add
            // up to the certificate
            const bool ok = tail_pub_verify(p, R.old_end, R.acked, A.L, cx->term, A.entries, spec, spec_lo, lane);
            if ((A.flags & APUS_FLAG_PROFILE) && lane == 0) { if (ok) { A.ctrl->phase_ns[0]++; A.ctrl->phase_ns[1] += globaltimer_ns() - W.cert_first_t; } else A.ctrl->phase_ns[2]++; }
            if (!ok) { new_entries = false; cum = R.acked; }   // not there yet (or not verifiable: a fenced publish will follow);
                                                               // nothing of it may be acked or walked
        }
        // commit moved, and I hold entries beyond what I applied
        const bool new_commit = (c != R.applied) && (R.old_end != A.L) && (R.applied != R.old_end);
        if (new_entries || new_commit) { cum_seen = cum; break; }
        // bounded launch: the leader says how many entries exist in total
        uint64_t fe;
        if (cx->target != ~0ull && fin_read(A.ctrl, cx->target, lane, fe) &&
            R.acked >= fe && (R.old_end == A.L || (R.applied == R.old_end && c == R.old_end))) { done = 1; cum_seen = R.acked; break; }
        if (hbw != W.last_hb) { W.last_hb = hbw; W.last_hb_t = globaltimer_ns(); if (lane == 0) apus_st_relaxed_sys(&A.hw->hb_seen, hbw); }
        if ((++W.spins & 0xffu) == 0 && f_housekeeping(cx, A, R, W, lane)) { done = 1; cum_seen = R.acked; break; }
    }
    // early ack: the tail publish was observed with acquire semantics (or its certificate verified), so every
    // entry up to it is resident and visible here (invariant I2); the reply bytes follow behind the ack word
    // unless APUS_F_FENCED_ACK asks for them first
    if (lane == 0) {
        if (!done && !(A.flags & APUS_FLAG_FENCED_ACK) && cum_seen > R.acked) apus_st_relaxed_sys(&A.lctrl->ack[A.me], cum_seen);
        S->end_seen = p.end; S->cum_seen = cum_seen; S->commit_seen = c; S->done = done;
        S->cert = (cum_seen > R.acked) ? p.cert : 0u; S->cert_start = p.start;
    }
}

// all threads, index mode: the entries in (acked, cum_seen] are found through the offset index the leader wrote next to
// the bytes; reply[me] = 1 in my copy and in the leader's (dare_ibv_rc.c:1833-1854)
__device__ __forceinline__ void f_ack_index(const apus_devctx_t *__restrict__ cx, const FollowerAt &A, FollowerShared *S, FollowerRep &R,
                                            uint64_t cum_seen, uint64_t end_seen, int tid, int nthr)
{
    const uint64_t n = cum_seen - R.acked;
    if (tid == 0) S->head_j = 0;
    __syncthreads();
    // FIDX index words per thread are loaded together before any is used: one round trip per FIDX * nthr
    // entries, not per nthr (a batch of a few tiles is thousands of entries)
    constexpr int FIDX = 8;
    for (uint64_t j0 = tid; j0 < n; j0 += (uint64_t)FIDX * nthr) {
        uint32_t w[FIDX];
#pragma unroll
        for (int q = 0; q < FIDX; q++) {
            const uint64_t j = j0 + (uint64_t)q * nthr;
            w[q] = 0;
            // (a self-certified publish names its one entry itself: its index word may still be in flight)
            if (j < n) w[q] = S->cert ? (uint32_t)S->cert_start : apus_ld_relaxed_sys_u32(&A.index[(uint32_t)(R.acked + 1 + j) & cx->idx_mask]);
        }
#pragma unroll
        for (int q = 0; q < FIDX; q++) {
            const uint64_t j = j0 + (uint64_t)q * nthr;
            if (j >= n) break;
            const uint64_t at = (uint64_t)(w[q] & ~APUS_IDX_HEAD_FLAG) + E_REPLY + (uint64_t)A.me;
            st_relaxed_sys_u8(A.entries + at, 1);
            st_relaxed_sys_u8(A.lentries + at, 1);
            if (w[q] & APUS_IDX_HEAD_FLAG) atomicMax(&S->head_j, (uint32_t)(j + 1));
        }
    }
    __syncthreads();
    if (S->head_j) {
        // poll_config_entries (dare_server.c:2163-2170): remember the head this entry carries
        const uint32_t w = apus_ld_relaxed_sys_u32(&A.index[(uint32_t)(R.acked + S->head_j) & cx->idx_mask]);
        const uint64_t off = (uint64_t)(w & ~APUS_IDX_HEAD_FLAG);
        R.pend_val = apus_ld_u64_any(A.entries, off + E_DATA);
        R.pend_end = (off + APUS_HDR_BYTES == A.L) ? 0 : off + APUS_HDR_BYTES;
    }
    R.old_end = end_seen;
}

// all threads, walk mode (APUS_F_FOLLOWER_WALK): parse the new bytes [old_end, end_seen) like the reference follower,
// window by window through shared memory; reply[me] = 1 in my copy and in the leader's (dare_ibv_rc.c:1833-1854)
__device__ __forceinline__ void f_ack_walk(const FollowerAt &A, FollowerShared *S, uint8_t *win, FollowerRep &R,
                                           uint64_t cum_seen, uint64_t end_seen, int tid, int nthr)
{
    uint64_t walked = 0;
    while (R.old_end != end_seen) {
        // window: contiguous bytes from old_end up to end_seen or the end of the ring
        if (tid == 0) {
            uint64_t lo = (R.old_end == A.L) ? 0 : R.old_end;
            if (A.L - lo < APUS_HDR_BYTES) lo = 0;                 // log_get_entry: header does not fit -> 0
            uint64_t hi = (end_seen > lo) ? end_seen : A.L;       // wrapped: first run to the ring's end
            if (lo == end_seen) hi = lo;
            if (hi - (lo & ~15ull) > APUS_FOLLOWER_WIN_BYTES) hi = (lo & ~15ull) + APUS_FOLLOWER_WIN_BYTES;
            S->win_lo = lo; S->win_hi = hi;
        }
        __syncthreads();
        const uint64_t lo = S->win_lo, hi = S->win_hi;
        if (lo == hi) { R.old_end = lo; break; }
        const uint64_t lo16 = lo & ~15ull;
        const uint32_t nch = (uint32_t)(((hi + 15ull) & ~15ull) - lo16) >> 4;
        cta_fetch_chunks(win, A.entries + lo16, nch, tid, nthr);
        __syncthreads();
        // serial walk over headers in shared memory (log_get_entry / log_fit_entry / log_entry_len)
        if (tid == 0) {
            uint64_t off = lo;
            uint32_t n = 0;
            uint64_t next = off;
            bool wrapped = false;
            uint64_t hv = 0, he = A.L;
            while (off < hi) {
                if (A.L - off < APUS_HDR_BYTES) { next = 0; wrapped = true; break; }   // jump to 0
                if (hi - off < APUS_HDR_BYTES) { next = off; break; }                // header not in window yet
                const uint8_t *e = win + (off - lo16);
                const uint32_t ty = e[E_TYPE];
                const uint32_t ln = (uint32_t)e[E_DATA] | ((uint32_t)e[E_DATA + 1] << 8);
                const uint32_t es = apus_entry_stride(ty, ln);
                if (A.L - off < es) { next = 0; wrapped = true; break; }              // ghost: entry continues at 0
                if (off + es > hi) { next = off; break; }                            // entry crosses the window
                if (ty == T_HEAD) {                                                  // poll_config_entries (dare_server.c:2163-2170)
                    hv = le_u64(e + E_DATA);
                    he = (off + es == A.L) ? 0 : off + es;
                }
                S->off[n++] = (uint32_t)(off - lo);
                off += es;
                next = off;
            }
            if (!wrapped && next == A.L) next = 0;      // rule E1 on walker offsets
            S->n = n; S->next = next;
            S->head_val = hv; S->head_end = he;
        }
        __syncthreads();
        const uint32_t n = S->n;
        for (uint32_t k = tid; k < n; k += nthr) {
            const uint64_t at = lo + S->off[k] + E_REPLY + (uint64_t)A.me;
            st_relaxed_sys_u8(A.entries + at, 1);
            st_relaxed_sys_u8(A.lentries + at, 1);
        }
        __syncthreads();
        const uint64_t next = S->next;
        if (n == 0 && next == R.old_end) {
            // no progress possible inside this window: protocol error
            if (tid == 0) apus_st_relaxed_sys(&A.hw->error, APUS_KERR_BAD_ENTRY);
            R.old_end = end_seen;
            break;
        }
        if (S->head_end != A.L) { R.pend_val = S->head_val; R.pend_end = S->head_end; }
        walked += n;
        R.old_end = next;
    }
    if (R.acked + walked != cum_seen && tid == 0) apus_st_relaxed_sys(&A.hw->error, APUS_KERR_COUNT_MISMATCH);
}

// either mode, the batch is persisted: the ack word (APUS_F_FENCED_ACK: only now, behind a fence over the reply bytes),
// then the header and control words
__device__ __forceinline__ void f_persist(const FollowerAt &A, FollowerRep &R, uint64_t cum_seen,
                                          uint64_t end_seen, int tid)
{
    R.acked = cum_seen;
    if (tid == 0) {
        if (A.flags & APUS_FLAG_FENCED_ACK) {
            __threadfence_system();                      // reply bytes before the ack word
            apus_st_relaxed_sys(&A.lctrl->ack[A.me], R.acked);   // the word the leader's quorum ranking polls
        }
        A.hdr->end = end_seen; A.hdr->old_end = R.old_end;
        A.ctrl->acked = R.acked;
        A.ctrl->pend_head_val = R.pend_val; A.ctrl->pend_head_end = R.pend_end;
    }
    R.last_progress = globaltimer_ns();
}

// thread 0, APUS_F_DEVICE_APPLY, a verified self-certifying publish: store the index word of its one entry myself.  The
// leader's store of that word carries no ordering before the publish (it may still be in flight), and device consumers
// find entries through the index.  The value is the leader's, so the order in which the two stores land does not
// matter; this one precedes the consumer record (cons_publish, same thread) in program order.
__device__ __forceinline__ void f_cert_index(const apus_devctx_t *__restrict__ cx, const FollowerAt &A, const FollowerRep &R,
                                             uint64_t cert_start)
{
    const_cast<uint32_t *>(A.index)[(uint32_t)(R.acked + 1) & cx->idx_mask] = (uint32_t)cert_start;
}

// all threads: follow the commit offset (invariant I4: never beyond what I hold), and adopt the head of a committed
// HEAD entry
__device__ __forceinline__ void f_follow_commit(const FollowerAt &A, FollowerRep &R, uint64_t commit_seen, int tid)
{
    if (R.old_end == A.L || R.applied == R.old_end || commit_seen == R.applied) return;
    const uint64_t from = R.applied;
    const uint64_t held = apus_ring_dist(from, R.old_end, A.L);          // bytes I hold beyond `applied`
    uint64_t want = apus_ring_dist(from, commit_seen, A.L);
    uint64_t to = commit_seen;
    if (want > held) { want = held; to = R.old_end; }             // the leader clamps the same way (dare_ibv_rc.c:1783-1787)
    if (!want) return;
    if (R.pend_end != A.L) {
        const uint64_t dh = apus_ring_dist(from, R.pend_end, A.L);
        if (dh > 0 && dh <= want) {
            // the HEAD entry is committed: adopt the head it carries (dare_server.c:2166-2169, 2182-2186)
            if (tid == 0) { A.hdr->head = R.pend_val; A.ctrl->pend_head_end = A.L; }
            R.pend_end = A.L;
        }
    }
    R.applied = to;
    if (tid == 0) {
        A.hdr->commit = R.applied;              // what this replica knows committed AND holds (I4)
        if (!(A.flags & (APUS_FLAG_HOST_APPLY | APUS_FLAG_DEVICE_APPLY))) {
            A.hdr->apply = R.applied;           // library use: nothing replays the log on the host
            apus_st_relaxed_sys(&A.lctrl->apply_off[A.me], R.applied);
        }
        if (A.flags & APUS_FLAG_DEVICE_APPLY) cons_publish(A.ctrl, R.applied, R.acked);
        // the host may replay [its apply, applied): everything before `applied` is committed and held here
        apus_st_relaxed_sys_2x64(&A.hw->commit_off, R.applied, R.acked);
    }
    R.last_progress = globaltimer_ns();
}

__device__ void follower_main(const apus_devctx_t *__restrict__ cx)
{
    FollowerShared *S = reinterpret_cast<FollowerShared *>(smem_raw);
    uint8_t *win = smem_raw + FS_BYTES;
    const int tid = threadIdx.x, nthr = blockDim.x;
    apus_ctrl_t *ctrl = reinterpret_cast<apus_ctrl_t *>(cx->region);
    apus_loghdr_t *hdr = reinterpret_cast<apus_loghdr_t *>(cx->region + APUS_HDR_OFF);
    const FollowerAt A = {ctrl, reinterpret_cast<apus_ctrl_t *>(cx->peer[cx->leader_idx]), hdr,
                          cx->region + cx->entries_off, cx->peer[cx->leader_idx] + cx->entries_off,
                          reinterpret_cast<const uint32_t *>(cx->region + APUS_INDEX_OFF), cx->hw, cx->log_len, cx->flags, cx->idx};
    FollowerRep R = {hdr->old_end, ctrl->acked, hdr->apply, ctrl->pend_head_val, ctrl->pend_head_end, globaltimer_ns()};
    FollowerPoll W = {0, false, hdr->apply, apus_ld_relaxed_sys(&ctrl->hb), globaltimer_ns(), globaltimer_ns() >> 8, 0, 0};

    for (;;) {
        if (tid < 32) f_poll(cx, A, S, R, W, tid);
        __syncthreads();
        if (S->done) break;
        const uint64_t end_seen = S->end_seen, cum_seen = S->cum_seen, commit_seen = S->commit_seen;
        if (cum_seen > R.acked) {
            if (A.flags & APUS_FLAG_WALK) f_ack_walk(A, S, win, R, cum_seen, end_seen, tid, nthr);
            else f_ack_index(cx, A, S, R, cum_seen, end_seen, tid, nthr);
            if ((A.flags & APUS_FLAG_DEVICE_APPLY) && S->cert && tid == 0) f_cert_index(cx, A, R, S->cert_start);
            f_persist(A, R, cum_seen, end_seen, tid);
        }
        f_follow_commit(A, R, commit_seen, tid);
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------
extern "C" __global__ void __launch_bounds__(APUS_KERNEL_THREADS, 1)
apus_replica_kernel(const apus_role_t *__restrict__ roles)
{
    const apus_role_t r = roles[blockIdx.x];
    if (r.kind == APUS_ROLE_LEADER) leader_main(r.ctx, r.worker);
    else if (r.kind == APUS_ROLE_FOLLOWER) follower_main(r.ctx);
}

extern "C" size_t apus_kernel_smem_bytes(void)
{
    size_t a = L_TOTAL, b = F_TOTAL;
    return a > b ? a : b;
}

/* load the replica kernel on the current device and set its shared-memory size, once per device.  Under lazy module
 * loading the first launch would load it, and a load may wait for the kernels running on the device: a resident
 * consumer (apus_consumer_attach) never ends by itself, so attach loads it first. */
extern "C" cudaError_t apus_kernels_load(void)
{
    static bool attr_set[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 64 && !attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(apus_replica_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)apus_kernel_smem_bytes());
        if (e != cudaSuccess) return e;
        attr_set[dev] = true;
    }
    return cudaSuccess;
}

extern "C" cudaError_t apus_launch_roles(const apus_role_t *d_roles, int n_roles, cudaStream_t stream)
{
    cudaError_t e = apus_kernels_load();
    if (e != cudaSuccess) return e;
    apus_replica_kernel<<<n_roles, APUS_KERNEL_THREADS, apus_kernel_smem_bytes(), stream>>>(d_roles);
    return cudaGetLastError();
}
