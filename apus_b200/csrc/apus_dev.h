/*
 * apus_dev.h -- device helpers shared by the persistent replica kernel (apus_kernels.cu) and the stream-ordered batch
 * kernels (apus_batch.cu): system-scope loads and stores, the entry format, and the consumer record that the follower
 * kernel writes and the consume kernels read.  Everything here is __device__ __forceinline__, so each translation unit
 * inlines its own copy and no relocatable device code is needed.  What a consumer reads with -- the loads, the entry
 * tests, the record's acquire, the cursor rule and the back-off -- is the public include/apus_consumer.cuh, which
 * applications' resident consumers compile too: one definition for both paths.
 */
#ifndef APUS_DEV_H
#define APUS_DEV_H

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "apus_layout.h"
#include "apus_consumer.cuh"

static_assert(APUS_ENT_IDX == E_IDX && APUS_ENT_TERM == E_TERM && APUS_ENT_REQID == E_REQID && APUS_ENT_CLTID == E_CLTID &&
              APUS_ENT_TYPE == E_TYPE && APUS_ENT_DATA == E_DATA && APUS_ENT_CMD == E_CMD &&
              APUS_INDEX_HEAD_BIT == APUS_IDX_HEAD_FLAG && APUS_ENTRY_HDR == APUS_HDR_BYTES,
              "the public consumer header describes the entry format the kernels write");
static_assert(APUS_NOOP == T_NOOP && APUS_CONFIG == T_CONFIG && APUS_HEAD == T_HEAD, "entry types");

// ---------------------------------------------------------------------------------
// memory-model helpers (system scope: peers and the host observe these)
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t ld_acquire_sys(const volatile void *p)
{
    uint64_t v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void ld_relaxed_sys_2x64(const volatile void *p, uint64_t &a, uint64_t &b)
{
    asm volatile("ld.relaxed.sys.global.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_u8(volatile void *p, uint8_t v)
{
    asm volatile("st.relaxed.sys.global.u8 [%0], %1;" ::"l"(p), "r"((uint32_t)v) : "memory");
}

// ---------------------------------------------------------------------------------
// entry format
// ---------------------------------------------------------------------------------
// bytes placed at entry+48 (sm_cmd_t image {u16 len; cmd}, dare_cid_t, or head offset)
__device__ __forceinline__ uint32_t data_bytes(uint32_t type, uint32_t len)
{
    if (type == T_NOOP) return 0;
    if (type == T_CONFIG) return 16;
    if (type == T_HEAD) return 8;
    return 2u + len;
}

// ---------------------------------------------------------------------------------
// The consumer record {committed-and-held offset, entries held} in my own control block (APUS_F_DEVICE_APPLY): the
// bound apus_consume_device's work trusts.  Writer: the follower's thread 0, once per commit advance.  That thread read
// the tail publish with ld.acquire.sys, which the leader stored on another GPU behind a fence.sc.sys over the entry
// bytes and index words (or it verified a certificate and stored the entry's index word itself, f_cert_index).  A
// release is cumulative: everything thread 0 has observed is ordered before the record for whoever acquires it.  The
// scope is .sys, not .gpu, so that the chain stays at the scope it started at (the writes came from a peer GPU); it
// costs one store per commit advance.  Readers, with ld.acquire.sys (apus_cons_read): the consume work's first kernel
// on the same GPU, the kernels that read the entries running after it in stream order; or a resident consumer's
// polling thread, whose CTA barrier hands the acquire to the threads that read the entries.
// On a leader (APUS_F_APPLY_ANY_ROLE) the writer is the commit warp's lane 0, once per commit advance, and every write
// the record covers was made on the leader's own GPU: the entry bytes and index words by its worker CTAs, each tile's
// behind a fence in the lane that stores its publish record's PR_END pair (t6_publish after its CTA barrier, the
// express path after a __syncwarp), so that pair is a release of the tile's stores.  The commit warp finds records with
// relaxed loads in several lanes, so before the record lane 0 re-reads the PR_END pair of EVERY record the advance
// commits with ld.acquire.gpu: each read synchronises with its own writer's fence, whatever order the workers took
// their turns in.  Then it stores the record with st.release.gpu (cons_publish_gpu), cumulative over all of them.  GPU
// scope is enough, since the writers, the bytes and the consume kernels are all on this GPU.
// ---------------------------------------------------------------------------------
static_assert(offsetof(apus_ctrl_t, cons_rec) == 896 && sizeof(apus_ctrl_t) == APUS_CTL_OFF,
              "the consumer words use the spare line after turn_ns and end where the control-plane words start");
static_assert(offsetof(apus_ctrl_t, cons_rec) % 16 == 0 && offsetof(apus_ctrl_t, cons_cur) % 16 == 0,
              "the consumer record and the cursor are 16 B words");
__device__ __forceinline__ void cons_publish(apus_ctrl_t *ctrl, uint64_t held_off, uint64_t held_entries)
{
    asm volatile("st.release.sys.global.v2.u64 [%0], {%1,%2};" ::"l"(ctrl->cons_rec), "l"(held_off), "l"(held_entries)
                 : "memory");
}
__device__ __forceinline__ void cons_publish_gpu(apus_ctrl_t *ctrl, uint64_t held_off, uint64_t held_entries)
{
    asm volatile("st.release.gpu.global.v2.u64 [%0], {%1,%2};" ::"l"(ctrl->cons_rec), "l"(held_off), "l"(held_entries)
                 : "memory");
}

#endif /* APUS_DEV_H */
