/*
 * apus_dev.h -- device helpers shared by the persistent replica kernel (apus_kernels.cu) and the stream-ordered batch
 * kernels (apus_batch.cu): system-scope loads and stores, the entry format, and the consumer record that the follower
 * kernel writes and the consume kernels read.  Everything here is __device__ __forceinline__, so each translation unit
 * inlines its own copy and no relocatable device code is needed.
 */
#ifndef APUS_DEV_H
#define APUS_DEV_H

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "apus_layout.h"

// ---------------------------------------------------------------------------------
// memory-model helpers (system scope: peers and the host observe these)
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t ld_relaxed_sys(const volatile void *p)
{
    uint64_t v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t ld_acquire_sys(const volatile void *p)
{
    uint64_t v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys_u32(const volatile void *p)
{
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void ld_acquire_sys_2x64(const volatile void *p, uint64_t &a, uint64_t &b)
{
    // an acquire LOAD is far cheaper than a system fence (tools/ubench measures both)
    asm volatile("ld.acquire.sys.global.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void ld_relaxed_sys_2x64(const volatile void *p, uint64_t &a, uint64_t &b)
{
    asm volatile("ld.relaxed.sys.global.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys(volatile void *p, uint64_t v)
{
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_2x64(volatile void *p, uint64_t a, uint64_t b)
{
    asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_u8(volatile void *p, uint8_t v)
{
    asm volatile("st.relaxed.sys.global.u8 [%0], %1;" ::"l"(p), "r"((uint32_t)v) : "memory");
}
__device__ __forceinline__ uint4 ld_relaxed_sys_v4(const void *p)
{
    uint4 v;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ void st_v4(void *p, uint4 v)
{
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}
__device__ __forceinline__ void st_u8(void *p, uint32_t v)
{
    asm volatile("st.global.u8 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---------------------------------------------------------------------------------
// entry format
// ---------------------------------------------------------------------------------
__device__ __forceinline__ bool has_cmd(uint32_t type)
{
    return !(type == T_NOOP || type == T_CONFIG || type == T_HEAD);
}
// bytes placed at entry+48 (sm_cmd_t image {u16 len; cmd}, dare_cid_t, or head offset)
__device__ __forceinline__ uint32_t data_bytes(uint32_t type, uint32_t len)
{
    if (type == T_NOOP) return 0;
    if (type == T_CONFIG) return 16;
    if (type == T_HEAD) return 8;
    return 2u + len;
}
__device__ __forceinline__ uint32_t entry_stride(uint32_t type, uint32_t len)
{
    return has_cmd(type) ? APUS_HDR_BYTES + len : APUS_HDR_BYTES;   // dare_log.h:228-234
}
__device__ __forceinline__ uint64_t ring_dist(uint64_t from, uint64_t to, uint64_t L)
{
    return to >= from ? to - from : L - (from - to);
}
// the u64 at log offset `at` of any alignment, with system-scope relaxed loads: one 8 B load, or eight byte reads out of
// 4 B-aligned words
__device__ __forceinline__ uint64_t ld_relaxed_sys_u64_any(const uint8_t *entries, uint64_t at)
{
    uint64_t v = ld_relaxed_sys(entries + (at & ~7ull));
    if (at & 7ull) {
        v = 0;
        for (int q = 7; q >= 0; q--) v = (v << 8) | (uint64_t)(ld_relaxed_sys_u32(entries + ((at + q) & ~3ull)) >> (8 * ((at + q) & 3ull)) & 0xffu);
    }
    return v;
}

// ---------------------------------------------------------------------------------
// The consumer record {committed-and-held offset, entries held} in my own control block (APUS_F_DEVICE_APPLY): the
// bound apus_consume_device's work trusts.  Writer: the follower's thread 0, once per commit advance.  That thread read
// the tail publish with ld.acquire.sys, which the leader stored on another GPU behind a fence.sc.sys over the entry
// bytes and index words (or it verified a certificate and stored the entry's index word itself, f_cert_index).  A
// release is cumulative: everything thread 0 has observed is ordered before the record for whoever acquires it.  The
// scope is .sys, not .gpu, so that the chain stays at the scope it started at (the writes came from a peer GPU); it
// costs one store per commit advance.  Reader: the consume work's first kernel on the same GPU, with ld.acquire.sys;
// the kernels that read the entries run after it in stream order.
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
__device__ __forceinline__ void cons_read(const apus_ctrl_t *ctrl, uint64_t &held_off, uint64_t &held_entries)
{
    ld_acquire_sys_2x64(ctrl->cons_rec, held_off, held_entries);
}
// committed entries past the consumers' cursor: the record holds entries 1 .. held_entries, the cursor stands at idx
// next_idx.  What a consume call may examine (apus_consume_head_kernel) and what a consume wait waits for
// (apus_consume_wait_kernel): one definition, so that a ready wait and the consume after it agree.
__device__ __forceinline__ uint64_t cons_avail(uint64_t held_entries, uint64_t next_idx)
{
    return held_entries + 1 > next_idx ? held_entries + 1 - next_idx : 0;
}

#endif /* APUS_DEV_H */
