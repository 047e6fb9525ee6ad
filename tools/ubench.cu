// tools/ubench.cu -- latency micro-benchmarks that size the replication protocol:
// how long a system-scope fence, a poll on local/peer/host memory and a flag
// ping-pong take on this machine (the o/L/G idea of the reference's LogGP probes,
// dare_ibv_rc.c:3323-3702, applied to NVLink/PCIe).  Build: make -C tools
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>
#include <algorithm>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__device__ __forceinline__ uint64_t gt() { uint64_t t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ uint64_t ldr(const volatile void *p) { uint64_t v; asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void str(volatile void *p, uint64_t v) { asm volatile("st.relaxed.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void st16(void *p, uint4 v) { asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory"); }

// mode 0: dependent loads (poll latency); 1: fence only; 2: warp stores 512 B then fence; 3: store 8 B + fence
__global__ void k_single(volatile uint64_t *target, uint8_t *buf, int mode, int iters, uint64_t *out_ns, long long *out_clk)
{
    uint64_t acc = 0;
    long long c0 = clock64();
    uint64_t t0 = gt();
    for (int i = 0; i < iters; i++) {
        if (mode == 0) { acc += ldr(target + (acc & 1)); }
        else if (mode == 1) { __threadfence_system(); }
        else if (mode == 2) { st16(buf + ((i & 63) * 512) + threadIdx.x * 16, make_uint4(i, i, i, i)); __threadfence_system(); }
        else if (mode == 3) { if (threadIdx.x == 0) str((volatile uint64_t *)buf + (i & 63) * 16, i); __threadfence_system(); }
        else if (mode == 4) { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
        else if (mode == 5) { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
        else if (mode == 6) { asm volatile("fence.sc.gpu;" ::: "memory"); }
        else if (mode == 7) { st16(buf + ((i & 63) * 512) + threadIdx.x * 16, make_uint4(i, i, i, i)); asm volatile("fence.acq_rel.sys;" ::: "memory"); }
        else if (mode == 8) { st16(buf + ((i & 63) * 512) + threadIdx.x * 16, make_uint4(i, i, i, i)); if (threadIdx.x == 0) asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(target + 8), "l"((uint64_t)i) : "memory"); }
        else if (mode == 9) { uint64_t v; asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(target + (acc & 1)) : "memory"); acc += v; }
        else if (mode == 10) { st16(buf + ((i & 63) * 512) + threadIdx.x * 16, make_uint4(i, i, i, i)); asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
        else if (mode == 11) { st16(buf + ((i & 63) * 512) + threadIdx.x * 16, make_uint4(i, i, i, i)); if (threadIdx.x == 0) asm volatile("red.release.sys.global.add.u64 [%0], %1;" :: "l"(target + 8), "l"((uint64_t)1) : "memory"); }
        else if (mode == 13) { acc += gt(); }
        else if (mode == 14) { acc += clock64(); }
        else if (mode == 12) { st16(buf + ((i & 63) * 512) + threadIdx.x * 16, make_uint4(i, i, i, i)); }
        else if (mode == 15 && threadIdx.x == 0) {
            const uint64_t o = atomicCAS((unsigned long long *)target, acc, acc + 1);
            acc = o == acc ? acc + 1 : o;
        }
    }
    uint64_t t1 = gt();
    long long c1 = clock64();
    if (threadIdx.x == 0) { out_ns[0] = t1 - t0 + (acc == 0xdeadbeef); out_clk[0] = c1 - c0; }
}

// ping-pong: block A writes flagB=i (optionally after data stores + fence), waits flagA==i
__global__ void k_ping(volatile uint64_t *my_flag, volatile uint64_t *peer_flag, uint8_t *peer_buf, int iters, int data_bytes, int fence, int first, uint64_t *out_ns)
{
    uint64_t t0 = gt();
    for (int i = 1; i <= iters; i++) {
        if (first) {
            if (data_bytes) { for (int b = threadIdx.x * 16; b < data_bytes; b += blockDim.x * 16) st16(peer_buf + b, make_uint4(i, i, i, i)); __syncthreads(); }
            if (threadIdx.x == 0) {
                if (fence == 1) __threadfence_system();
                if (fence == 2) asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(peer_flag), "l"((uint64_t)i) : "memory");
                else if (fence == 3) { asm volatile("fence.acq_rel.sys;" ::: "memory"); str(peer_flag, i); }
                else str(peer_flag, i);
                while (ldr(my_flag) < (uint64_t)i) ;
            }
            __syncthreads();
        } else {
            if (threadIdx.x == 0) { while (ldr(my_flag) < (uint64_t)i) ; if (fence == 1) __threadfence_system(); str(peer_flag, i); }
            __syncthreads();
        }
    }
    uint64_t t1 = gt();
    if (threadIdx.x == 0) out_ns[0] = t1 - t0;
}


// self-certifying replication experiment (round-2 design, DESIGN.md section 7): the writer stores a 128 B entry with
// eight relaxed 16 B stores and then a certificate word {seq, checksum} with a relaxed 8 B store -- NO fence between
// them.  The reader polls the certificate, loads the entry, recomputes the checksum and retries until it matches
// (a torn read = data still in flight), then acks.  Reports the round trip and how many torn reads were seen.
__device__ __forceinline__ uint32_t mix4(uint4 v) { return (v.x * 0x9E3779B1u) ^ (v.y * 0x85EBCA77u) ^ (v.z * 0xC2B2AE3Du) ^ (v.w * 0x27D4EB2Fu); }
__device__ __forceinline__ uint4 ld16(const uint8_t *p) { uint4 v; asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory"); return v; }
__global__ void k_selfcert(volatile uint64_t *my_flag, volatile uint64_t *peer_cert, uint8_t *peer_ring, volatile uint64_t *my_cert, uint8_t *my_ring,
                           volatile uint64_t *peer_flag, int iters, int writer, uint64_t *out)
{
    const int lane = threadIdx.x & 31;
    uint64_t t0 = gt(), torn = 0;
    for (int i = 1; i <= iters; i++) {
        uint8_t *slot_w = peer_ring + (size_t)(i & 255) * 128, *slot_r = my_ring + (size_t)(i & 255) * 128;
        if (writer) {
            uint4 v = make_uint4(i * 7 + lane, i ^ (lane << 8), i + 0x1234567, lane * 0x01010101u + i);
            uint32_t h = lane < 8 ? mix4(v) : 0;
            if (lane < 8) st16(slot_w + lane * 16, v);
            for (int s = 4; s > 0; s >>= 1) h ^= __shfl_xor_sync(0xffffffffu, h, s);
            if (lane == 0) {
                str(peer_cert, ((uint64_t)h << 32) | (uint32_t)i);           // relaxed, no fence
                while (ldr(my_flag) < (uint64_t)i) ;
            }
            __syncwarp();
        } else {
            uint64_t c;
            do { c = ldr(my_cert); } while ((uint32_t)c != (uint32_t)i);
            for (;;) {
                uint4 v = lane < 8 ? ld16(slot_r + lane * 16) : make_uint4(0, 0, 0, 0);
                uint32_t h = lane < 8 ? mix4(v) : 0;
                for (int s = 4; s > 0; s >>= 1) h ^= __shfl_xor_sync(0xffffffffu, h, s);
                h = __shfl_sync(0xffffffffu, h, 0);
                if (h == (uint32_t)(c >> 32)) break;
                torn++;
            }
            if (lane == 0) str(peer_flag, i);
            __syncwarp();
        }
    }
    uint64_t t1 = gt();
    if (threadIdx.x == 0) { out[0] = t1 - t0; out[1] = torn; }
}

// interference: CTA 0 measures dependent-load latency while CTAs 1..n hammer fences / stores
__global__ void k_interfere(volatile uint64_t *target, uint8_t *buf, int mode, int iters, uint64_t *out_ns, volatile int *stop)
{
    if (blockIdx.x == 0) {
        uint64_t acc = 0;
        uint64_t t0 = gt();
        for (int i = 0; i < iters; i++) acc += ldr(target + (acc & 1));
        uint64_t t1 = gt();
        if (threadIdx.x == 0) { out_ns[0] = t1 - t0 + (acc == 0xdeadbeef); *stop = 1; }
    } else {
        int i = 0;
        while (!*stop) {
            i++;
            if (mode == 1) __threadfence_system();
            else if (mode == 2) asm volatile("fence.acq_rel.gpu;" ::: "memory");
            else if (mode == 3) { st16(buf + blockIdx.x * 65536 + ((i & 63) * 512) + threadIdx.x * 16, make_uint4(i, i, i, i)); }
            else if (mode == 4) { st16(buf + blockIdx.x * 65536 + ((i & 63) * 512) + threadIdx.x * 16, make_uint4(i, i, i, i)); if ((i & 15) == 0) __threadfence_system(); }
            else if (mode == 5) { uint64_t v; asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(target + 16) : "memory"); if (v == 12345) break; }
        }
    }
}

// claim counter (the leader's T0, DESIGN.md §3a): k CTAs take claims of `step` slots from one counter until `total`
// slots are claimed.  w[0] = counter, w[16] = doorbell (== total), w[32..33] = claim-sizing words, each on its own line.
// proto 0: load counter + doorbell, re-read the doorbell with acquire, load the sizing words, then the compare-and-swap;
//          a lost compare-and-swap starts over.
// proto 1: the sequence of t0_claim: counter, doorbell (relaxed) and sizing words in one round trip, then the
//          compare-and-swap with an acquire re-read of the doorbell issued beside it; a lost compare-and-swap is retried
//          at once from the value it returned (each retry again with its acquire).
__global__ void k_claim(uint64_t *w, int proto, uint64_t total, uint64_t step, uint64_t *out)
{
    if (threadIdx.x != 0) return;
    unsigned long long *ctr = (unsigned long long *)w;
    uint64_t won = 0, tries = 0;
    const uint64_t t0 = gt();
    for (;;) {
        uint64_t c, t, a, b;
        if (proto == 0) {
            t = ldr(w + 16); c = ldr(w);
            if (t > c) asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(t) : "l"(w + 16) : "memory");
            if (c >= total) break;
            a = ldr(w + 32); b = ldr(w + 33);
            const uint64_t nn = step + ((a + b) & 1);   // (a, b are 0: the sizing loads are a dependency, as in T0)
            tries++;
            if (atomicCAS(ctr, c, c + nn) == c) won++;
        } else {
            c = ldr(w); t = ldr(w + 16); a = ldr(w + 32); b = ldr(w + 33);
            const uint64_t nn = step + ((a + b) & 1);
            while (c < t && c < total) {
                tries++;
                const uint64_t was = atomicCAS(ctr, c, c + nn);
                uint64_t ta;
                asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(ta) : "l"(w + 16) : "memory");
                if (was == c) { won++; break; }
                c = was;
            }
            if (c >= total) break;
        }
    }
    const uint64_t t1 = gt();
    atomicAdd((unsigned long long *)out, (unsigned long long)won);
    atomicAdd((unsigned long long *)out + 1, (unsigned long long)tries);
    atomicMax((unsigned long long *)out + 2, (unsigned long long)(t1 - t0));
}

static void run_claim(uint64_t *dflag, int proto, int k)
{
    const uint64_t total = 1ull << 20, step = 256;
    uint64_t *o; CK(cudaMallocManaged(&o, 64));
    for (int rep = 0; rep < 2; rep++) {                     // first launch warms up
        CK(cudaMemset(dflag, 0, 4096)); memset(o, 0, 64);
        CK(cudaMemcpy(dflag + 16, &total, 8, cudaMemcpyHostToDevice));
        k_claim<<<k, 32>>>(dflag, proto, total, step, o); CK(cudaDeviceSynchronize());
    }
    printf("claims, %2d CTAs, %s: %.2f claims/us, %.2f compare-and-swaps per claim\n", k,
           proto == 0 ? "load/acquire/load/CAS, restart on loss" : "one load round, CAS + acquire, retry from returned value",
           (double)o[0] * 1000.0 / (double)o[2], (double)o[1] / (double)o[0]);
    cudaFree(o);
}

static void run_interfere(volatile uint64_t *target, uint8_t *buf, const char *name, int mode, int nblk)
{
    uint64_t *ns; int *stop;
    CK(cudaMallocManaged(&ns, 8)); CK(cudaMallocManaged(&stop, 4));
    *stop = 0;
    k_interfere<<<nblk, 32>>>(target, buf, mode, 20000, ns, stop); CK(cudaDeviceSynchronize());
    printf("poll local L2 while %d other CTAs %s: %.1f ns\n", nblk - 1, name, (double)ns[0] / 20000);
    cudaFree(ns); cudaFree(stop);
}

static double run_single(volatile uint64_t *target, uint8_t *buf, int mode, int iters, int threads)
{
    uint64_t *ns; long long *clk;
    CK(cudaMallocManaged(&ns, 8)); CK(cudaMallocManaged(&clk, 8));
    k_single<<<1, threads>>>(target, buf, mode, 10, ns, clk); CK(cudaDeviceSynchronize());
    k_single<<<1, threads>>>(target, buf, mode, iters, ns, clk); CK(cudaDeviceSynchronize());
    double r = (double)ns[0] / iters;
    printf("    (%.0f clk/iter)\n", (double)clk[0] / iters);
    cudaFree(ns); cudaFree(clk);
    return r;
}

int main()
{
    int ndev = 0; CK(cudaGetDeviceCount(&ndev));
    printf("devices: %d\n", ndev);
    CK(cudaSetDevice(0));
    uint64_t *dflag; uint8_t *dbuf; CK(cudaMalloc(&dflag, 4096)); CK(cudaMemset(dflag, 0, 4096)); CK(cudaMalloc(&dbuf, 1 << 20));
    uint64_t *hflag; CK(cudaHostAlloc(&hflag, 4096, cudaHostAllocMapped)); hflag[0] = 0; hflag[1] = 0;
    uint64_t *hflag_d; CK(cudaHostGetDevicePointer(&hflag_d, hflag, 0));
    printf("poll local L2 (dependent ld.relaxed.sys): "); printf("%.1f ns\n", run_single(dflag, dbuf, 0, 20000, 32));
    printf("poll host-mapped (dependent ld.relaxed.sys over PCIe): "); printf("%.1f ns\n", run_single(hflag_d, dbuf, 0, 5000, 32));
    printf("fence.sys, nothing outstanding: "); printf("%.1f ns\n", run_single(dflag, dbuf, 1, 20000, 32));
    printf("warp 512 B local stores + fence.sys: "); printf("%.1f ns\n", run_single(dflag, dbuf, 2, 20000, 32));
    printf("8 B local store + fence.sys: "); printf("%.1f ns\n", run_single(dflag, dbuf, 3, 20000, 32));
    printf("8 B host-mapped store + fence.sys: "); printf("%.1f ns\n", run_single(dflag, (uint8_t *)hflag_d + 1024, 3, 5000, 32));
    printf("fence.acq_rel.sys, nothing outstanding: "); printf("%.1f ns\n", run_single(dflag, dbuf, 4, 20000, 32));
    printf("fence.acq_rel.gpu, nothing outstanding: "); printf("%.1f ns\n", run_single(dflag, dbuf, 5, 20000, 32));
    printf("fence.sc.gpu, nothing outstanding: "); printf("%.1f ns\n", run_single(dflag, dbuf, 6, 20000, 32));
    printf("warp 512 B local stores + fence.acq_rel.sys: "); printf("%.1f ns\n", run_single(dflag, dbuf, 7, 20000, 32));
    printf("warp 512 B local stores + st.release.sys flag: "); printf("%.1f ns\n", run_single(dflag, dbuf, 8, 20000, 32));
    printf("ld.acquire.sys local (dependent): "); printf("%.1f ns\n", run_single(dflag, dbuf, 9, 20000, 32));
    printf("warp 512 B local stores + fence.acq_rel.gpu: "); printf("%.1f ns\n", run_single(dflag, dbuf, 10, 20000, 32));
    printf("warp 512 B local stores + red.release.sys: "); printf("%.1f ns\n", run_single(dflag, dbuf, 11, 20000, 32));
    printf("read %%globaltimer: "); printf("%.1f ns\n", run_single(dflag, dbuf, 13, 20000, 32));
    printf("read clock64: "); printf("%.1f ns\n", run_single(dflag, dbuf, 14, 20000, 32));
    printf("warp 512 B local stores only (issue rate): "); printf("%.1f ns\n", run_single(dflag, dbuf, 12, 20000, 32));
    CK(cudaMemset(dflag, 0, 4096));
    printf("atomicCAS local L2 (dependent chain): "); printf("%.1f ns\n", run_single(dflag, dbuf, 15, 20000, 32));
    CK(cudaMemset(dflag, 0, 4096));
    for (int proto = 0; proto < 2; proto++)
        for (int k = 1; k <= 16; k *= 4) run_claim(dflag, proto, k);
    CK(cudaMemset(dflag, 0, 4096));
    run_interfere(dflag, dbuf, "do nothing", 0, 1);
    run_interfere(dflag, dbuf, "loop fence.sc.sys", 1, 2);
    run_interfere(dflag, dbuf, "loop fence.sc.sys", 1, 8);
    run_interfere(dflag, dbuf, "loop fence.acq_rel.gpu", 2, 8);
    run_interfere(dflag, dbuf, "stream 512 B stores", 3, 8);
    run_interfere(dflag, dbuf, "stream stores + fence.sys every 16", 4, 8);
    run_interfere(dflag, dbuf, "spin ld.acquire.gpu on a neighbour line", 5, 8);
    // same-GPU ping-pong between two CTAs
    for (int cfg = 0; cfg < 5; cfg++) {
        int data = cfg == 0 ? 0 : (cfg == 1 ? 128 : (cfg == 2 ? 32768 : 128)), fence = cfg == 0 ? 0 : (cfg <= 2 ? 1 : (cfg == 3 ? 2 : 3));
        CK(cudaMemset(dflag, 0, 4096));
        uint64_t *ns; CK(cudaMallocManaged(&ns, 16));
        cudaStream_t s1, s2; CK(cudaStreamCreateWithFlags(&s1, cudaStreamNonBlocking)); CK(cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking));
        int iters = 20000;
        k_ping<<<1, 256, 0, s1>>>(dflag, dflag + 64, dbuf, iters, data, fence, 1, ns);
        k_ping<<<1, 256, 0, s2>>>(dflag + 64, dflag, dbuf, iters, 0, fence, 0, ns + 1);
        CK(cudaDeviceSynchronize());
        printf("same-GPU ping-pong, %d B data, fence=%d: %.1f ns round trip\n", data, fence, (double)ns[0] / iters);
        cudaFree(ns);
    }
    {   // self-certifying writes, two CTAs of one GPU
        uint8_t *ring; uint64_t *w; CK(cudaMalloc(&ring, 256 * 128)); CK(cudaMalloc(&w, 4096)); CK(cudaMemset(w, 0, 4096)); CK(cudaMemset(ring, 0, 256 * 128));
        uint64_t *o; CK(cudaMallocManaged(&o, 64)); memset(o, 0, 64);
        cudaStream_t s1, s2; CK(cudaStreamCreateWithFlags(&s1, cudaStreamNonBlocking)); CK(cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking));
        int iters = 20000;
        // w[0] = writer's ack flag, w[64] = certificate word (reader side)
        k_selfcert<<<1, 32, 0, s1>>>(w, w + 64, ring, nullptr, nullptr, nullptr, iters, 1, o);
        k_selfcert<<<1, 32, 0, s2>>>(nullptr, nullptr, nullptr, w + 64, ring, w, iters, 0, o + 2);
        CK(cudaDeviceSynchronize());
        printf("same-GPU self-certifying 128 B entry (no fence): %.1f ns round trip, %llu torn reads in %d\n", (double)o[0] / iters, (unsigned long long)o[3], iters);
    }
    if (ndev >= 2) {
        int can = 0; CK(cudaDeviceCanAccessPeer(&can, 0, 1));
        printf("peer access 0->1: %d\n", can);
        if (can) {
            CK(cudaDeviceEnablePeerAccess(1, 0));
            CK(cudaSetDevice(1)); CK(cudaDeviceEnablePeerAccess(0, 0));
            uint64_t *pflag; uint8_t *pbuf; CK(cudaMalloc(&pflag, 4096)); CK(cudaMemset(pflag, 0, 4096)); CK(cudaMalloc(&pbuf, 1 << 20));
            CK(cudaSetDevice(0));
            printf("poll PEER memory over NVLink (dependent loads): "); printf("%.1f ns\n", run_single(pflag, dbuf, 0, 5000, 32));
            printf("warp 512 B PEER stores + fence.sys: "); printf("%.1f ns\n", run_single(dflag, pbuf, 2, 5000, 32));
            printf("8 B PEER store + fence.sys: "); printf("%.1f ns\n", run_single(dflag, pbuf, 3, 5000, 32));
            printf("warp 512 B PEER stores + fence.acq_rel.sys: "); printf("%.1f ns\n", run_single(dflag, pbuf, 7, 5000, 32));
            printf("warp 512 B PEER stores + st.release.sys PEER flag: "); printf("%.1f ns\n", run_single(pflag, pbuf, 8, 5000, 32));
            printf("warp 512 B PEER stores only (issue rate): "); printf("%.1f ns\n", run_single(dflag, pbuf, 12, 5000, 32));
            for (int cfg = 0; cfg < 7; cfg++) {
                int data = cfg == 0 ? 0 : (cfg == 1 ? 128 : (cfg == 2 ? 4096 : (cfg == 3 ? 32768 : (cfg == 4 ? 128 : (cfg == 5 ? 128 : 32768)))));
                int fence = cfg == 0 ? 0 : (cfg <= 3 ? 1 : (cfg == 4 ? 2 : 3));
                CK(cudaSetDevice(0)); CK(cudaMemset(dflag, 0, 4096));
                CK(cudaSetDevice(1)); CK(cudaMemset(pflag, 0, 4096)); CK(cudaDeviceSynchronize());
                uint64_t *ns; CK(cudaMallocManaged(&ns, 16));
                int iters = 10000;
                CK(cudaSetDevice(1)); k_ping<<<1, 256>>>(pflag, dflag, dbuf, iters, 0, fence, 0, ns + 1);
                CK(cudaSetDevice(0)); k_ping<<<1, 256>>>(dflag, pflag, pbuf, iters, data, fence, 1, ns);
                CK(cudaSetDevice(0)); CK(cudaDeviceSynchronize()); CK(cudaSetDevice(1)); CK(cudaDeviceSynchronize());
                printf("NVLink ping-pong GPU0<->GPU1, %d B data, fence=%d: %.1f ns round trip\n", data, fence, (double)ns[0] / iters);
                cudaFree(ns);
            }
            {   // self-certifying writes over NVLink: writer on GPU 0, entry ring + certificate in GPU 1's memory, ack flag in GPU 0's
                uint8_t *ring1; uint64_t *w1, *w0; uint64_t *o; CK(cudaMallocManaged(&o, 64)); memset(o, 0, 64);
                CK(cudaSetDevice(1)); CK(cudaMalloc(&ring1, 256 * 128)); CK(cudaMalloc(&w1, 4096)); CK(cudaMemset(w1, 0, 4096)); CK(cudaMemset(ring1, 0, 256 * 128)); CK(cudaDeviceSynchronize());
                CK(cudaSetDevice(0)); CK(cudaMalloc(&w0, 4096)); CK(cudaMemset(w0, 0, 4096)); CK(cudaDeviceSynchronize());
                int iters = 10000;
                CK(cudaSetDevice(1)); k_selfcert<<<1, 32>>>(nullptr, nullptr, nullptr, w1, ring1, w0, iters, 0, o + 2);
                CK(cudaSetDevice(0)); k_selfcert<<<1, 32>>>(w0, w1, ring1, nullptr, nullptr, nullptr, iters, 1, o);
                CK(cudaSetDevice(0)); CK(cudaDeviceSynchronize()); CK(cudaSetDevice(1)); CK(cudaDeviceSynchronize());
                printf("NVLink self-certifying 128 B entry (no fence) GPU0->GPU1, ack back: %.1f ns round trip, %llu torn reads in %d\n",
                       (double)o[0] / iters, (unsigned long long)o[3], iters);
            }
        }
    }
    return 0;
}
