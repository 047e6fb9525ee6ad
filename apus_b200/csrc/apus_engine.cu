/*
 * apus_engine.cu -- host side of the C ABI declared in include/apus_gpu.h.
 *
 * Thin by design: allocate the replica's HBM region, map peers (peer access or
 * CUDA IPC -- the replacement for ibv_reg_mr + the raddr/rkey exchange of
 * dare_ibv_rc.c:245-273 / dare_ibv_ud.c:1116-1119), feed the leader's submission
 * ring (the replacement for the malloc'd tailq_entry_t list of message.h:11-22),
 * launch / stop / observe the persistent kernels of apus_kernels.cu, and enqueue
 * the stream-ordered batch kernels of apus_batch.cu.  All replication work
 * happens in those kernels; nothing here touches entry bytes, and there is no
 * CPU fallback.
 */
#include <cuda.h>
#include <cuda_runtime.h>
#include <emmintrin.h>
#include <pthread.h>
#include <sched.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include "apus_gpu.h"
#include "apus_layout.h"
#include "apus_slot.h"

extern "C" cudaError_t apus_launch_roles(const apus_role_t *d_roles, int n_roles, cudaStream_t stream);
extern "C" cudaError_t apus_kernels_load(void);
extern "C" size_t apus_kernel_smem_bytes(void);
extern "C" cudaError_t apus_batch_load(void);
extern "C" cudaError_t apus_synth_enqueue(apus_slot_t *ring, uint32_t mask, uint8_t *pay, uint64_t first_slot, uint32_t n,
                                          uint32_t type, uint32_t conn, uint64_t first_req, uint32_t len, uint32_t seed,
                                          uint64_t pay_pos0, uint32_t need, uint32_t first_flags, int sms,
                                          cudaStream_t stream);
extern "C" cudaError_t apus_pack_enqueue(const apus_pack_args_t *a, apus_hostwords_t *hw, uint64_t *bell, uint64_t upto,
                                         cudaStream_t stream);
extern "C" cudaError_t apus_consume_enqueue(const apus_consume_args_t *a, cudaStream_t stream);
extern "C" cudaError_t apus_consume_wait_enqueue(const uint8_t *region, apus_hostwords_t *hw, uint64_t epoch,
                                                 uint32_t min_entries, uint64_t timeout_ns, uint32_t *outcome,
                                                 cudaStream_t stream);
extern "C" cudaError_t apus_read_fence_enqueue(const apus_fence_args_t *a, cudaStream_t stream);
extern "C" cudaError_t apus_consume_mark_enqueue(const uint8_t *region, const apus_cons_state_t *st, uint64_t *mark,
                                                 cudaStream_t stream);

#define MAX_ROLES 160          /* CTAs of one fused launch: leader workers + local followers */
static __thread char g_err[512];

static int fail(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return APUS_ERROR;
}

#define CK(call)                                                                             \
    do {                                                                                     \
        cudaError_t _e = (call);                                                             \
        if (_e != cudaSuccess)                                                               \
            return fail("%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

/* driver entry points for fabric mode (VMM + multicast, see the fabric section below) and for stream-ordered commit
 * waits, fetched at run time */
struct drv_t {
    CUresult (*MemCreate)(CUmemGenericAllocationHandle *, size_t, const CUmemAllocationProp *, unsigned long long);
    CUresult (*MemAddressReserve)(CUdeviceptr *, size_t, size_t, CUdeviceptr, unsigned long long);
    CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long);
    CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc *, size_t);
    CUresult (*MemGetAllocationGranularity)(size_t *, const CUmemAllocationProp *, CUmemAllocationGranularity_flags);
    CUresult (*MemUnmap)(CUdeviceptr, size_t);
    CUresult (*MemRelease)(CUmemGenericAllocationHandle);
    CUresult (*MemAddressFree)(CUdeviceptr, size_t);
    CUresult (*MulticastCreate)(CUmemGenericAllocationHandle *, const CUmulticastObjectProp *);
    CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice);
    CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long);
    CUresult (*MulticastGetGranularity)(size_t *, const CUmulticastObjectProp *, CUmulticastGranularity_flags);
    CUresult (*DeviceGetAttribute)(int *, CUdevice_attribute, CUdevice);
    CUresult (*StreamWaitValue64)(CUstream, CUdeviceptr, cuuint64_t, unsigned int);
    int ok;
};
static drv_t g_drv;
static int drv_load(void)
{
    if (g_drv.ok) return APUS_OK;
#define DRV(field, name) do { void *fn = NULL; cudaDriverEntryPointQueryResult qr;                                   \
        if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn) {                    \
            cudaGetLastError(); return fail("driver entry point %s is not available", name); }                      \
        *(void **)(&g_drv.field) = fn; } while (0)
    DRV(MemCreate, "cuMemCreate"); DRV(MemAddressReserve, "cuMemAddressReserve"); DRV(MemMap, "cuMemMap");
    DRV(MemSetAccess, "cuMemSetAccess"); DRV(MemGetAllocationGranularity, "cuMemGetAllocationGranularity");
    DRV(MemUnmap, "cuMemUnmap"); DRV(MemRelease, "cuMemRelease"); DRV(MemAddressFree, "cuMemAddressFree");
    DRV(MulticastCreate, "cuMulticastCreate"); DRV(MulticastAddDevice, "cuMulticastAddDevice");
    DRV(MulticastBindMem, "cuMulticastBindMem"); DRV(MulticastGetGranularity, "cuMulticastGetGranularity");
    DRV(DeviceGetAttribute, "cuDeviceGetAttribute"); DRV(StreamWaitValue64, "cuStreamWaitValue64");
#undef DRV
    g_drv.ok = 1;
    return APUS_OK;
}
#define CU(call) do { CUresult _e = (call); if (_e != CUDA_SUCCESS) return fail("%s failed: driver error %d (%s:%d)", #call, (int)_e, __FILE__, __LINE__); } while (0)

struct StageLock {
    pthread_mutex_t *m;
    explicit StageLock(pthread_mutex_t *mu) : m(mu) { pthread_mutex_lock(m); }
    ~StageLock() { pthread_mutex_unlock(m); }
};

struct DeviceGuard {
    int prev;
    bool ok;
    explicit DeviceGuard(int dev) : prev(-1), ok(false)
    {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        ok = (cudaSetDevice(dev) == cudaSuccess);
    }
    ~DeviceGuard()
    {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

/* Resident kernels: an application's own persistent kernel, handed a view by apus_<name>_attach and ended by its stop
 * word.  Each kind's flag is read under its own lock: the consumer's under cons_mu (cons_stream_run reads it), the
 * reader's under g_live_mu (apus_replica_connect and reader_forget read it), the submitter's under none. */
enum res_kind { RES_CONSUMER, RES_SUBMITTER, RES_READER, RES_KINDS };
struct resident_t { int attached; cudaStream_t stream; };   /* stream: the one it was launched on */
static const struct {
    const char *name, *owner;     /* in messages: "apus_<name>_attach: a resident <name> ... (one per <owner>)" */
    decltype(&apus_hostwords_t::consumer_stop) stop;   /* its stop word */
    bool same_device;             /* attach refuses a stream of another device */
} k_res[RES_KINDS] = {
    {"consumer", "replica", &apus_hostwords_t::consumer_stop, false},
    {"submitter", "leader", &apus_hostwords_t::submitter_stop, true},
    {"reader", "replica", &apus_hostwords_t::reader_stop, true},
};

#define PEER_MAGIC 0x4150555342323030ull /* "APUSB200" */

struct peer_blob {
    uint64_t magic;
    int64_t  pid;
    int32_t  device;
    uint32_t pad;
    uint64_t ptr;
    uint64_t bytes;
    cudaIpcMemHandle_t ipc;
};
static_assert(sizeof(peer_blob) <= sizeof(apus_peer_handle_t), "peer handle too small");

struct apus_replica {
    apus_config_t cfg;
    uint64_t log_len;
    uint64_t entries_off;
    uint32_t idx_cap;
    uint8_t *region;
    size_t   region_bytes;
    apus_devctx_t  h_ctx;
    apus_devctx_t *d_ctx;
    apus_role_t   *d_roles;       /* table used when this replica owns a launch */
    apus_hostwords_t *hw;         /* pinned + mapped */
    apus_hostwords_t *hw_dev;
    /* submission ring (leader) */
    apus_slot_t *ring_desc_host;  /* pinned: the slot ring itself (mapped mode) or its staging mirror */
    uint8_t     *ring_pay_host;
    apus_slot_t *ring_desc_dev;   /* device-visible address the kernel reads */
    uint8_t     *ring_pay_dev;
    uint64_t    *sub_tail_dev;    /* device doorbell (device mode) */
    uint64_t    *sub_tail_stage;  /* pinned staging word for the device doorbell */
    uint32_t ring_slots, ring_bytes;
    uint64_t submitted, flushed;  /* tickets handed out / tickets whose slots the device can read */
    uint64_t belled;              /* doorbell value the kernel has been given */
    /* fabric mode (APUS_F_FABRIC): the region is a VMM allocation that can be bound to an NVSwitch multicast object */
    CUmemGenericAllocationHandle vmm_handle;
    size_t   vmm_bytes;           /* region_bytes rounded up to the allocation granularity */
    CUmemGenericAllocationHandle mc_handle;   /* leader: the group's multicast object ... */
    uint8_t *mc_region;           /* ... mapped: one store here lands in every replica's region */
    uint8_t *stage;               /* pinned bounce buffer for log reads */
    pthread_mutex_t stage_mu;     /* ... used by the consensus thread and by inspection calls from other threads */
    size_t   stage_bytes;
    uint64_t pay_head;            /* payload bytes handed out (monotone; position = % ring_bytes) */
    uint64_t pay_flushed;         /* payload bytes already made visible to the kernel */
    uint64_t *pay_end;            /* [ticket & mask] = pay_head after that ticket's image */
    int      wrap_next;           /* the next external image gets APUS_SLOT_WRAP (a device batch may end before its
                                     reservation does) */
    int      defer;
    /* launch */
    cudaStream_t stream, copy_stream;
    cudaEvent_t  ev_start, ev_stop;
    cudaEvent_t  ev_copy[2];      /* caller's stream -> copy_stream -> caller's stream (device batches, side_stream_run) */
    apus_replica *launch_owner;   /* replica whose stream/events carry the launch */
    int      in_flight;
    uint64_t launches;
    void    *peer_ptr[APUS_MAX_SERVERS];
    int      peer_is_ipc[APUS_MAX_SERVERS];
    uint32_t *d_lat;
    /* device batches (apus_submit_device) and stream-ordered commit waits (apus_stream_wait_committed) */
    uint64_t *pack_blk;           /* per packing block: APUS_PACK_BLK_WORDS (apus_pack_sizes_kernel) */
    cudaEvent_t *waits;           /* recorded right after each enqueued commit wait, not yet seen complete */
    int      n_waits, cap_waits;
    uint64_t wait_max;            /* highest ticket a stream has been made to wait for */
    /* device consumers (APUS_F_DEVICE_APPLY, apus_consume_device): their own stream, so that host-synchronous calls on
     * copy_stream never queue behind them */
    cudaStream_t cons_stream;
    cudaEvent_t ev_cons[2];       /* caller's stream -> cons_stream -> caller's stream */
    cudaEvent_t ev_fence;         /* recorded on cons_stream right behind the latest read fence (under cons_mu) */
    uint64_t fences;              /* read fences enqueued so far (under cons_mu) */
    apus_cons_state_t *cons_st;   /* consume state + APUS_CONS_BLK_WORDS per consume block (index-ring capacity / block size) */
    pthread_mutex_t cons_mu;      /* one enqueue at a time: the two events are shared by every caller */
    uint64_t cons_enqueued;       /* consume, wait and mark enqueues so far (under cons_mu): a seed needs none */
    resident_t res[RES_KINDS];    /* an attached consumer alone moves the cursor, an active submitter the ring */
    int      sub_active;          /* the attached submitter holds the ring (0: none attached, or it is dormant) */
    apus_submitter_state_t *sub_st;   /* device: the resident submitter's state, followed by pay_end[ring_slots] */
    /* the pinned block a resident reader reads its role and the peers' regions from.  The member words change under
     * g_live_mu */
    apus_reader_block_t *rb;      /* pinned + mapped, allocated at create */
    apus_reader_block_t *rb_dev;
    apus_replica *live_next;      /* the process's live replicas (g_live, under g_live_mu) */
};

/* Every live replica of this process, for the read fences: a fence reads the regions of the peers its replica maps, so
 * apus_replica_destroy(p) unmaps p from every replica that maps it and waits for their pending fences before p's region
 * is freed.  It and apus_read_fence hold g_live_mu while they do so (lock order: g_live_mu, then a replica's cons_mu). */
static pthread_mutex_t g_live_mu = PTHREAD_MUTEX_INITIALIZER;
static apus_replica *g_live = NULL;

extern "C" int apus_abi_version(void) { return APUS_ABI_VERSION; }
extern "C" const char *apus_last_error(void) { return g_err; }
extern "C" int apus_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

/* NUMA node of the host memory closest to a GPU (-1 = unknown): pinned rings and commit words should live there, and
 * the threads that write / spin on them should run there -- a far-socket ring costs every PCIe poll a QPI/UPI hop */
extern "C" int apus_device_numa_node(int device)
{
    char bus[64] = {0}, path[160];
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char *c = bus; *c; c++) if (*c >= 'A' && *c <= 'F') *c = (char)(*c - 'A' + 'a');
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE *f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

static inline int is_leader(const apus_replica *r) { return r->cfg.server_idx == r->cfg.leader_idx; }

/* end every consume wait enqueued so far (apus_consume_wait): each carries the epoch it was enqueued under */
static inline void consume_wait_release(apus_replica *r)
{
    if (r->hw) __atomic_fetch_add(&r->hw->cons_wait_epoch, 1ull, __ATOMIC_SEQ_CST);
}

/* detach and destroy (under the kind's lock): end the attached resident kernel of kind k by moving its stop word, and
 * wait for the stream it was launched on.  APUS_ERROR when none is attached */
static int resident_stop(apus_replica *r, res_kind k)
{
    if (!r->res[k].attached) return fail("apus_%s_detach: no resident %s is attached", k_res[k].name, k_res[k].name);
    __atomic_fetch_add(&(r->hw->*k_res[k].stop), 1ull, __ATOMIC_SEQ_CST);
    cudaStreamSynchronize(r->res[k].stream);
    r->res[k] = resident_t{};
    return APUS_OK;
}

/* the last checks of every attach: none of kind k is attached, and, where the kind asks, `stream` (which detach
 * synchronises) is on r's GPU.  Then no lazy load of ours may wait for the resident kernel from here on */
static int resident_attach_check(apus_replica *r, res_kind k, void *stream)
{
    const char *name = k_res[k].name, *owner = k_res[k].owner;
    if (r->res[k].attached) return fail("apus_%s_attach: a resident %s is attached already (one per %s)", name, name, owner);
    int sdev = r->cfg.device;
    if (k_res[k].same_device) CK(cudaStreamGetDevice((cudaStream_t)stream, &sdev));
    if (sdev != r->cfg.device)
        return fail("apus_%s_attach: the stream is on device %d, the %s on device %d", name, sdev, owner, r->cfg.device);
    CK(apus_kernels_load());
    return APUS_OK;
}

/* the log part of a resident view: r's log ring, its offset index and its consumer record */
template <typename View>
static void view_log(const apus_replica *r, View *v)
{
    v->entries = r->region + r->entries_off;
    v->log_len = r->log_len;
    v->index = reinterpret_cast<const uint32_t *>(r->region + APUS_INDEX_OFF);
    v->idx_mask = r->idx_cap - 1;
    v->rec = reinterpret_cast<const uint64_t *>(r->region + offsetof(apus_ctrl_t, cons_rec));
}

/* the first peer of r mapped through CUDA IPC, or -1 (fences read the peers' regions: they are for one process) */
static int ipc_peer(const apus_replica *r)
{
    for (int i = 0; i < APUS_MAX_SERVER_COUNT; i++)
        if (r->peer_is_ipc[i] && r->peer_ptr[i]) return i;
    return -1;
}

/* the SID this replica knows, [TERM|L|IDX] (dare_server.h:46-61): its SID word and the reader block's role word */
static inline uint64_t role_sid(const apus_replica *r) { return (r->cfg.term << 9) | (1ull << 8) | r->cfg.leader_idx; }

/* Clear member word i of r's reader block (under g_live_mu), then wait until no fence that may have read the old word
 * still reads that region: the host's half of the handshake of include/apus_reader.cuh.  A busy word is odd only across
 * one fence's N + 2 remote loads.  Without an attached reader no fence runs (detach synchronised its stream). */
static void reader_forget(apus_replica *r, int i)
{
    if (!r->rb || !r->rb->member[i]) return;
    r->rb->member[i] = 0;
    __sync_synchronize();
    if (!r->res[RES_READER].attached) return;
    for (int s = 0; s < APUS_READER_SLOTS; s++) {
        const uint64_t b = r->rb->busy[s];
        if (b & 1)
            while (r->rb->busy[s] == b) _mm_pause();
    }
}

/* the calls that write the submission ring: a resident submitter, while active, alone writes it */
static int ring_writer_gate(const apus_replica *r, const char *what)
{
    if (!r) return fail("null argument");
    if (r->sub_active)
        return fail("%s: a resident submitter is attached (apus_submitter_detach first): it alone writes the ring", what);
    return APUS_OK;
}

static int ensure_host_ring(apus_replica *r)
{
    /* device ring: the pinned staging copy of the ring is only needed when the HOST submits (lazily allocated:
     * a ring filled by apus_submit_synth never touches host memory) */
    if (r->ring_desc_host) return APUS_OK;
    CK(cudaHostAlloc(&r->ring_desc_host, sizeof(apus_slot_t) * r->ring_slots, cudaHostAllocMapped | cudaHostAllocPortable));
    CK(cudaHostAlloc(&r->ring_pay_host, r->ring_bytes, cudaHostAllocMapped | cudaHostAllocPortable));
    return APUS_OK;
}

static int fabric_alloc_region(apus_replica *r);
static int leader_ring_init(apus_replica *r)
{
    if (r->pay_end) return APUS_OK;                      /* already a leader once */
    if (!r->ring_slots) { r->ring_slots = r->cfg.ring_slots ? r->cfg.ring_slots : (1u << 16);
                          r->ring_bytes = r->cfg.ring_bytes ? r->cfg.ring_bytes : (16u << 20); }
    r->pay_end = (uint64_t *)calloc(r->ring_slots, sizeof(uint64_t));
    if (!r->pay_end) return fail("out of memory");
    if (r->cfg.ring_mode == APUS_RING_HOST_MAPPED) {
        if (ensure_host_ring(r) != APUS_OK) return APUS_ERROR;
        memset(r->ring_desc_host, 0, sizeof(apus_slot_t) * r->ring_slots);     /* no stamp matches ticket 0 */
        CK(cudaHostGetDevicePointer(&r->ring_desc_dev, r->ring_desc_host, 0));
        CK(cudaHostGetDevicePointer(&r->ring_pay_dev, r->ring_pay_host, 0));
    } else {
        CK(cudaMalloc(&r->ring_desc_dev, sizeof(apus_slot_t) * r->ring_slots));
        CK(cudaMalloc(&r->ring_pay_dev, r->ring_bytes));
        CK(cudaMalloc(&r->sub_tail_dev, 128));
        CK(cudaMemset(r->sub_tail_dev, 0, 128));
        CK(cudaHostAlloc(&r->sub_tail_stage, 64, cudaHostAllocPortable));
        CK(cudaMalloc(&r->pack_blk, APUS_PACK_BLK_WORDS * sizeof(uint64_t) * apus_pack_blocks(r->ring_slots)));
        /* a resident submitter's state, allocated with the ring: apus_submitter_attach allocates nothing */
        CK(cudaMalloc(&r->sub_st, sizeof(apus_submitter_state_t) + 8ull * r->ring_slots));
        CK(apus_batch_load());
    }
    return APUS_OK;
}

static int replica_init(apus_replica *r, const apus_config_t *cfg, uint64_t log_len)
{
    r->log_len = log_len;
    uint32_t cap = 1024;
    while ((uint64_t)cap * 64ull < log_len) cap <<= 1;
    r->idx_cap = cap;
    r->entries_off = (APUS_INDEX_OFF + (uint64_t)cap * 4ull + 4095ull) & ~4095ull;
    r->region_bytes = r->entries_off + log_len;
    if (r->cfg.flags & APUS_F_FABRIC) { if (fabric_alloc_region(r) != APUS_OK) return APUS_ERROR; }
    else CK(cudaMalloc(&r->region, r->region_bytes));
    CK(cudaMemset(r->region, 0, r->region_bytes));
    /* log_new(): end = tail = old_end = len (dare_log.h:129-134) */
    apus_loghdr_t h;
    memset(&h, 0, sizeof h);
    h.len = log_len; h.end = log_len; h.tail = log_len; h.old_end = log_len;
    CK(cudaMemcpy(r->region + APUS_HDR_OFF, &h, sizeof h, cudaMemcpyHostToDevice));
    apus_ctrl_t c;
    memset(&c, 0, sizeof c);
    c.next_idx = 1;
    c.pend_head_end = log_len;   /* no HEAD entry pending */
    if (r->cfg.flags & APUS_F_DEVICE_APPLY) {
        /* the consumers start at offset 0 with idx 1, where the first entry goes; nothing is committed yet */
        c.cons_cur[1] = 1;
        c.cons_on = (r->cfg.flags & APUS_F_APPLY_ANY_ROLE) ? 2 : 1;    /* what a leader adjusting this replica looks at */
        pthread_mutex_init(&r->cons_mu, NULL);
        CK(cudaStreamCreateWithFlags(&r->cons_stream, cudaStreamNonBlocking));
        for (cudaEvent_t &e : r->ev_cons) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&r->ev_fence, cudaEventDisableTiming));
        const size_t sb = sizeof(apus_cons_state_t) + 8ull * APUS_CONS_BLK_WORDS * ((cap + APUS_CONS_THREADS - 1) / APUS_CONS_THREADS);
        CK(cudaMalloc(&r->cons_st, sb));
        CK(cudaMemset(r->cons_st, 0, sb));
        CK(apus_batch_load());
    }
    CK(cudaMemcpy(r->region, &c, sizeof c, cudaMemcpyHostToDevice));

    CK(cudaHostAlloc(&r->hw, sizeof(apus_hostwords_t), cudaHostAllocMapped | cudaHostAllocPortable));
    memset((void *)r->hw, 0, sizeof(apus_hostwords_t));
    r->hw->cons_wait_outcome = ~0ull;                                  /* no consume wait has run */
    r->hw->fence_outcome = ~0ull;                                      /* no read fence has run */
    CK(cudaHostGetDevicePointer(&r->hw_dev, r->hw, 0));
    pthread_mutex_init(&r->stage_mu, NULL);
    r->stage_bytes = 1u << 20;
    CK(cudaHostAlloc(&r->stage, r->stage_bytes, cudaHostAllocPortable));
    CK(cudaMalloc(&r->d_ctx, sizeof(apus_devctx_t)));
    CK(cudaMalloc(&r->d_roles, sizeof(apus_role_t) * MAX_ROLES));
    CK(cudaMalloc(&r->d_lat, sizeof(uint32_t) * APUS_LAT_RING));
    CK(cudaMemset(r->d_lat, 0, sizeof(uint32_t) * APUS_LAT_RING));
    CK(cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&r->copy_stream, cudaStreamNonBlocking));
    for (cudaEvent_t &e : r->ev_copy) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CK(cudaEventCreate(&r->ev_start));
    CK(cudaEventCreate(&r->ev_stop));

    if (is_leader(r) && leader_ring_init(r) != APUS_OK) return APUS_ERROR;
    /* control-plane words: SID of a group whose leader is known from the start, no votes */
    {
        apus_ctlwords_t w;
        memset(&w, 0, sizeof w);
        w.sid = role_sid(r);
        for (int i = 0; i < 16; i++) w.vote_ack[i] = log_len;
        CK(cudaMemcpy(r->region + APUS_CTL_OFF, &w, sizeof w, cudaMemcpyHostToDevice));
    }
    r->peer_ptr[cfg->server_idx] = r->region;
    CK(cudaHostAlloc(&r->rb, sizeof(apus_reader_block_t), cudaHostAllocMapped | cudaHostAllocPortable));
    memset((void *)r->rb, 0, sizeof(apus_reader_block_t));
    r->rb->role = role_sid(r);
    r->rb->member[cfg->server_idx] = (uint64_t)(uintptr_t)r->region;
    CK(cudaHostGetDevicePointer(&r->rb_dev, r->rb, 0));
    return APUS_OK;
}

extern "C" int apus_replica_create(const apus_config_t *cfg, apus_replica_t **out)
{
    if (!cfg || !out) return fail("null argument");
    if (cfg->struct_size != sizeof(apus_config_t) && cfg->struct_size != APUS_CONFIG_SIZE_V1)
        return fail("apus_config_t size mismatch (ABI)");
    if (cfg->group_size < 1 || cfg->group_size > APUS_MAX_SERVER_COUNT) return fail("group_size out of range");
    if (cfg->server_idx >= cfg->group_size || cfg->leader_idx >= cfg->group_size) return fail("bad server/leader idx");
    int ndev = apus_device_count();
    if (ndev <= 0) return fail("no CUDA device: the engine has no CPU fallback");
    if (cfg->device < 0 || cfg->device >= ndev) return fail("device %d out of range (%d present)", cfg->device, ndev);
    /* every parameter is validated BEFORE anything is allocated */
    uint64_t log_len = cfg->log_size ? cfg->log_size : APUS_LOG_SIZE;
    if (log_len % 4096 || log_len < 8192) return fail("log_size must be a multiple of 4096 (>= 8192)");
    if (log_len > (1ull << 31)) return fail("log_size above 2 GiB is not supported (32-bit offset index)");
    uint32_t slots = cfg->ring_slots ? cfg->ring_slots : (1u << 16);
    uint32_t bytes = cfg->ring_bytes ? cfg->ring_bytes : (16u << 20);
    if ((cfg->flags & APUS_F_DEVICE_APPLY) && (cfg->flags & APUS_F_HOST_APPLY))
        return fail("APUS_F_DEVICE_APPLY and APUS_F_HOST_APPLY exclude each other: one consumer reports the apply offset");
    if ((cfg->flags & APUS_F_APPLY_ANY_ROLE) && !(cfg->flags & APUS_F_DEVICE_APPLY))
        return fail("APUS_F_APPLY_ANY_ROLE needs APUS_F_DEVICE_APPLY: it lets the device consumers work in every role");
    if ((cfg->flags & APUS_F_DEVICE_APPLY) && !(cfg->flags & APUS_F_APPLY_ANY_ROLE) && cfg->server_idx == cfg->leader_idx)
        return fail("APUS_F_DEVICE_APPLY is for followers");
    if (slots & (slots - 1)) return fail("ring_slots must be a power of two");
    if (bytes % 4096 || bytes < (1u << 17)) return fail("ring_bytes must be a multiple of 4096, >= 128 KiB");
    if (bytes / 16 > 0x00ffffffu) return fail("ring_bytes too large for the 24-bit descriptor offset");

    DeviceGuard g(cfg->device);
    if (!g.ok) return fail("cudaSetDevice(%d) failed", cfg->device);
    apus_replica *r = (apus_replica *)calloc(1, sizeof(*r));
    if (!r) return fail("out of memory");
    memset(&r->cfg, 0, sizeof r->cfg);
    memcpy(&r->cfg, cfg, cfg->struct_size);
    r->cfg.struct_size = sizeof(apus_config_t);
    if (!(r->cfg.flags & APUS_F_EXPLICIT)) r->cfg.flags |= APUS_F_DEVICE_STATS;
    if (cfg->server_idx == cfg->leader_idx) { r->ring_slots = slots; r->ring_bytes = bytes; }
    if (replica_init(r, cfg, log_len) != APUS_OK) {
        /* one cleanup path: whatever was allocated so far goes away with the partial object (g_err is kept) */
        char keep[sizeof g_err];
        memcpy(keep, g_err, sizeof keep);
        apus_replica_destroy(r);
        memcpy(g_err, keep, sizeof keep);
        return APUS_ERROR;
    }
    pthread_mutex_lock(&g_live_mu);
    r->live_next = g_live;
    g_live = r;
    pthread_mutex_unlock(&g_live_mu);
    *out = r;
    return APUS_OK;
}

extern "C" void apus_replica_destroy(apus_replica_t *r)
{
    if (!r) return;
    /* fences of other replicas that read my region.  Out of the live list first: a fence enqueued from now on counts me
     * as not connected.  Every replica of the process that maps me forgets my address, so that a replica created later
     * at the same address is never taken for me.  One that has a fence still pending ends its consume waits and fences
     * (the shared release epoch: a fence may sit behind a pending consume wait) and waits for its latest fence; one with
     * no fence pending is left alone.  The wait is for work on its consume stream up to that fence, which ends within
     * microseconds of the release unless that stream waits on a caller's stream; meanwhile g_live_mu is held, so
     * replica creation, destruction and fences in this process wait too. */
    {
        StageLock ll(&g_live_mu);
        for (apus_replica **p = &g_live; *p; p = &(*p)->live_next)
            if (*p == r) { *p = r->live_next; break; }
        for (apus_replica *q = g_live; q && r->region; q = q->live_next) {
            bool maps = false;
            for (int i = 0; i < APUS_MAX_SERVER_COUNT; i++)
                if (i != q->cfg.server_idx && !q->peer_is_ipc[i] && q->peer_ptr[i] == (void *)r->region) {
                    q->peer_ptr[i] = NULL;
                    reader_forget(q, i);
                    maps = true;
                }
            if (!maps || !q->fences) continue;
            DeviceGuard gq(q->cfg.device);
            if (cudaEventQuery(q->ev_fence) == cudaSuccess) continue;
            cudaGetLastError();
            consume_wait_release(q);
            cudaEventSynchronize(q->ev_fence);
        }
    }
    DeviceGuard g(r->cfg.device);
    /* a resident consumer reads the region and the pinned words, and freeing memory waits for every kernel on the GPU:
     * end it first */
    if (r->cons_stream) {
        StageLock cl(&r->cons_mu);
        if (r->res[RES_CONSUMER].attached) resident_stop(r, RES_CONSUMER);
    }
    if (r->res[RES_SUBMITTER].attached) resident_stop(r, RES_SUBMITTER);   /* it writes the ring and reads the pinned words */
    if (r->res[RES_READER].attached) resident_stop(r, RES_READER);  /* it reads the regions, the pinned words and the block */
    if (r->in_flight && r->hw) {
        r->hw->stop = 1;
        cudaEventSynchronize(r->launch_owner ? r->launch_owner->ev_stop : r->ev_stop);
    }
    /* streams still waiting on the committed-tickets word poll the hostwords page freed below: release them first.
     * The kernels are stopped, so nothing else writes the word; the value is at or above every ticket waited on
     * (the wait compares as a signed 64-bit difference, so UINT64_MAX would read as "below") */
    if (r->n_waits) {
        if (r->hw->committed_tickets < r->wait_max) r->hw->committed_tickets = r->wait_max;
        __sync_synchronize();
        for (int i = 0; i < r->n_waits; i++) { cudaEventSynchronize(r->waits[i]); cudaEventDestroy(r->waits[i]); }
    }
    free(r->waits);
    if (r->copy_stream) cudaStreamSynchronize(r->copy_stream);      /* device batches still packing into the rings */
    /* consume waits poll the hostwords page freed below: end them rather than wait for their timeouts */
    if (r->cons_stream) consume_wait_release(r);
    if (r->cons_stream) cudaStreamSynchronize(r->cons_stream);      /* consume work still reading the region */
    for (int i = 0; i < APUS_MAX_SERVER_COUNT; i++)
        if (r->peer_is_ipc[i] && r->peer_ptr[i]) cudaIpcCloseMemHandle(r->peer_ptr[i]);
    if (r->cfg.ring_mode != APUS_RING_HOST_MAPPED) {
        if (r->ring_desc_dev) cudaFree(r->ring_desc_dev);
        if (r->ring_pay_dev) cudaFree(r->ring_pay_dev);
        if (r->sub_tail_dev) cudaFree(r->sub_tail_dev);
        if (r->sub_tail_stage) cudaFreeHost(r->sub_tail_stage);
        if (r->pack_blk) cudaFree(r->pack_blk);
    }
    if (r->ring_desc_host) cudaFreeHost(r->ring_desc_host);
    if (r->ring_pay_host) cudaFreeHost(r->ring_pay_host);
    if (r->stage) cudaFreeHost(r->stage);
    if (r->d_lat) cudaFree(r->d_lat);
    if (r->d_roles) cudaFree(r->d_roles);
    if (r->d_ctx) cudaFree(r->d_ctx);
    if (r->ev_start) cudaEventDestroy(r->ev_start);
    if (r->ev_stop) cudaEventDestroy(r->ev_stop);
    for (cudaEvent_t e : {r->ev_copy[0], r->ev_copy[1], r->ev_cons[0], r->ev_cons[1], r->ev_fence})
        if (e) cudaEventDestroy(e);
    if (r->cons_st) cudaFree(r->cons_st);
    if (r->sub_st) cudaFree(r->sub_st);
    if (r->cons_stream) cudaStreamDestroy(r->cons_stream);
    if (r->stream) cudaStreamDestroy(r->stream);
    if (r->copy_stream) cudaStreamDestroy(r->copy_stream);
    if (r->hw) cudaFreeHost((void *)r->hw);
    if (r->rb) cudaFreeHost((void *)r->rb);
    if (r->vmm_handle && g_drv.ok) {
        if (r->mc_region) { g_drv.MemUnmap((CUdeviceptr)r->mc_region, r->vmm_bytes); g_drv.MemAddressFree((CUdeviceptr)r->mc_region, r->vmm_bytes); }
        if (r->mc_handle) g_drv.MemRelease(r->mc_handle);
        if (r->region) { g_drv.MemUnmap((CUdeviceptr)r->region, r->vmm_bytes); g_drv.MemAddressFree((CUdeviceptr)r->region, r->vmm_bytes); }
        g_drv.MemRelease(r->vmm_handle);
    } else if (r->region) cudaFree(r->region);
    cudaGetLastError();
    free(r->pay_end);
    free(r);
}

extern "C" int apus_replica_export(apus_replica_t *r, apus_peer_handle_t *out)
{
    if (!r || !out) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    peer_blob b;
    memset(&b, 0, sizeof b);
    b.magic = PEER_MAGIC; b.pid = (int64_t)getpid(); b.device = r->cfg.device;
    b.ptr = (uint64_t)(uintptr_t)r->region; b.bytes = r->region_bytes;
    if (!r->vmm_handle) CK(cudaIpcGetMemHandle(&b.ipc, r->region));       /* (fabric regions: same-process peers only, this round) */
    memset(out, 0, sizeof *out);
    memcpy(out, &b, sizeof b);
    return APUS_OK;
}

extern "C" int apus_replica_connect(apus_replica_t *r, uint8_t peer_idx, const apus_peer_handle_t *peer)
{
    if (!r || !peer) return fail("null argument");
    if (peer_idx >= r->cfg.group_size) return fail("peer idx out of range");
    if (peer_idx == r->cfg.server_idx) return APUS_OK;
    peer_blob b;
    memcpy(&b, peer, sizeof b);
    if (b.magic != PEER_MAGIC) return fail("bad peer handle");
    if (b.bytes != r->region_bytes) return fail("peer region size differs (log_size mismatch)");
    DeviceGuard g(r->cfg.device);
    if (b.pid == (int64_t)getpid()) {
        if (b.device != r->cfg.device) {
            int can = 0;
            CK(cudaDeviceCanAccessPeer(&can, r->cfg.device, b.device));
            if (!can) return fail("device %d cannot access peer device %d", r->cfg.device, b.device);
            cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
                return fail("cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e));
            cudaGetLastError();
        }
        StageLock ll(&g_live_mu);
        if (r->rb->member[peer_idx] != b.ptr) reader_forget(r, peer_idx);    /* another replica was mapped there */
        r->peer_ptr[peer_idx] = (void *)(uintptr_t)b.ptr;
        r->peer_is_ipc[peer_idx] = 0;
        r->rb->member[peer_idx] = b.ptr;
    } else {
        void *p = NULL;
        if (r->vmm_handle) return fail("fabric-mode regions are shared between replicas of one process only");
        StageLock ll(&g_live_mu);
        if (r->res[RES_READER].attached)
            return fail("apus_replica_connect: a resident reader is attached, and readers do not read peers mapped "
                        "through CUDA IPC (apus_reader_detach first)");
        reader_forget(r, peer_idx);                      /* IPC-mapped peers are never entered */
        CK(cudaIpcOpenMemHandle(&p, b.ipc, cudaIpcMemLazyEnablePeerAccess));
        r->peer_ptr[peer_idx] = p;
        r->peer_is_ipc[peer_idx] = 1;
    }
    return APUS_OK;
}

static void fill_ctx(apus_replica *r, uint64_t target)
{
    apus_devctx_t *c = &r->h_ctx;
    memset(c, 0, sizeof *c);
    c->idx = r->cfg.server_idx; c->group_size = r->cfg.group_size; c->leader_idx = r->cfg.leader_idx;
    c->quorum = (uint8_t)(r->cfg.group_size / 2 + 1);        /* dare_ibv_rc.c:1741 */
    c->flags = r->cfg.flags & 0x7fffffffu;
    c->term = r->cfg.term; c->log_len = r->log_len; c->target = target;
    c->entries_off = r->entries_off; c->idx_mask = r->idx_cap - 1;
    c->n_workers = r->cfg.leader_ctas ? r->cfg.leader_ctas : 4;
    if (c->n_workers > 96) c->n_workers = 96;
    c->epoch = (uint32_t)(r->launches + 1);
    c->doorbell_relay = (r->cfg.ring_mode == APUS_RING_HOST_MAPPED && c->n_workers >= 2) ? 1u : 0u;
    c->slot_poll = (r->cfg.ring_mode == APUS_RING_HOST_MAPPED) ? 1u : 0u;
    c->hb_period_ns = (uint64_t)r->cfg.hb_period_us * 1000ull;
    c->hb_timeout_ns = (target == ~0ull) ? (uint64_t)r->cfg.hb_timeout_us * 1000ull : 0;   /* bounded launches end on their own */
    c->region = r->region;
    c->mc_region = r->mc_region;
    for (int i = 0; i < APUS_MAX_SERVER_COUNT; i++)
        c->peer[i] = (i == r->cfg.server_idx) ? NULL : (uint8_t *)r->peer_ptr[i];
    c->sub_slots = r->ring_desc_dev; c->sub_pay = r->ring_pay_dev;
    c->sub_mask = r->ring_slots ? r->ring_slots - 1 : 0;
    c->sub_tail = (r->cfg.ring_mode == APUS_RING_HOST_MAPPED) ? (const volatile uint64_t *)&r->hw_dev->sub_tail
                                                              : (const volatile uint64_t *)r->sub_tail_dev;
    c->hw = r->hw_dev;
    c->lat_ns = r->d_lat;
}

static int submitter_hand_over(apus_replica *r);
extern "C" int apus_replicas_launch(apus_replica_t **rs, int n, uint64_t target)
{
    if (!rs || n < 1 || n > 64) return fail("bad replica list");
    apus_replica *owner = rs[0];
    for (int i = 0; i < n; i++) {
        if (!rs[i]) return fail("null replica");
        if (rs[i]->cfg.device != owner->cfg.device) return fail("replicas of one launch must share a device");
        if (rs[i]->in_flight) return fail("replica %d already has a launch in flight", (int)rs[i]->cfg.server_idx);
        if (!is_leader(rs[i]) && !rs[i]->peer_ptr[rs[i]->cfg.leader_idx]) return fail("follower not connected to its leader");
    }
    DeviceGuard g(owner->cfg.device);
    /* a leader's dormant submitter takes the ring over before the kernel runs: the host's tickets come first */
    for (int i = 0; i < n; i++)
        if (is_leader(rs[i]) && rs[i]->res[RES_SUBMITTER].attached && !rs[i]->sub_active &&
            submitter_hand_over(rs[i]) != APUS_OK)
            return APUS_ERROR;
    apus_role_t roles[MAX_ROLES];
    int nroles = 0;
    for (int i = 0; i < n; i++) {
        apus_replica *r = rs[i];
        fill_ctx(r, target);
        r->hw->stop = 0; r->hw->error = 0; r->hw->leader_suspect = 0;
        CK(cudaMemcpyAsync(r->d_ctx, &r->h_ctx, sizeof(apus_devctx_t), cudaMemcpyHostToDevice, owner->stream));
        if (is_leader(r)) {
            for (uint32_t w = 0; w < r->h_ctx.n_workers; w++) {
                if (nroles >= MAX_ROLES) return fail("too many roles in one launch");
                roles[nroles].kind = APUS_ROLE_LEADER; roles[nroles].worker = w; roles[nroles].ctx = r->d_ctx; nroles++;
            }
        } else {
            if (nroles >= MAX_ROLES) return fail("too many roles in one launch");
            roles[nroles].kind = APUS_ROLE_FOLLOWER; roles[nroles].worker = 0; roles[nroles].ctx = r->d_ctx; nroles++;
        }
    }
    CK(cudaMemcpyAsync(owner->d_roles, roles, sizeof(apus_role_t) * nroles, cudaMemcpyHostToDevice, owner->stream));
    /* roles[] is on the stack: the copy above must have read it before we return */
    CK(cudaStreamSynchronize(owner->stream));
    CK(cudaEventRecord(owner->ev_start, owner->stream));
    CK(apus_launch_roles(owner->d_roles, nroles, owner->stream));
    CK(cudaEventRecord(owner->ev_stop, owner->stream));
    for (int i = 0; i < n; i++) {
        rs[i]->launch_owner = owner;
        rs[i]->in_flight = 1;
        rs[i]->launches++;
    }
    return APUS_OK;
}

extern "C" int apus_replica_wait(apus_replica_t *r, int64_t timeout_ms)
{
    if (!r) return fail("null argument");
    if (!r->in_flight) return APUS_OK;
    apus_replica *o = r->launch_owner;
    DeviceGuard g(o->cfg.device);
    if (timeout_ms < 0) {
        CK(cudaEventSynchronize(o->ev_stop));
    } else {
        struct timespec t0, t;
        clock_gettime(CLOCK_MONOTONIC, &t0);
        for (;;) {
            cudaError_t e = cudaEventQuery(o->ev_stop);
            if (e == cudaSuccess) break;
            if (e != cudaErrorNotReady) return fail("kernel failed: %s", cudaGetErrorString(e));
            clock_gettime(CLOCK_MONOTONIC, &t);
            int64_t ms = (t.tv_sec - t0.tv_sec) * 1000 + (t.tv_nsec - t0.tv_nsec) / 1000000;
            if (ms > timeout_ms) { snprintf(g_err, sizeof g_err, "timeout"); return APUS_RETRY; }
            usleep(50);
        }
    }
    r->in_flight = 0;
    if (r->hw->error) return fail("kernel reported protocol error %llu", (unsigned long long)r->hw->error);
    return APUS_OK;
}

extern "C" int apus_replica_last_launch_ms(apus_replica_t *r, float *ms)
{
    if (!r || !ms || !r->launch_owner) return fail("no launch");
    DeviceGuard g(r->launch_owner->cfg.device);
    CK(cudaEventElapsedTime(ms, r->launch_owner->ev_start, r->launch_owner->ev_stop));
    return APUS_OK;
}

extern "C" int apus_replicas_stop(apus_replica_t **rs, int n)
{
    if (!rs) return fail("null argument");
    for (int i = 0; i < n; i++) rs[i]->hw->stop = 1;
    /* nothing commits on a stopped replica: its pending consume waits end now instead of at their timeouts */
    for (int i = 0; i < n; i++) consume_wait_release(rs[i]);
    __sync_synchronize();
    int rc = APUS_OK;
    for (int i = 0; i < n; i++) {
        int e = apus_replica_wait(rs[i], 30000);
        if (e != APUS_OK) rc = e;
    }
    return rc;
}

/* ---- submission ------------------------------------------------------------------ */
extern "C" uint8_t apus_synth_byte(uint32_t seed, uint64_t req_id, uint32_t k) { return synth_byte(seed, req_id, k); }

/* Where the data image of a request goes: inline in its slot (<= APUS_SLOT_INLINE bytes) or into the payload byte
 * ring (slot_place: include/apus_slot_format.h).  pay_end[ticket & mask] = the pay_head counter after that ticket's image.  Returns
 * the type_off word; *ppos = ring position of an external image.  APUS_RETRY when the payload ring has no room. */
static inline int place_image(apus_replica *r, uint8_t type, uint32_t nb, uint64_t consumed, uint64_t *head_io,
                              uint32_t *type_off_out, uint64_t *ppos)
{
    uint32_t flags = 0;
    const uint32_t need = slot_ext_bytes(nb);
    if (need) {
        const uint64_t tail = consumed ? r->pay_end[(consumed - 1) & (r->ring_slots - 1)] : 0;
        uint32_t wrap = 0;
        if (slot_place(r->ring_bytes, *head_io, tail, need, ppos, head_io, &wrap)) return APUS_RETRY;
        flags = APUS_SLOT_EXT | ((wrap || r->wrap_next) ? APUS_SLOT_WRAP : 0u);
        r->wrap_next = 0;
    }
    *type_off_out = slot_type_off(type, flags, need ? *ppos : 0);
    return APUS_OK;
}

static inline void write_slot(apus_slot_t *d, uint8_t *paydst, uint64_t ticket, uint8_t type, uint32_t type_off,
                              uint16_t conn, uint64_t req_id, const void *cmd, uint16_t len, uint32_t nb)
{
    if (paydst) {
        slot_put_image(paydst, type, len, cmd, nb);
    } else {
        uint8_t img[APUS_SLOT_INLINE];
        slot_put_image(img, type, len, cmd, nb);
        slot_put_inline(d, img, nb);
    }
    slot_finish(d, ticket, type_off, conn, req_id, len);
}

static int ring_put(apus_replica *r, uint8_t type, uint16_t conn, uint64_t req_id, const void *cmd, uint16_t len)
{
    const uint64_t consumed = r->hw->consumed;
    const uint32_t mask = r->ring_slots - 1;
    if (r->submitted - consumed >= r->ring_slots) return APUS_RETRY;
    if (!r->ring_desc_host && ensure_host_ring(r) != APUS_OK) return APUS_ERROR;
    const uint32_t nb = slot_image_bytes(type, len);
    uint64_t head = r->pay_head, pos = 0;
    uint32_t type_off = 0;
    int rc = place_image(r, type, nb, consumed, &head, &type_off, &pos);
    if (rc != APUS_OK) return rc;
    write_slot(&r->ring_desc_host[r->submitted & mask], (type_off & APUS_SLOT_EXT) ? r->ring_pay_host + pos : NULL,
               r->submitted + 1, type, type_off, conn, req_id, cmd, len, nb);
    r->pay_end[r->submitted & mask] = head;
    r->pay_head = head;
    r->submitted++;
    return APUS_OK;
}

/* give the kernel the doorbell value `upto` (slots up to it are readable by the device) */
static int ring_bell(apus_replica *r, uint64_t upto)
{
    if (upto <= r->belled) return APUS_OK;
    if (r->cfg.ring_mode == APUS_RING_HOST_MAPPED) {
        __sync_synchronize();                        /* descriptors + payload before the doorbell */
        r->hw->sub_tail = upto;
    } else {
        *r->sub_tail_stage = upto;
        CK(cudaMemcpyAsync(r->sub_tail_dev, r->sub_tail_stage, 8, cudaMemcpyHostToDevice, r->copy_stream));
        CK(cudaStreamSynchronize(r->copy_stream));
    }
    r->belled = upto;
    return APUS_OK;
}

/* make the slots [flushed, submitted) readable by the device (device ring: copy them over) */
static int ring_push(apus_replica *r)
{
    if (r->flushed == r->submitted) return APUS_OK;
    if (r->cfg.ring_mode == APUS_RING_HOST_MAPPED) {
        r->flushed = r->submitted;
        r->pay_flushed = r->pay_head;
        return APUS_OK;
    }
    DeviceGuard g(r->cfg.device);
    const uint32_t mask = r->ring_slots - 1;
    /* descriptors [flushed, submitted) in at most two runs */
    uint64_t f = r->flushed;
    while (f < r->submitted) {
        uint64_t i0 = f & mask;
        uint64_t run = r->submitted - f;
        if (i0 + run > r->ring_slots) run = r->ring_slots - i0;
        CK(cudaMemcpyAsync(r->ring_desc_dev + i0, r->ring_desc_host + i0, run * sizeof(apus_slot_t),
                           cudaMemcpyHostToDevice, r->copy_stream));
        f += run;
    }
    /* payload bytes [pay_flushed, pay_head) of the byte ring, in at most two runs */
    const uint64_t R = r->ring_bytes;
    uint64_t pf = r->pay_flushed;
    while (pf < r->pay_head) {
        uint64_t p0 = pf % R;
        uint64_t run = r->pay_head - pf;
        if (p0 + run > R) run = R - p0;
        CK(cudaMemcpyAsync(r->ring_pay_dev + p0, r->ring_pay_host + p0, run, cudaMemcpyHostToDevice, r->copy_stream));
        pf += run;
    }
    CK(cudaStreamSynchronize(r->copy_stream));
    r->flushed = r->submitted;
    r->pay_flushed = r->pay_head;
    return APUS_OK;
}

static int ring_flush(apus_replica *r)
{
    int rc = ring_push(r);
    if (rc != APUS_OK) return rc;
    DeviceGuard g(r->cfg.device);
    return ring_bell(r, r->submitted);
}

extern "C" int apus_submit(apus_replica_t *r, uint8_t type, uint16_t connection_id, uint64_t req_id,
                           const void *cmd, uint16_t len, uint64_t *ticket)
{
    if (ring_writer_gate(r, "apus_submit") != APUS_OK) return APUS_ERROR;
    if (!is_leader(r)) return fail("submit on a follower (proxy.c:235 only submits when is_leader())");
    if (len && !cmd) return fail("null payload");
    int rc = ring_put(r, type, connection_id, req_id, cmd, len);
    if (rc != APUS_OK) { if (rc == APUS_RETRY) snprintf(g_err, sizeof g_err, "submission ring full"); return rc; }
    if (ticket) *ticket = r->submitted;
    if (!r->defer) return ring_flush(r);
    return APUS_OK;
}

extern "C" int apus_submit_batch(apus_replica_t *r, uint32_t n, const uint8_t *types, const uint16_t *conns,
                                 const uint64_t *req_ids, const uint16_t *lens, const void *payloads,
                                 size_t stride, uint64_t *first_ticket)
{
    if (!r || !types || !conns || !req_ids || !lens) return fail("null argument");
    if (ring_writer_gate(r, "apus_submit_batch") != APUS_OK) return APUS_ERROR;
    if (!is_leader(r)) return fail("submit on a follower");
    uint64_t t0 = r->submitted + 1;
    /* all or nothing: remember the ring state */
    const uint64_t save_sub = r->submitted, save_head = r->pay_head;
    const int save_wrap = r->wrap_next;
    for (uint32_t k = 0; k < n; k++) {
        const uint8_t *p = payloads ? (const uint8_t *)payloads + (size_t)k * stride : NULL;
        int rc = ring_put(r, types[k], conns[k], req_ids[k], p, lens[k]);
        if (rc != APUS_OK) {
            r->submitted = save_sub; r->pay_head = save_head; r->wrap_next = save_wrap;
            if (rc == APUS_RETRY) snprintf(g_err, sizeof g_err, "submission ring full");
            return rc;
        }
    }
    if (first_ticket) *first_ticket = t0;
    if (!r->defer) return ring_flush(r);
    return APUS_OK;
}

/* ---- bulk submission of one request shape, filled by several host threads ------------------------ */
struct fill_job {
    apus_replica *r;
    uint32_t n;
    uint8_t type; uint16_t conn; uint64_t first_req; uint16_t len;
    const uint8_t *payloads; size_t stride;
    uint64_t first_slot;          /* r->submitted when the job was cut */
    const uint32_t *type_off;     /* per request (external images) or NULL: all inline */
    const uint64_t *pos;
    uint32_t type_off_inline;
};
static void fill_range(const fill_job *j, uint32_t k0, uint32_t k1)
{
    apus_replica *r = j->r;
    const uint32_t mask = r->ring_slots - 1;
    const uint32_t nb = slot_image_bytes(j->type, j->len);
    for (uint32_t k = k0; k < k1; k++) {
        const uint64_t s = j->first_slot + k;
        const uint32_t to = j->type_off ? j->type_off[k] : j->type_off_inline;
        write_slot(&r->ring_desc_host[s & mask], (to & APUS_SLOT_EXT) ? r->ring_pay_host + j->pos[k] : NULL, s + 1, j->type, to,
                   j->conn, j->first_req + k, j->payloads ? j->payloads + (size_t)k * j->stride : NULL, j->len, nb);
    }
}

#define POOL_MAX 16
static struct {
    pthread_mutex_t mu;
    pthread_cond_t cv;
    pthread_t th[POOL_MAX];
    int nthreads, started;
    const fill_job *job;
    volatile uint64_t gen;                 /* job generation */
    volatile uint32_t next, done_parts, parts, chunk;
    volatile uint8_t *done;                /* per part: filled */
    volatile uint32_t adv, adv_lock;       /* parts [0, adv) are filled and their doorbell has been rung */
    int progressive;                       /* ring the doorbell as the filled prefix grows (host-mapped ring) */
} g_pool = { PTHREAD_MUTEX_INITIALIZER, PTHREAD_COND_INITIALIZER };

static void pool_work(const fill_job *j)
{
    for (;;) {
        const uint32_t p = __atomic_fetch_add(&g_pool.next, 1, __ATOMIC_ACQ_REL);
        if (p >= g_pool.parts) break;
        const uint32_t k0 = p * g_pool.chunk, k1 = (k0 + g_pool.chunk < j->n) ? k0 + g_pool.chunk : j->n;
        fill_range(j, k0, k1);
        if (g_pool.progressive) {
            /* the kernel may start on the filled PREFIX while the rest is still being written: whoever gets the
             * advance lock moves the doorbell over every part that is complete and contiguous */
            __atomic_store_n(&g_pool.done[p], 1, __ATOMIC_RELEASE);
            if (__sync_bool_compare_and_swap(&g_pool.adv_lock, 0, 1)) {
                uint32_t a = g_pool.adv;
                while (a < g_pool.parts && __atomic_load_n(&g_pool.done[a], __ATOMIC_ACQUIRE)) a++;
                if (a != g_pool.adv) {
                    uint64_t upto = j->first_slot + (uint64_t)a * g_pool.chunk;
                    if (upto > j->first_slot + j->n) upto = j->first_slot + j->n;
                    __sync_synchronize();
                    j->r->hw->sub_tail = upto;
                    j->r->belled = upto;
                    g_pool.adv = a;
                }
                __atomic_store_n(&g_pool.adv_lock, 0, __ATOMIC_RELEASE);
            }
        }
        __atomic_fetch_add(&g_pool.done_parts, 1, __ATOMIC_ACQ_REL);
    }
}
static void *pool_main(void *)
{
    uint64_t seen = 0;
    for (;;) {
        /* spin briefly for the next job (bulk submits come back to back), then sleep */
        uint64_t g = seen;
        for (int i = 0; i < 200000 && (g = __atomic_load_n(&g_pool.gen, __ATOMIC_ACQUIRE)) == seen; i++) _mm_pause();
        if (g == seen) {
            pthread_mutex_lock(&g_pool.mu);
            while ((g = g_pool.gen) == seen) pthread_cond_wait(&g_pool.cv, &g_pool.mu);
            pthread_mutex_unlock(&g_pool.mu);
        }
        seen = g;
        pool_work(g_pool.job);
    }
    return NULL;
}
static pthread_mutex_t g_pool_run = PTHREAD_MUTEX_INITIALIZER;     /* one bulk job at a time per process */
static void pool_run(const fill_job *j)
{
    pthread_mutex_lock(&g_pool_run);
    pthread_mutex_lock(&g_pool.mu);
    if (!g_pool.started) {
        int want = 8;
        const char *e = getenv("apus_submit_threads");
        if (e) want = atoi(e);
        long cores = sysconf(_SC_NPROCESSORS_ONLN);
        if (want > cores - 1) want = (int)cores - 1;
        if (want > POOL_MAX) want = POOL_MAX;
        if (want < 1) want = 1;
        g_pool.nthreads = want - 1;                         /* the caller is a worker too */
        for (int i = 0; i < g_pool.nthreads; i++)
            if (pthread_create(&g_pool.th[i], NULL, pool_main, NULL)) { g_pool.nthreads = i; break; }
        g_pool.started = 1;
    }
    g_pool.job = j;
    g_pool.chunk = 4096;
    g_pool.parts = (j->n + g_pool.chunk - 1) / g_pool.chunk;
    g_pool.next = 0; g_pool.done_parts = 0;
    g_pool.progressive = (j->r->cfg.ring_mode == APUS_RING_HOST_MAPPED && !j->r->defer && j->r->flushed == j->r->submitted);
    g_pool.adv = 0; g_pool.adv_lock = 0;
    static uint8_t *done_buf; static uint32_t done_cap;
    if (done_cap < g_pool.parts) { free(done_buf); done_cap = g_pool.parts * 2; done_buf = (uint8_t *)malloc(done_cap); }
    memset(done_buf, 0, g_pool.parts);
    g_pool.done = done_buf;
    __atomic_fetch_add(&g_pool.gen, 1, __ATOMIC_RELEASE);
    pthread_cond_broadcast(&g_pool.cv);
    pthread_mutex_unlock(&g_pool.mu);
    pool_work(j);
    while (__atomic_load_n(&g_pool.done_parts, __ATOMIC_ACQUIRE) < g_pool.parts) _mm_pause();
    pthread_mutex_unlock(&g_pool_run);
}

extern "C" int apus_submit_uniform(apus_replica_t *r, uint32_t n, uint8_t type, uint16_t connection_id,
                                   uint64_t first_req_id, uint16_t len, const void *payloads, size_t stride,
                                   uint64_t *first_ticket)
{
    if (ring_writer_gate(r, "apus_submit_uniform") != APUS_OK) return APUS_ERROR;
    if (!is_leader(r)) return fail("submit on a follower");
    if (len && !payloads) return fail("null payload");
    if (n == 0) return APUS_OK;
    const uint64_t consumed = r->hw->consumed;
    if (r->submitted + n - consumed > r->ring_slots) { snprintf(g_err, sizeof g_err, "submission ring full"); return APUS_RETRY; }
    if (!r->ring_desc_host && ensure_host_ring(r) != APUS_OK) return APUS_ERROR;
    const uint32_t mask = r->ring_slots - 1;
    const uint32_t nb = slot_image_bytes(type, len);
    fill_job j;
    memset(&j, 0, sizeof j);
    j.r = r; j.n = n; j.type = type; j.conn = connection_id; j.first_req = first_req_id; j.len = len;
    j.payloads = (const uint8_t *)payloads; j.stride = stride; j.first_slot = r->submitted;
    uint32_t *tos = NULL; uint64_t *poss = NULL;
    uint64_t head = r->pay_head;
    if (nb > APUS_SLOT_INLINE) {
        /* external images: positions are handed out serially (cheap), the copies run in parallel */
        tos = (uint32_t *)malloc(sizeof(uint32_t) * n); poss = (uint64_t *)malloc(sizeof(uint64_t) * n);
        if (!tos || !poss) { free(tos); free(poss); return fail("out of memory"); }
        const int save_wrap = r->wrap_next;
        for (uint32_t k = 0; k < n; k++) {
            int rc = place_image(r, type, nb, consumed, &head, &tos[k], &poss[k]);
            if (rc != APUS_OK) {
                free(tos); free(poss); r->wrap_next = save_wrap;
                snprintf(g_err, sizeof g_err, "payload ring full");
                return rc;
            }
            r->pay_end[(r->submitted + k) & mask] = head;
        }
        j.type_off = tos; j.pos = poss;
    } else {
        j.type_off_inline = slot_type_off(type, 0, 0);
        for (uint32_t k = 0; k < n; k++) r->pay_end[(r->submitted + k) & mask] = head;
    }
    if (n >= 16384) pool_run(&j); else fill_range(&j, 0, n);
    free(tos); free(poss);
    r->pay_head = head;
    if (first_ticket) *first_ticket = r->submitted + 1;
    r->submitted += n;
    if (!r->defer) return ring_flush(r);
    return APUS_OK;
}

/* ---- device-generated requests ---------------------------------------------------------------------- */
extern "C" int apus_submit_synth(apus_replica_t *r, uint32_t n, uint8_t type, uint16_t connection_id,
                                 uint64_t first_req_id, uint16_t len, uint32_t seed, uint64_t *first_ticket)
{
    if (ring_writer_gate(r, "apus_submit_synth") != APUS_OK) return APUS_ERROR;
    if (!is_leader(r)) return fail("submit on a follower");
    if (r->cfg.ring_mode != APUS_RING_DEVICE) return fail("apus_submit_synth needs the device submission ring");
    if (type == APUS_NOOP || type == APUS_CONFIG || type == APUS_HEAD) return fail("apus_submit_synth: request types only");
    if (n == 0) return APUS_OK;
    const uint64_t consumed = r->hw->consumed;
    if (r->submitted + n - consumed > r->ring_slots) { snprintf(g_err, sizeof g_err, "submission ring full"); return APUS_RETRY; }
    if (r->flushed != r->submitted) { int rc = ring_push(r); if (rc != APUS_OK) return rc; }
    const uint32_t mask = r->ring_slots - 1;
    const uint32_t need = slot_ext_bytes(slot_image_bytes(type, len));
    uint64_t pos0 = 0, head = r->pay_head;
    if (need) {
        const uint64_t R = r->ring_bytes;
        pos0 = head % R;
        const uint64_t tail = consumed ? r->pay_end[(consumed - 1) & mask] : 0;
        if (pos0 + (uint64_t)n * need > R || (head - tail) + (uint64_t)n * need > R)
            return fail("apus_submit_synth: %u images of %u B do not fit the payload ring without wrapping", n, need);
    }
    DeviceGuard g(r->cfg.device);
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, r->cfg.device));
    CK(apus_synth_enqueue(r->ring_desc_dev, mask, r->ring_pay_dev, r->submitted, n, type, connection_id, first_req_id, len,
                          seed, pos0, need, r->wrap_next ? APUS_SLOT_WRAP : 0u, sms, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    if (need) r->wrap_next = 0;
    for (uint32_t k = 0; k < n; k++) { head += need; r->pay_end[(r->submitted + k) & mask] = head; }
    r->pay_head = head; r->pay_flushed = head;
    if (first_ticket) *first_ticket = r->submitted + 1;
    r->submitted += n;
    r->flushed = r->submitted;
    if (!r->defer) return ring_bell(r, r->submitted);
    return APUS_OK;
}

/* ---- stream-ordered side-stream work (device batches, device consumers) --------------------------------------- */
/* `enqueue` puts work on the side stream `side` in the caller's stream order: the side stream first waits for
 * everything the caller's stream did before this call, and the caller's stream then waits for that work.  ev is the
 * side stream's event pair; `what` names the enqueue in an error. */
template <typename Enqueue>
static int side_stream_run(cudaStream_t caller, cudaStream_t side, cudaEvent_t ev[2], const char *what, Enqueue enqueue)
{
    CK(cudaEventRecord(ev[0], caller));
    CK(cudaStreamWaitEvent(side, ev[0], 0));
    const cudaError_t e = enqueue();
    if (e != cudaSuccess) return fail("%s failed: %s", what, cudaGetErrorString(e));
    CK(cudaEventRecord(ev[1], side));
    CK(cudaStreamWaitEvent(caller, ev[1], 0));
    return APUS_OK;
}

/* ---- device batches: requests in device memory, packed into the HBM ring in stream order ------------------- */
/* the part of a device batch both layouts share: room in both rings, the placement of the `res`-byte reservation, the
 * three passes and the doorbell on copy_stream in the caller's stream order, and the space accounting */
static int submit_packing(apus_replica_t *r, const char *what, apus_pack_args_t a, uint64_t res, void *stream,
                          uint64_t *first_ticket)
{
    const uint32_t n = a.n;
    if (n > r->ring_slots) return fail("%s: %u requests can never fit a ring of %u slots", what, n, r->ring_slots);
    if (res > r->ring_bytes)
        return fail("%s: a reservation of %llu B can never fit a payload ring of %u B", what, (unsigned long long)res,
                    r->ring_bytes);
    const uint64_t consumed = r->hw->consumed;
    if (r->submitted + n - consumed > r->ring_slots) { snprintf(g_err, sizeof g_err, "submission ring full"); return APUS_RETRY; }
    const uint32_t mask = r->ring_slots - 1;
    const uint64_t head0 = r->pay_head, tail = consumed ? r->pay_end[(consumed - 1) & mask] : 0;
    uint64_t pos = 0, head = head0;
    uint32_t wrap = 0;
    if (res && slot_place(r->ring_bytes, head0, tail, res, &pos, &head, &wrap)) {
        snprintf(g_err, sizeof g_err, "payload ring full");
        return APUS_RETRY;
    }
    if (r->flushed != r->submitted) { int rc = ring_push(r); if (rc != APUS_OK) return rc; }
    DeviceGuard g(r->cfg.device);
    a.ring = r->ring_desc_dev; a.pay = r->ring_pay_dev; a.blk = r->pack_blk;
    a.first_slot = r->submitted; a.res_pos = pos; a.mask = mask;
    const uint64_t upto = r->submitted + n;
    uint64_t *bell = r->defer ? NULL : r->sub_tail_dev;
    if (side_stream_run((cudaStream_t)stream, r->copy_stream, r->ev_copy, "apus_pack_enqueue",
                        [&] { return apus_pack_enqueue(&a, r->hw_dev, bell, upto, r->copy_stream); }) != APUS_OK)
        return APUS_ERROR;
    /* space accounting: the reservation is freed only when the whole batch has been consumed */
    for (uint32_t k = 0; k + 1 < n; k++) r->pay_end[(r->submitted + k) & mask] = head0;
    r->pay_end[(upto - 1) & mask] = head;
    r->pay_head = head; r->pay_flushed = head;
    if (res) r->wrap_next = 1;
    if (first_ticket) *first_ticket = r->submitted + 1;
    r->submitted = upto;
    r->flushed = upto;
    if (!r->defer) r->belled = upto;
    return APUS_OK;
}

extern "C" int apus_submit_device(apus_replica_t *r, uint32_t n, const uint8_t *types, const uint16_t *connection_ids,
                                  const uint64_t *req_ids, const uint16_t *lens, const void *payloads, size_t stride,
                                  void *stream, uint64_t *first_ticket)
{
    if (ring_writer_gate(r, "apus_submit_device") != APUS_OK) return APUS_ERROR;
    if (!is_leader(r)) return fail("submit on a follower");
    if (r->cfg.ring_mode != APUS_RING_DEVICE) return fail("apus_submit_device needs the device submission ring");
    if (n == 0) return APUS_OK;
    if (!types || !connection_ids || !req_ids || !lens || (!payloads && stride)) return fail("null argument");
    /* lens are unknown here: reserve the worst case, round16(2 + stride) per request (nothing when that is inline) */
    const uint64_t per = slot_ext_bytes(2u + (uint32_t)(stride < 0xffffu ? stride : 0xffffu));
    apus_pack_args_t a;
    memset(&a, 0, sizeof a);
    a.types = types; a.conns = connection_ids; a.req_ids = req_ids; a.lens = lens; a.payloads = (const uint8_t *)payloads;
    a.stride = stride; a.n = n;
    return submit_packing(r, "apus_submit_device", a, (uint64_t)n * per, stream, first_ticket);
}

extern "C" int apus_submit_device_packed(apus_replica_t *r, uint32_t n, const uint8_t *types,
                                         const uint16_t *connection_ids, const uint64_t *req_ids, const uint64_t *offsets,
                                         const void *values, uint64_t values_bytes, void *stream, uint64_t *first_ticket)
{
    if (ring_writer_gate(r, "apus_submit_device_packed") != APUS_OK) return APUS_ERROR;
    if (!is_leader(r)) return fail("submit on a follower");
    if (r->cfg.ring_mode != APUS_RING_DEVICE) return fail("apus_submit_device_packed needs the device submission ring");
    if (n == 0) return APUS_OK;
    if (!types || !connection_ids || !req_ids || !offsets || (!values && values_bytes)) return fail("null argument");
    /* the kernels load whole elements: a misaligned array would fault on the device, so refuse it here */
    if (((uintptr_t)offsets | (uintptr_t)req_ids) & 7u || (uintptr_t)connection_ids & 1u)
        return fail("apus_submit_device_packed: misaligned array (offsets and req_ids need 8 B, connection_ids 2 B)");
    apus_pack_args_t a;
    memset(&a, 0, sizeof a);
    a.types = types; a.conns = connection_ids; a.req_ids = req_ids; a.offsets = offsets;
    a.payloads = (const uint8_t *)values; a.values_bytes = values_bytes; a.n = n;
    return submit_packing(r, "apus_submit_device_packed", a, slot_packed_reserve(n, values_bytes), stream, first_ticket);
}

extern "C" int apus_device_submit_status(apus_replica_t *r, uint64_t *rejected, uint64_t *first_rejected_ticket)
{
    if (!r) return fail("null argument");
    uint64_t n = r->hw->dev_rejected, first = r->hw->dev_first_rejected;
    if (r->res[RES_SUBMITTER].attached) {                /* ... and what the resident submitter has counted so far */
        DeviceGuard g(r->cfg.device);
        apus_submitter_state_t s;
        CK(cudaMemcpyAsync(&s, r->sub_st, sizeof s, cudaMemcpyDeviceToHost, r->copy_stream));
        CK(cudaStreamSynchronize(r->copy_stream));
        n += s.rejected;
        if (!first && s.rejected) first = s.first_rejected;
    }
    if (rejected) *rejected = n;
    if (first_rejected_ticket) *first_rejected_ticket = first;
    return APUS_OK;
}

/* ---- stream-ordered commit waits ------------------------------------------------------------------------ */
extern "C" int apus_stream_wait_committed(apus_replica_t *r, uint64_t ticket, void *stream)
{
    if (!r) return fail("null argument");
    if (!is_leader(r)) return fail("apus_stream_wait_committed: the committed-tickets word is the leader's");
    if (ticket >> 63) return fail("apus_stream_wait_committed: ticket out of range");
    if (drv_load() != APUS_OK) return APUS_ERROR;
    DeviceGuard g(r->cfg.device);
    int ok = 0;
    CU(g_drv.DeviceGetAttribute(&ok, CU_DEVICE_ATTRIBUTE_CAN_USE_64_BIT_STREAM_MEM_OPS, r->cfg.device));
    if (!ok)
        return fail("apus_stream_wait_committed: device %d has no 64-bit stream memory operations "
                    "(CU_DEVICE_ATTRIBUTE_CAN_USE_64_BIT_STREAM_MEM_OPS = 0)", r->cfg.device);
    /* forget the waits that have completed; the others are released by apus_replica_destroy */
    int m = 0;
    for (int i = 0; i < r->n_waits; i++) {
        if (cudaEventQuery(r->waits[i]) == cudaSuccess) cudaEventDestroy(r->waits[i]);
        else r->waits[m++] = r->waits[i];
    }
    cudaGetLastError();
    r->n_waits = m;
    if (r->n_waits == r->cap_waits) {
        const int cap = r->cap_waits ? 2 * r->cap_waits : 16;
        cudaEvent_t *w = (cudaEvent_t *)realloc(r->waits, sizeof(cudaEvent_t) * cap);
        if (!w) return fail("out of memory");
        r->waits = w; r->cap_waits = cap;
    }
    cudaEvent_t ev;
    CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    const CUresult e = g_drv.StreamWaitValue64((CUstream)stream, (CUdeviceptr)&r->hw_dev->committed_tickets, ticket,
                                               CU_STREAM_WAIT_VALUE_GEQ);
    if (e != CUDA_SUCCESS) { cudaEventDestroy(ev); return fail("cuStreamWaitValue64 failed: driver error %d", (int)e); }
    if (cudaEventRecord(ev, (cudaStream_t)stream) != cudaSuccess) {
        cudaEventDestroy(ev);
        return fail("cudaEventRecord after the commit wait failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    r->waits[r->n_waits++] = ev;
    if (ticket > r->wait_max) r->wait_max = ticket;
    return APUS_OK;
}

extern "C" const volatile uint64_t *apus_committed_word(apus_replica_t *r)
{
    return r ? &r->hw_dev->committed_tickets : NULL;
}

extern "C" int apus_submit_defer(apus_replica_t *r, int defer)
{
    if (ring_writer_gate(r, "apus_submit_defer") != APUS_OK) return APUS_ERROR;
    r->defer = defer;
    return APUS_OK;
}
extern "C" int apus_submit_flush(apus_replica_t *r)
{
    if (ring_writer_gate(r, "apus_submit_flush") != APUS_OK) return APUS_ERROR;
    return ring_flush(r);
}
extern "C" int apus_submit_release(apus_replica_t *r, uint64_t ticket)
{
    if (ring_writer_gate(r, "apus_submit_release") != APUS_OK) return APUS_ERROR;
    if (ticket > r->submitted) return fail("release beyond what was submitted");
    int rc = ring_push(r);
    if (rc != APUS_OK) return rc;
    DeviceGuard g(r->cfg.device);
    return ring_bell(r, ticket);
}

extern "C" uint64_t apus_committed_tickets(apus_replica_t *r) { return r ? r->hw->committed_tickets : 0; }

extern "C" int apus_progress(apus_replica_t *r, uint64_t *offset, uint64_t *count)
{
    if (!r) return fail("null argument");
    /* {commit_off, committed_tickets} is written by the kernel with ONE 16 B store: read it with one 16 B load */
    const __m128i v = _mm_load_si128((const __m128i *)(const void *)&r->hw->commit_off);
    uint64_t w[2];
    _mm_storeu_si128((__m128i *)w, v);
    if (offset) *offset = w[0];
    if (count) *count = w[1];
    return r->hw->error ? fail("kernel reported protocol error %llu", (unsigned long long)r->hw->error) : APUS_OK;
}

extern "C" int apus_wait_committed(apus_replica_t *r, uint64_t ticket, int64_t timeout_us)
{
    if (!r) return fail("null argument");
    if (r->hw->committed_tickets >= ticket) return APUS_OK;
    struct timespec t0, t;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    uint32_t spins = 0;
    while (r->hw->committed_tickets < ticket) {
        if ((++spins & 0x3ff) == 0) {
            if (r->hw->error) return fail("kernel reported protocol error %llu", (unsigned long long)r->hw->error);
            if (timeout_us >= 0) {
                clock_gettime(CLOCK_MONOTONIC, &t);
                int64_t us = (t.tv_sec - t0.tv_sec) * 1000000 + (t.tv_nsec - t0.tv_nsec) / 1000;
                if (us > timeout_us) { snprintf(g_err, sizeof g_err, "timeout"); return APUS_RETRY; }
            }
        }
    }
    return APUS_OK;
}

/* Closed loop with ONE request in flight, timed on the host around the two ABI steps a
 * proxy thread performs (enqueue, then spin until committed -- proxy.c:108-161). */
extern "C" int apus_closed_loop(apus_replica_t *r, uint32_t n, uint16_t payload_len, uint16_t connection_id,
                                uint64_t first_req_id, uint32_t *lat_ns)
{
    if (!r || !lat_ns) return fail("null argument");
    if (ring_writer_gate(r, "apus_closed_loop") != APUS_OK) return APUS_ERROR;
    if (!is_leader(r)) return fail("submit on a follower");
    uint8_t *buf = (uint8_t *)malloc(payload_len ? payload_len : 1);
    if (!buf) return fail("out of memory");
    for (uint32_t k = 0; k < payload_len; k++) buf[k] = (uint8_t)(k * 131u + 7u);
    struct timespec t0, t1;
    for (uint32_t i = 0; i < n; i++) {
        clock_gettime(CLOCK_MONOTONIC, &t0);
        int rc = ring_put(r, APUS_SEND, connection_id, first_req_id + i, buf, payload_len);
        if (rc == APUS_OK) rc = ring_flush(r);
        if (rc != APUS_OK) { free(buf); return rc == APUS_RETRY ? rc : fail("closed loop: submit failed"); }
        const uint64_t ticket = r->submitted;
        uint32_t spins = 0;
        while (r->hw->committed_tickets < ticket) {
            if ((++spins & 0xffffff) == 0) {
                clock_gettime(CLOCK_MONOTONIC, &t1);
                if (t1.tv_sec - t0.tv_sec > 10 || r->hw->error) { free(buf); return fail("closed loop: commit timeout"); }
            }
        }
        clock_gettime(CLOCK_MONOTONIC, &t1);
        int64_t ns = (t1.tv_sec - t0.tv_sec) * 1000000000ll + (t1.tv_nsec - t0.tv_nsec);
        lat_ns[i] = ns > 0xffffffffll ? 0xffffffffu : (uint32_t)ns;
    }
    free(buf);
    return APUS_OK;
}

/* ---- inspection ---------------------------------------------------------------- */
extern "C" int apus_log_offsets(apus_replica_t *r, apus_log_offsets_t *out)
{
    if (!r || !out) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    apus_loghdr_t h;
    CK(cudaMemcpyAsync(&h, r->region + APUS_HDR_OFF, sizeof h, cudaMemcpyDeviceToHost, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    out->head = h.head; out->apply = h.apply; out->commit = h.commit; out->end = h.end;
    out->tail = h.tail; out->old_end = h.old_end; out->old_commit = h.old_commit; out->len = h.len;
    return APUS_OK;
}

extern "C" int apus_log_read(apus_replica_t *r, uint64_t off, uint64_t len, void *dst)
{
    if (!r || !dst) return fail("null argument");
    if (off + len > r->log_len) return fail("range beyond the log");
    DeviceGuard g(r->cfg.device);
    StageLock sl(&r->stage_mu);
    /* through the pinned bounce buffer: a pageable destination would make every copy a synchronous staged one */
    uint8_t *out = (uint8_t *)dst;
    while (len) {
        const uint64_t run = len < r->stage_bytes ? len : r->stage_bytes;
        CK(cudaMemcpyAsync(r->stage, r->region + r->entries_off + off, run, cudaMemcpyDeviceToHost, r->copy_stream));
        CK(cudaStreamSynchronize(r->copy_stream));
        memcpy(out, r->stage, run);
        out += run; off += run; len -= run;
    }
    return APUS_OK;
}

extern "C" int apus_log_read_range(apus_replica_t *r, uint64_t from, uint64_t to, void *dst, uint64_t cap, uint64_t *got)
{
    if (!r || !dst || !got) return fail("null argument");
    if (from >= r->log_len || to >= r->log_len) return fail("range beyond the log");
    const uint64_t L = r->log_len;
    uint64_t n1 = to >= from ? to - from : L - from, n2 = to >= from ? 0 : to;
    if (n1 > cap) { n1 = cap; n2 = 0; }
    if (n1 + n2 > cap) n2 = cap - n1;
    int rc = n1 ? apus_log_read(r, from, n1, dst) : APUS_OK;
    if (rc == APUS_OK && n2) rc = apus_log_read(r, 0, n2, (uint8_t *)dst + n1);
    *got = n1 + n2;
    return rc;
}

extern "C" int apus_set_applied(apus_replica_t *r, uint64_t offset)
{
    if (!r) return fail("null argument");
    if (offset >= r->log_len) return fail("offset beyond the log");
    r->hw->host_apply = offset;          /* the follower kernel forwards it to the leader's pruning rule */
    return APUS_OK;
}

/* ---- device consumers: committed entries straight into device memory, in stream order ----------------------- */
/* Which replicas each consumer call accepts.  CONS_STATUS (status and release): a replica created with
 * APUS_F_DEVICE_APPLY.  CONS_STREAM (the calls that enqueue consume work): the same, but a leader only with
 * APUS_F_APPLY_ANY_ROLE, and that refusal comes first.  CONS_ANY_ROLE (fences and seeds): both flags. */
enum consumer_kind { CONS_STATUS, CONS_STREAM, CONS_ANY_ROLE };

static int consumer_gate(const apus_replica *r, const char *what, consumer_kind kind)
{
    if (!r) return fail("null argument");
    if (kind == CONS_ANY_ROLE) {
        const uint32_t need = APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE;
        if ((r->cfg.flags & need) != need)
            return fail("%s needs a replica created with APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE", what);
        return APUS_OK;
    }
    if (kind == CONS_STREAM && is_leader(r) && !(r->cfg.flags & APUS_F_APPLY_ANY_ROLE))
        return fail("%s: consumption is a follower's (the leader's log is its own)", what);
    if (!(r->cfg.flags & APUS_F_DEVICE_APPLY)) return fail("%s needs a replica created with APUS_F_DEVICE_APPLY", what);
    return APUS_OK;
}

/* One enqueue on the consume stream, in the caller's stream order and in call order with every consume call, wait, mark
 * and fence of this replica.  Under cons_mu it counts the enqueue (apus_consume_seed refuses a replica that has had
 * one) and reads the release epoch that `enqueue(epoch)` hands to a wait or fence: read in the order of the enqueues, so
 * that a release after this call ends what it enqueues. */
template <typename Enqueue>
static int cons_stream_run(apus_replica *r, void *stream, const char *what, Enqueue enqueue, bool moves_cursor = true)
{
    DeviceGuard g(r->cfg.device);
    StageLock sl(&r->cons_mu);
    if (moves_cursor && r->res[RES_CONSUMER].attached)
        return fail("%s: a resident consumer is attached (apus_consumer_detach first): it alone moves the cursor", what);
    const uint64_t epoch = r->hw->cons_wait_epoch;
    r->cons_enqueued++;
    return side_stream_run((cudaStream_t)stream, r->cons_stream, r->ev_cons, what, [&] { return enqueue(epoch); });
}

/* what both layouts share, once the arguments are checked: max_n clipped to the index ring, and the five kernels on the
 * consume stream */
static int consume_enqueue(apus_replica_t *r, apus_consume_args_t a, uint32_t max_n, void *stream)
{
    /* at most idx_cap entries lie between the cursor and what the follower holds (each is >= 64 B of one lap) */
    const uint32_t n = max_n < r->idx_cap ? max_n : r->idx_cap;
    a.region = r->region; a.entries_off = r->entries_off; a.log_len = r->log_len;
    a.idx_mask = r->idx_cap - 1; a.max_n = n; a.nblk = (n + APUS_CONS_THREADS - 1) / APUS_CONS_THREADS;
    a.st = r->cons_st; a.hw = r->hw_dev;
    return cons_stream_run(r, stream, "apus_consume_enqueue",
                           [&](uint64_t) { return apus_consume_enqueue(&a, r->cons_stream); });
}

extern "C" int apus_consume_device(apus_replica_t *r, uint32_t max_n, uint64_t *idx, uint8_t *types,
                                   uint16_t *connection_ids, uint64_t *req_ids, uint16_t *lens, void *payloads,
                                   size_t stride, uint32_t *count, void *stream)
{
    if (consumer_gate(r, "apus_consume_device", CONS_STREAM) != APUS_OK) return APUS_ERROR;
    if (max_n == 0) return fail("apus_consume_device: max_n is 0");
    if (!idx || !types || !connection_ids || !req_ids || !lens || !count || (!payloads && stride)) return fail("null argument");
    /* the kernels store whole elements: a misaligned array would fault on the device, so refuse it here */
    if (((uintptr_t)idx | (uintptr_t)req_ids) & 7u || ((uintptr_t)connection_ids | (uintptr_t)lens) & 1u || (uintptr_t)count & 3u)
        return fail("apus_consume_device: misaligned array (idx and req_ids need 8 B, count 4 B, connection_ids and lens 2 B)");
    apus_consume_args_t a;
    memset(&a, 0, sizeof a);
    a.stride = stride;
    a.idx = idx; a.types = types; a.conns = connection_ids; a.req_ids = req_ids; a.lens = lens;
    a.payloads = (uint8_t *)payloads; a.count = count;
    return consume_enqueue(r, a, max_n, stream);
}

extern "C" int apus_consume_device_packed(apus_replica_t *r, uint32_t max_n, uint64_t *idx, uint8_t *types,
                                          uint16_t *connection_ids, uint64_t *req_ids, uint64_t *offsets, void *values,
                                          uint64_t values_cap, uint32_t *count, void *stream)
{
    if (consumer_gate(r, "apus_consume_device_packed", CONS_STREAM) != APUS_OK) return APUS_ERROR;
    if (max_n == 0) return fail("apus_consume_device_packed: max_n is 0");
    if (!idx || !types || !connection_ids || !req_ids || !offsets || !count || (!values && values_cap))
        return fail("null argument");
    if (((uintptr_t)idx | (uintptr_t)req_ids | (uintptr_t)offsets) & 7u || (uintptr_t)connection_ids & 1u ||
        (uintptr_t)count & 3u)
        return fail("apus_consume_device_packed: misaligned array (idx, req_ids and offsets need 8 B, count 4 B, "
                    "connection_ids 2 B)");
    apus_consume_args_t a;
    memset(&a, 0, sizeof a);
    a.idx = idx; a.types = types; a.conns = connection_ids; a.req_ids = req_ids; a.offsets = offsets;
    a.payloads = (uint8_t *)values; a.values_cap = values_cap; a.count = count;
    return consume_enqueue(r, a, max_n, stream);
}

extern "C" int apus_consume_status(apus_replica_t *r, uint64_t *cursor_offset, uint64_t *next_idx, uint64_t *need_stride,
                                   uint64_t *error)
{
    if (consumer_gate(r, "apus_consume_status", CONS_STATUS) != APUS_OK) return APUS_ERROR;
    if (cursor_offset) *cursor_offset = r->hw->cons_cursor;
    if (next_idx) *next_idx = r->hw->cons_next_idx ? r->hw->cons_next_idx : 1;   /* before the first call: idx 1 */
    if (need_stride) *need_stride = r->hw->cons_need_stride;
    if (error) *error = r->hw->cons_error;
    return APUS_OK;
}

#define APUS_WAIT_MAX_US 60000000u     /* every consume wait ends by itself, after at most a minute */

extern "C" int apus_consume_wait(apus_replica_t *r, uint32_t min_entries, uint32_t timeout_us, uint32_t *outcome,
                                 void *stream)
{
    if (consumer_gate(r, "apus_consume_wait", CONS_STREAM) != APUS_OK) return APUS_ERROR;
    if (min_entries == 0 || min_entries > r->idx_cap)
        return fail("apus_consume_wait: min_entries %u outside [1, %u] (the index ring's capacity)", min_entries, r->idx_cap);
    if (timeout_us == 0 || timeout_us > APUS_WAIT_MAX_US)
        return fail("apus_consume_wait: timeout_us %u outside [1, %u]", timeout_us, APUS_WAIT_MAX_US);
    if ((uintptr_t)outcome & 3u) return fail("apus_consume_wait: misaligned outcome (4 B)");
    return cons_stream_run(r, stream, "apus_consume_wait_enqueue", [&](uint64_t epoch) {
        return apus_consume_wait_enqueue(r->region, r->hw_dev, epoch, min_entries, 1000ull * timeout_us, outcome,
                                         r->cons_stream);
    });
}

extern "C" int apus_consume_wait_release(apus_replica_t *r)
{
    if (consumer_gate(r, "apus_consume_wait_release", CONS_STATUS) != APUS_OK) return APUS_ERROR;
    consume_wait_release(r);
    return APUS_OK;
}

extern "C" int apus_consume_wait_status(apus_replica_t *r, uint64_t *outcome, uint64_t *available)
{
    if (consumer_gate(r, "apus_consume_wait_status", CONS_STATUS) != APUS_OK) return APUS_ERROR;
    if (outcome) *outcome = r->hw->cons_wait_outcome;
    if (available) *available = r->hw->cons_wait_avail;
    return APUS_OK;
}

extern "C" int apus_consume_mark(apus_replica_t *r, uint64_t *mark, void *stream)
{
    if (consumer_gate(r, "apus_consume_mark", CONS_STREAM) != APUS_OK) return APUS_ERROR;
    if (!mark) return fail("null argument");
    if ((uintptr_t)mark & 15u) return fail("apus_consume_mark: misaligned mark (16 B)");
    return cons_stream_run(r, stream, "apus_consume_mark_enqueue",
                           [&](uint64_t) { return apus_consume_mark_enqueue(r->region, r->cons_st, mark, r->cons_stream); });
}

extern "C" int apus_read_fence(apus_replica_t *r, uint32_t timeout_us, uint64_t *index, uint32_t *outcome, void *stream)
{
    if (consumer_gate(r, "apus_read_fence", CONS_ANY_ROLE) != APUS_OK) return APUS_ERROR;
    if (timeout_us == 0 || timeout_us > APUS_WAIT_MAX_US)
        return fail("apus_read_fence: timeout_us %u outside [1, %u]", timeout_us, APUS_WAIT_MAX_US);
    if (!index) return fail("null argument");
    if ((uintptr_t)index & 7u || (uintptr_t)outcome & 3u)
        return fail("apus_read_fence: misaligned index (8 B) or outcome (4 B)");
    const int ipc = ipc_peer(r);
    if (ipc >= 0) return fail("apus_read_fence: peer %d is mapped through CUDA IPC (fences are for groups hosted in one process)", ipc);
    apus_fence_args_t a;
    memset(&a, 0, sizeof a);
    a.region = r->region; a.hw = r->hw_dev; a.term = r->cfg.term;
    a.entries_off = r->entries_off; a.log_len = r->log_len; a.timeout_ns = 1000ull * timeout_us;
    a.index = index; a.outcome = outcome; a.idx_mask = r->idx_cap - 1;
    a.n = r->cfg.group_size; a.leader = r->cfg.leader_idx;
    /* under g_live_mu (taken before cons_mu): a peer destroyed before this point is no longer mapped here
     * (apus_replica_destroy clears it), and one destroyed after it waits for this fence */
    StageLock ll(&g_live_mu);
    for (int i = 0; i < a.n; i++) a.member[i] = (const uint8_t *)r->peer_ptr[i];
    a.member[r->cfg.server_idx] = r->region;
    return cons_stream_run(r, stream, "apus_read_fence_enqueue", [&](uint64_t epoch) {
        a.epoch = epoch;
        r->fences++;
        const cudaError_t e = apus_read_fence_enqueue(&a, r->cons_stream);
        return e == cudaSuccess ? cudaEventRecord(r->ev_fence, r->cons_stream) : e;
    }, false);
}

extern "C" int apus_read_fence_status(apus_replica_t *r, uint64_t *outcome, uint64_t *index)
{
    if (consumer_gate(r, "apus_read_fence_status", CONS_ANY_ROLE) != APUS_OK) return APUS_ERROR;
    if (outcome) *outcome = r->hw->fence_outcome;
    if (index) *index = r->hw->fence_index;
    return APUS_OK;
}

extern "C" int apus_consumer_attach(apus_replica_t *r, void *stream, apus_consumer_view_t *out)
{
    if (consumer_gate(r, "apus_consumer_attach", CONS_STREAM) != APUS_OK) return APUS_ERROR;
    if (!out) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    StageLock sl(&r->cons_mu);
    if (resident_attach_check(r, RES_CONSUMER, stream) != APUS_OK) return APUS_ERROR;
    CK(cudaStreamSynchronize(r->cons_stream));           /* consume work enqueued before: its cursor is where we start */
    apus_consumer_view_t v;
    memset(&v, 0, sizeof v);
    view_log(r, &v);
    v.cur = reinterpret_cast<uint64_t *>(r->region + offsetof(apus_ctrl_t, cons_cur));
    v.error = &r->cons_st->error;
    v.status = const_cast<uint64_t *>(&r->hw_dev->cons_cursor);
    v.stop = const_cast<const uint64_t *>(&r->hw_dev->consumer_stop);
    v.stop_epoch = r->hw->consumer_stop;
    r->res[RES_CONSUMER] = resident_t{1, (cudaStream_t)stream};
    *out = v;
    return APUS_OK;
}

extern "C" int apus_consumer_detach(apus_replica_t *r)
{
    if (!r) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    if (!(r->cfg.flags & APUS_F_DEVICE_APPLY)) return resident_stop(r, RES_CONSUMER);   /* none attached, no cons_mu */
    StageLock sl(&r->cons_mu);
    return resident_stop(r, RES_CONSUMER);
}

/* ---- resident readers: an application's kernel runs read fences itself ---------------------------------------- */
/* the offsets a reader view carries are part of the ABI: a reader compiled against an older header reads the same words */
static_assert(APUS_REGION_CONS_REC == 896 && APUS_REGION_CONS_ON == 928 && APUS_REGION_SID == 1024,
              "the words a fence reads in another region keep their offsets");
static_assert(APUS_READER_SLOTS == sizeof(((apus_reader_block_t *)0)->busy) / 8 &&
              APUS_MAX_SERVER_COUNT == sizeof(((apus_reader_block_t *)0)->member) / 8, "the reader block's arrays");

extern "C" int apus_reader_attach(apus_replica_t *r, void *stream, apus_reader_view_t *out)
{
    if (consumer_gate(r, "apus_reader_attach", CONS_ANY_ROLE) != APUS_OK) return APUS_ERROR;
    if (!out) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    StageLock ll(&g_live_mu);                            /* connect and destroy change the member words under it */
    const int ipc = ipc_peer(r);                         /* (never with a reader attached: connect refuses it) */
    if (ipc >= 0)
        return fail("apus_reader_attach: peer %d is mapped through CUDA IPC (readers are for groups hosted in one "
                    "process)", ipc);
    if (resident_attach_check(r, RES_READER, stream) != APUS_OK) return APUS_ERROR;
    apus_reader_view_t v;
    memset(&v, 0, sizeof v);
    view_log(r, &v);
    v.role = const_cast<const uint64_t *>(&r->rb_dev->role);
    v.busy = const_cast<uint64_t *>(r->rb_dev->busy);
    v.member = const_cast<const uint64_t *>(r->rb_dev->member);
    v.n = r->cfg.group_size;
    v.own = r->cfg.server_idx;
    v.on_off = APUS_REGION_CONS_ON; v.rec_off = APUS_REGION_CONS_REC; v.sid_off = APUS_REGION_SID;
    v.release = const_cast<const uint64_t *>(&r->hw_dev->cons_wait_epoch);
    v.stop = const_cast<const uint64_t *>(&r->hw_dev->reader_stop);
    v.stop_epoch = r->hw->reader_stop;
    r->res[RES_READER] = resident_t{1, (cudaStream_t)stream};
    *out = v;
    return APUS_OK;
}

extern "C" int apus_reader_detach(apus_replica_t *r)
{
    if (!r) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    return resident_stop(r, RES_READER);
}

/* ---- resident submitters: an application's kernel writes the leader's HBM ring itself -------------------------- */
/* The hand-over of a leader's ring from the host to its attached, dormant submitter (attach on a leader, and the
 * first launch that runs a dormant one's replica as leader): everything the host has submitted reaches the ring and
 * the doorbell, then the accounting words and pay_end reach the submitter's state, then the term it holds the ring in,
 * and last the lock word, which the host has held since attach (APUS_SUBMITTER_HOST_HELD): each copy is complete
 * before the next begins, and the reserving thread's CAS acquires the lock only once it reads the host's 0
 * (include/apus_submitter.cuh).  While the host holds the lock no kernel thread holds it. */
static int submitter_hand_over(apus_replica *r)
{
    if (ring_flush(r) != APUS_OK) return APUS_ERROR;
    CK(cudaStreamSynchronize(r->copy_stream));
    apus_submitter_state_t s;
    memset(&s, 0, sizeof s);
    s.submitted = r->submitted; s.pay_head = r->pay_head; s.wrap_next = r->wrap_next ? 1 : 0;
    s.consumed = r->hw->consumed; s.lead_term = r->cfg.term;
    const size_t a = offsetof(apus_submitter_state_t, submitted), b = offsetof(apus_submitter_state_t, rejected);
    CK(cudaMemcpyAsync((char *)r->sub_st + a, (const char *)&s + a, b - a, cudaMemcpyHostToDevice, r->copy_stream));
    CK(cudaMemcpyAsync(r->sub_st + 1, r->pay_end, 8ull * r->ring_slots, cudaMemcpyHostToDevice, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    CK(cudaMemcpyAsync(&r->sub_st->lead_term, &s.lead_term, 8, cudaMemcpyHostToDevice, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    CK(cudaMemcpyAsync(&r->sub_st->lock, &s.lock, 8, cudaMemcpyHostToDevice, r->copy_stream));   /* the release: 0 */
    CK(cudaStreamSynchronize(r->copy_stream));
    r->sub_active = 1;
    return APUS_OK;
}

extern "C" int apus_submitter_attach(apus_replica_t *r, void *stream, apus_submitter_view_t *out)
{
    if (!r || !out) return fail("null argument");
    if (r->cfg.ring_mode != APUS_RING_DEVICE)
        return fail("apus_submitter_attach needs the device submission ring%s",
                    is_leader(r) ? "" : " (this is a follower on a host-mapped ring)");
    DeviceGuard g(r->cfg.device);
    if (resident_attach_check(r, RES_SUBMITTER, stream) != APUS_OK) return APUS_ERROR;
    if (leader_ring_init(r) != APUS_OK) return APUS_ERROR;      /* a follower's ring: the view's words exist from now */
    /* dormant, the lock held by the host, nothing reserved: no kernel of this submitter runs yet, so the whole state is
     * written */
    apus_submitter_state_t s;
    memset(&s, 0, sizeof s);
    s.lock = APUS_SUBMITTER_HOST_HELD; s.first_rejected = ~0ull; s.lead_term = APUS_SUBMITTER_DORMANT;
    CK(cudaMemcpyAsync(r->sub_st, &s, sizeof s, cudaMemcpyHostToDevice, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    if (is_leader(r) && submitter_hand_over(r) != APUS_OK) return APUS_ERROR;
    apus_submitter_view_t v;
    memset(&v, 0, sizeof v);
    v.slots = reinterpret_cast<uint8_t *>(r->ring_desc_dev);
    v.pay = r->ring_pay_dev;
    v.doorbell = r->sub_tail_dev;
    v.ring_slots = r->ring_slots; v.ring_bytes = r->ring_bytes;
    v.state = r->sub_st;
    v.pay_end = reinterpret_cast<uint64_t *>(r->sub_st + 1);
    v.consumed = const_cast<const uint64_t *>(&r->hw_dev->consumed);
    v.committed = const_cast<const uint64_t *>(&r->hw_dev->committed_tickets);
    v.stop = const_cast<const uint64_t *>(&r->hw_dev->submitter_stop);
    v.stop_epoch = r->hw->submitter_stop;
    r->res[RES_SUBMITTER] = resident_t{1, (cudaStream_t)stream};
    *out = v;
    return APUS_OK;
}

extern "C" int apus_submitter_detach(apus_replica_t *r)
{
    if (!r) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    if (resident_stop(r, RES_SUBMITTER) != APUS_OK) return APUS_ERROR;
    if (!r->sub_active) return APUS_OK;                  /* dormant: the host has kept the ring */
    r->sub_active = 0;
    /* hand the ring back: the doorbell P is what the leader may read; reservations past it are dropped */
    apus_submitter_state_t s;
    uint64_t P = 0;
    CK(cudaMemcpyAsync(&P, r->sub_tail_dev, 8, cudaMemcpyDeviceToHost, r->copy_stream));
    CK(cudaMemcpyAsync(&s, r->sub_st, sizeof s, cudaMemcpyDeviceToHost, r->copy_stream));
    CK(cudaMemcpyAsync(r->pay_end, r->sub_st + 1, 8ull * r->ring_slots, cudaMemcpyDeviceToHost, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    r->submitted = r->flushed = r->belled = P;
    r->pay_head = r->pay_flushed = P ? r->pay_end[(P - 1) & (r->ring_slots - 1)] : 0;
    r->wrap_next = 1;                                    /* a dropped reservation may have moved the payload counter */
    if (s.rejected) {
        if (!r->hw->dev_first_rejected) r->hw->dev_first_rejected = s.first_rejected;
        r->hw->dev_rejected += s.rejected;
    }
    return APUS_OK;
}

extern "C" uint64_t apus_leader_suspect(apus_replica_t *r) { return r ? r->hw->leader_suspect : 0; }
extern "C" uint64_t apus_last_commit_ns(apus_replica_t *r) { return r ? r->hw->last_commit_ns : 0; }

extern "C" int apus_get_stats(apus_replica_t *r, apus_stats_t *out)
{
    if (!r || !out) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    apus_ctrl_t c;
    CK(cudaMemcpyAsync(&c, r->region, sizeof c, cudaMemcpyDeviceToHost, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    memset(out, 0, sizeof *out);
    out->tickets_submitted = r->submitted;
    if (r->sub_active) {                                 /* the resident submitter's published tickets: the doorbell */
        CK(cudaMemcpyAsync(&out->tickets_submitted, r->sub_tail_dev, 8, cudaMemcpyDeviceToHost, r->copy_stream));
        CK(cudaStreamSynchronize(r->copy_stream));
    }
    out->tickets_consumed = c.consumed;
    out->tickets_committed = c.committed_tickets;
    out->entries_acked = c.acked;
    out->bytes_replicated = c.bytes_replicated;
    out->batches = c.batches;
    out->kernel_launches = r->launches;
    out->lat_samples = c.lat_count;
    out->auto_heads = c.auto_heads;
    /* published-but-uncommitted entries count too (`published` itself follows the commit) */
    out->entries_published = c.pub_seen > c.published ? c.pub_seen : c.published;
    for (int i = 0; i < 8; i++) { out->phase_ns[i] = c.phase_ns[i]; out->turn_ns[i] = c.turn_ns[i]; }
    return APUS_OK;
}

extern "C" int apus_latency_samples(apus_replica_t *r, uint32_t *dst, uint32_t max, uint32_t *n)
{
    if (!r || !dst || !n) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    apus_ctrl_t c;
    CK(cudaMemcpyAsync(&c, r->region, sizeof c, cudaMemcpyDeviceToHost, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    uint64_t have = c.lat_count < APUS_LAT_RING ? c.lat_count : APUS_LAT_RING;
    uint32_t take = (uint32_t)(have < max ? have : max);
    uint32_t *tmp = (uint32_t *)malloc(sizeof(uint32_t) * APUS_LAT_RING);
    if (!tmp) return fail("out of memory");
    cudaError_t e = cudaMemcpyAsync(tmp, r->d_lat, sizeof(uint32_t) * APUS_LAT_RING, cudaMemcpyDeviceToHost, r->copy_stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(r->copy_stream);
    if (e != cudaSuccess) { free(tmp); return fail("latency copy failed: %s", cudaGetErrorString(e)); }
    for (uint32_t k = 0; k < take; k++)
        dst[k] = tmp[(c.lat_count - take + k) & (APUS_LAT_RING - 1)];
    free(tmp);
    *n = take;
    return APUS_OK;
}



/* ==================================================================================================
 * Fabric mode: VMM regions + NVSwitch multicast (tools/probe_fabric checks that cuMulticast* is supported and
 * measures `multimem.st.v4`, which lands the source bytes in EVERY member -- the leader's egress for the replicate
 * step drops from (N-1)x to 1x).  The driver entry points are fetched at run time
 * (cudaGetDriverEntryPoint): the library keeps loading on a box without libcuda (CPU-only test runs).
 * This round: groups whose replicas live in ONE process (tests, sweeps, `bench.py --spread`); one process per
 * replica would pass the allocation and multicast handles as POSIX file descriptors (pidfd_getfd).
 * ================================================================================================== */
static int fabric_alloc_region(apus_replica *r)
{
    if (drv_load() != APUS_OK) return APUS_ERROR;
    int ndev = apus_device_count();
    CUmemAllocationProp ap;
    memset(&ap, 0, sizeof ap);
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ap.location.id = r->cfg.device;
    ap.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;     /* (as probed; also what one process per replica will export) */
    size_t gran = 0;
    CU(g_drv.MemGetAllocationGranularity(&gran, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    if (gran < (2u << 20)) gran = 2u << 20;
    r->vmm_bytes = (r->region_bytes + gran - 1) / gran * gran;
    CU(g_drv.MemCreate(&r->vmm_handle, r->vmm_bytes, &ap, 0));
    CUdeviceptr va = 0;
    CU(g_drv.MemAddressReserve(&va, r->vmm_bytes, gran, 0, 0));
    CU(g_drv.MemMap(va, r->vmm_bytes, 0, r->vmm_handle, 0));
    CUmemAccessDesc acc[64];
    for (int d = 0; d < ndev && d < 64; d++) { acc[d].location.type = CU_MEM_LOCATION_TYPE_DEVICE; acc[d].location.id = d; acc[d].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE; }
    CU(g_drv.MemSetAccess(va, r->vmm_bytes, acc, (size_t)(ndev < 64 ? ndev : 64)));       /* every GPU of the box may store here */
    r->region = (uint8_t *)va;
    return APUS_OK;
}

/* All replicas of ONE group, in this process, on pairwise different GPUs, created with APUS_F_FABRIC: bind their
 * regions to one multicast object and give the leader the multicast mapping.  From the next launch on the leader's
 * T5 step issues ONE `multimem.st` per 16 B chunk instead of one store per replica. */
extern "C" int apus_group_multicast(apus_replica_t **rs, int n)
{
    if (!rs || n < 2 || n > APUS_MAX_SERVER_COUNT) return fail("bad replica list");
    if (drv_load() != APUS_OK) return APUS_ERROR;
    apus_replica *lead = NULL;
    for (int i = 0; i < n; i++) {
        if (!rs[i] || !rs[i]->vmm_handle) return fail("replica %d was not created with APUS_F_FABRIC", i);
        if (rs[i]->in_flight) return fail("stop the kernels first");
        if (rs[i]->vmm_bytes != rs[0]->vmm_bytes) return fail("regions differ in size");
        for (int j = 0; j < i; j++) if (rs[j]->cfg.device == rs[i]->cfg.device) return fail("multicast needs one GPU per replica");
        int mc = 0;
        CU(g_drv.DeviceGetAttribute(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, rs[i]->cfg.device));
        if (!mc) return fail("device %d does not support multicast", rs[i]->cfg.device);
        if (is_leader(rs[i])) lead = rs[i];
    }
    if (!lead) return fail("no leader in the list");
    if (lead->mc_region) return APUS_OK;
    CUmulticastObjectProp mp;
    memset(&mp, 0, sizeof mp);
    mp.numDevices = (unsigned)n; mp.size = lead->vmm_bytes; mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t mgran = 0;
    CU(g_drv.MulticastGetGranularity(&mgran, &mp, CU_MULTICAST_GRANULARITY_MINIMUM));
    if (lead->vmm_bytes % mgran) return fail("region size %zu is not a multiple of the multicast granularity %zu", lead->vmm_bytes, mgran);
    CU(g_drv.MulticastCreate(&lead->mc_handle, &mp));
    for (int i = 0; i < n; i++) CU(g_drv.MulticastAddDevice(lead->mc_handle, rs[i]->cfg.device));
    for (int i = 0; i < n; i++) {
        DeviceGuard g(rs[i]->cfg.device);
        CU(g_drv.MulticastBindMem(lead->mc_handle, 0, rs[i]->vmm_handle, 0, rs[i]->vmm_bytes, 0));
    }
    DeviceGuard g(lead->cfg.device);
    CUdeviceptr va = 0;
    CU(g_drv.MemAddressReserve(&va, lead->vmm_bytes, mgran, 0, 0));
    CU(g_drv.MemMap(va, lead->vmm_bytes, 0, lead->mc_handle, 0));
    CUmemAccessDesc acc;
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE; acc.location.id = lead->cfg.device; acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    CU(g_drv.MemSetAccess(va, lead->vmm_bytes, &acc, 1));
    lead->mc_region = (uint8_t *)va;
    return APUS_OK;
}

/* ==================================================================================================
 * Control plane on NVLink words (SURVEY.md s8f N1).  Transport and log surgery only; the election policy
 * (dare_server.c:1264-1743) lives with the caller, apus_b200/csrc/dare_entry.c.
 * ================================================================================================== */
#define SID_TERM(s) ((s) >> 9)

static int own_read(apus_replica *r, size_t off, void *dst, size_t len)
{
    StageLock sl(&r->stage_mu);
    CK(cudaMemcpyAsync(r->stage, r->region + off, len, cudaMemcpyDeviceToHost, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    memcpy(dst, r->stage, len);
    return APUS_OK;
}
static int own_write(apus_replica *r, size_t off, const void *src, size_t len)
{
    StageLock sl(&r->stage_mu);
    memcpy(r->stage, src, len);
    CK(cudaMemcpyAsync(r->region + off, r->stage, len, cudaMemcpyHostToDevice, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    return APUS_OK;
}
/* a peer's region through the mapping the kernels store through (peer access or CUDA IPC): host-initiated copies */
static int peer_read(apus_replica *r, uint8_t peer, size_t off, void *dst, size_t len)
{
    StageLock sl(&r->stage_mu);
    if (!r->peer_ptr[peer]) return fail("peer %u is not connected", (unsigned)peer);
    CK(cudaMemcpyAsync(r->stage, (uint8_t *)r->peer_ptr[peer] + off, len, cudaMemcpyDefault, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    memcpy(dst, r->stage, len);
    return APUS_OK;
}
static int peer_write(apus_replica *r, uint8_t peer, size_t off, const void *src, size_t len)
{
    StageLock sl(&r->stage_mu);
    if (!r->peer_ptr[peer]) return fail("peer %u is not connected", (unsigned)peer);
    memcpy(r->stage, src, len);
    CK(cudaMemcpyAsync((uint8_t *)r->peer_ptr[peer] + off, r->stage, len, cudaMemcpyDefault, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    return APUS_OK;
}

extern "C" int apus_ctl_read(apus_replica_t *r, apus_ctl_view_t *out)
{
    if (!r || !out) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    apus_ctlwords_t w;
    if (own_read(r, APUS_CTL_OFF, &w, sizeof w) != APUS_OK) return APUS_ERROR;
    memset(out, 0, sizeof *out);
    out->sid = w.sid; out->leader_sid = w.leader_sid; out->adj_end = w.adj_end; out->adj_count = w.adj_count;
    for (int i = 0; i < APUS_MAX_SERVER_COUNT; i++) {
        out->vote_ack[i] = w.vote_ack[i];
        out->vote_req[i].sid = w.vote_req[i].sid; out->vote_req[i].index = w.vote_req[i].index;
        out->vote_req[i].term = w.vote_req[i].term;
        out->vote_req[i].cid[0] = w.vote_req[i].cid[0]; out->vote_req[i].cid[1] = w.vote_req[i].cid[1];
    }
    return APUS_OK;
}

extern "C" int apus_ctl_set_sid(apus_replica_t *r, uint64_t sid)
{
    if (!r) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    return own_write(r, APUS_CTL_OFF + offsetof(apus_ctlwords_t, sid), &sid, 8);
}

extern "C" int apus_ctl_reset_votes(apus_replica_t *r)
{
    if (!r) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    uint64_t v[16];
    for (int i = 0; i < 16; i++) v[i] = r->log_len;              /* dare_server.c:1300: vote_ack[i] = log->len */
    return own_write(r, APUS_CTL_OFF + offsetof(apus_ctlwords_t, vote_ack), v, sizeof v);
}

extern "C" int apus_ctl_clear_vote_request(apus_replica_t *r, uint8_t from_idx)
{
    if (!r || from_idx >= APUS_MAX_SERVER_COUNT) return fail("bad argument");
    DeviceGuard g(r->cfg.device);
    uint64_t z = 0;
    return own_write(r, APUS_CTL_OFF + offsetof(apus_ctlwords_t, vote_req) + sizeof(apus_vote_req_t) * from_idx, &z, 8);
}

extern "C" int apus_ctl_send_vote_request(apus_replica_t *r, uint8_t peer_idx, uint64_t sid, uint64_t index, uint64_t term,
                                          const void *cid16)
{
    if (!r || peer_idx >= r->cfg.group_size) return fail("bad argument");
    DeviceGuard g(r->cfg.device);
    apus_vote_req_t q;
    memset(&q, 0, sizeof q);
    q.index = index; q.term = term;
    if (cid16) memcpy(q.cid, cid16, 16);
    /* the sid word is what the voter polls: the rest of the record goes first */
    const size_t base = APUS_CTL_OFF + offsetof(apus_ctlwords_t, vote_req) + sizeof(apus_vote_req_t) * r->cfg.server_idx;
    if (peer_write(r, peer_idx, base + 8, (uint8_t *)&q + 8, sizeof q - 8) != APUS_OK) return APUS_ERROR;
    return peer_write(r, peer_idx, base, &sid, 8);
}

extern "C" int apus_ctl_send_vote_ack(apus_replica_t *r, uint8_t candidate_idx, uint64_t commit)
{
    if (!r || candidate_idx >= r->cfg.group_size) return fail("bad argument");
    DeviceGuard g(r->cfg.device);
    return peer_write(r, candidate_idx, APUS_CTL_OFF + offsetof(apus_ctlwords_t, vote_ack) + 8u * r->cfg.server_idx, &commit, 8);
}

/* the entry with cumulative number `cum` (== its idx: every entry ever appended is counted, idx starts at 1):
 * offset from the offset index, {idx, term} and stride from its header */
static int entry_at(apus_replica *r, int peer, uint64_t cum, uint64_t *off, uint64_t *idx, uint64_t *term, uint32_t *stride)
{
    uint32_t w = 0;
    const size_t ioff = APUS_INDEX_OFF + 4ull * (cum & (r->idx_cap - 1));
    int rc = peer < 0 ? own_read(r, ioff, &w, 4) : peer_read(r, (uint8_t)peer, ioff, &w, 4);
    if (rc != APUS_OK) return rc;
    const uint64_t o = w & ~APUS_IDX_HEAD_FLAG;
    if (o + APUS_HDR_BYTES > r->log_len) return fail("offset index names an offset beyond the log");
    uint8_t h[64];
    rc = peer < 0 ? own_read(r, r->entries_off + o, h, 64) : peer_read(r, (uint8_t)peer, r->entries_off + o, h, 64);
    if (rc != APUS_OK) return rc;
    memcpy(idx, h + E_IDX, 8); memcpy(term, h + E_TERM, 8);
    uint16_t len; memcpy(&len, h + E_DATA, 2);
    const uint8_t ty = h[E_TYPE];
    *stride = (ty == T_NOOP || ty == T_CONFIG || ty == T_HEAD) ? APUS_HDR_BYTES : APUS_HDR_BYTES + len;
    *off = o;
    return APUS_OK;
}

extern "C" int apus_ctl_heartbeat(apus_replica_t *r, uint64_t *word)
{
    if (!r || !word) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    return own_read(r, offsetof(apus_ctrl_t, hb), word, sizeof *word);
}

extern "C" int apus_ctl_last_entry(apus_replica_t *r, uint64_t *idx, uint64_t *term, uint64_t *commit, uint64_t *end)
{
    if (!r || !idx || !term) return fail("null argument");
    if (r->in_flight) return fail("the replica's kernel must be stopped (exclusive log access)");
    DeviceGuard g(r->cfg.device);
    apus_loghdr_t h; apus_ctrl_t c;
    if (own_read(r, APUS_HDR_OFF, &h, sizeof h) != APUS_OK || own_read(r, 0, &c, sizeof c) != APUS_OK) return APUS_ERROR;
    if (commit) *commit = h.commit;
    if (end) *end = h.end;
    const uint64_t count = is_leader(r) ? c.published : c.acked;
    *idx = 0; *term = 0;
    if (h.end == r->log_len || count == 0) return APUS_OK;            /* empty log */
    uint64_t off; uint32_t stride;
    if (entry_at(r, -1, count, &off, idx, term, &stride) != APUS_OK) return APUS_ERROR;
    if (*idx != count) return fail("entry counter %llu does not match the idx %llu of the last entry", (unsigned long long)count, (unsigned long long)*idx);
    return APUS_OK;
}

/* bytes from log offset `from` forward to `to` on a ring of L bytes */
static inline uint64_t ring_dist_h(uint64_t from, uint64_t to, uint64_t L) { return to >= from ? to - from : L - (from - to); }

static int copy_to_peer(apus_replica *r, uint8_t peer, size_t off, size_t len)
{
    if (!len) return APUS_OK;
    CK(cudaMemcpyAsync((uint8_t *)r->peer_ptr[peer] + off, r->region + off, len, cudaMemcpyDefault, r->copy_stream));
    return APUS_OK;
}

extern "C" int apus_consume_seed(apus_replica_t *r, uint64_t cursor_offset, uint64_t next_idx)
{
    if (consumer_gate(r, "apus_consume_seed", CONS_ANY_ROLE) != APUS_OK) return APUS_ERROR;
    if (is_leader(r)) return fail("apus_consume_seed: a leader's consumers stand on its own log");
    if (r->in_flight) return fail("apus_consume_seed: stop the kernel first");
    if (cursor_offset >= r->log_len || next_idx == 0)
        return fail("apus_consume_seed: cursor %llu outside the log of %llu B, or next idx 0", (unsigned long long)cursor_offset,
                    (unsigned long long)r->log_len);
    DeviceGuard g(r->cfg.device);
    StageLock cl(&r->cons_mu);
    apus_loghdr_t h; apus_ctrl_t c;
    if (own_read(r, APUS_HDR_OFF, &h, sizeof h) != APUS_OK || own_read(r, 0, &c, sizeof c) != APUS_OK) return APUS_ERROR;
    if (h.end != r->log_len || c.acked != 0) return fail("apus_consume_seed: the replica holds entries (its log must be empty)");
    if (r->cons_enqueued) return fail("apus_consume_seed: consume work has been enqueued on this replica");
    if (c.cons_cur[0] != 0 || c.cons_cur[1] != 1) return fail("apus_consume_seed: the consumers have moved");
    /* the record names the seed and nothing past it: no entry is held until the leader's adjustment resends them */
    c.cons_rec[0] = cursor_offset; c.cons_rec[1] = next_idx - 1;
    c.cons_cur[0] = cursor_offset; c.cons_cur[1] = next_idx;
    c.cons_seeded = 1;
    const size_t from = offsetof(apus_ctrl_t, cons_rec), to = offsetof(apus_ctrl_t, cons_seeded) + 8;
    if (own_write(r, from, (const uint8_t *)&c + from, to - from) != APUS_OK) return APUS_ERROR;
    r->hw->cons_cursor = cursor_offset;
    r->hw->cons_next_idx = next_idx;
    return APUS_OK;
}

/* the idx of the entry that starts at my head: my next idx when my log is empty or my head is my end, 0 when no entry
 * of mine starts there */
static int head_idx(apus_replica *r, const apus_loghdr_t &mh, uint64_t mine, uint64_t *hidx)
{
    *hidx = 0;
    if (mh.end == r->log_len || mh.head == mh.end) { *hidx = mine + 1; return APUS_OK; }
    uint8_t eh[8];
    uint64_t v, o, i2, t2; uint32_t s2;
    if (own_read(r, r->entries_off + mh.head + E_IDX, eh, 8) != APUS_OK) return APUS_ERROR;
    memcpy(&v, eh, 8);
    if (v == 0 || v > mine || entry_at(r, -1, v, &o, &i2, &t2, &s2) != APUS_OK || o != mh.head || i2 != v) return APUS_OK;
    *hidx = v;
    return APUS_OK;
}

/* Whether {cur, nidx} inside [head, commit] of my log is a position my consumers can stand at: the one the consume tail
 * kernel leaves behind entry nidx - 1, its end (0 for an entry that ends at the ring's end).  So entry nidx starts at
 * cur; or entry nidx starts at 0 behind a wrap gap that begins at cur, where entry nidx - 1 ends; or no entry past cur
 * is committed: cur is my commit offset and nidx is one past my committed entries. */
static int consumer_boundary(apus_replica *r, uint64_t cur, uint64_t nidx, uint64_t commit, uint64_t committed, bool *ok)
{
    *ok = false;
    if (cur == commit && nidx == committed + 1) { *ok = true; return APUS_OK; }
    if (nidx > committed) return APUS_OK;
    uint64_t o, i, t; uint32_t s;
    if (entry_at(r, -1, nidx, &o, &i, &t, &s) != APUS_OK) return APUS_ERROR;
    if (i != nidx) return APUS_OK;
    if (o == cur) { *ok = true; return APUS_OK; }
    if (o != 0 || nidx < 2) return APUS_OK;
    if (entry_at(r, -1, nidx - 1, &o, &i, &t, &s) != APUS_OK) return APUS_ERROR;
    *ok = i == nidx - 1 && o + s == cur;
    return APUS_OK;
}

extern "C" int apus_ctl_adjust_follower(apus_replica_t *r, uint8_t peer, uint64_t sid, uint64_t *resent)
{
    if (!r || peer >= r->cfg.group_size || peer == r->cfg.server_idx) return fail("bad argument");
    if (!is_leader(r)) return fail("log adjustment is the leader's job");
    if (r->in_flight) return fail("the leader's kernel must be stopped");
    if (!r->peer_ptr[peer]) return fail("peer %u is not connected", (unsigned)peer);
    DeviceGuard g(r->cfg.device);
    const uint64_t L = r->log_len;
    apus_loghdr_t mh, fh; apus_ctrl_t mc, fc;
    if (own_read(r, APUS_HDR_OFF, &mh, sizeof mh) != APUS_OK || own_read(r, 0, &mc, sizeof mc) != APUS_OK) return APUS_ERROR;
    if (peer_read(r, peer, APUS_HDR_OFF, &fh, sizeof fh) != APUS_OK || peer_read(r, peer, 0, &fc, sizeof fc) != APUS_OK) return APUS_ERROR;
    if (fc.cons_on == 1) return fail("peer %u consumes on the device (APUS_F_DEVICE_APPLY): no log adjustment", (unsigned)peer);
    const uint64_t mine = mc.published, theirs = fc.acked;      /* idx of the last entry each of us holds */
    /* last entry we share: walk down from min(mine, theirs) comparing {offset, idx, term} (the leader's log is the
     * truth, log_find_remote_end_offset, dare_log.h:362-394).  Entries up to the follower's commit are shared by
     * construction (they are committed), so the walk ends there at the latest. */
    uint64_t j = mine < theirs ? mine : theirs;
    uint64_t keep_end = (mh.end == L) ? L : 0;                   /* offset right behind the last shared entry */
    bool found = false;
    while (j > 0) {
        uint64_t o1, i1, t1, o2, i2, t2; uint32_t s1, s2;
        if (entry_at(r, -1, j, &o1, &i1, &t1, &s1) != APUS_OK || entry_at(r, peer, j, &o2, &i2, &t2, &s2) != APUS_OK) return APUS_ERROR;
        if (o1 == o2 && i1 == i2 && t1 == t2 && i1 == j) { keep_end = o1 + s1; if (keep_end == L) keep_end = 0; found = true; break; }
        j--;
    }
    if (!found) { j = 0; keep_end = 0; }
    /* a peer whose device consumers run in any role (cons_on == 2): nothing they have read, or may read on their
     * current record, is rewritten -- checked before anything is written */
    uint64_t rec[2] = { fc.cons_rec[0], fc.cons_rec[1] };
    bool rewrite_rec = false, seeded = false;
    const uint64_t cur = fc.cons_cur[0], nidx = fc.cons_cur[1];
    if (fc.cons_on) {
        if (j > 0) {
            if (nidx - 1 > j || ring_dist_h(cur, rec[0], L) > ring_dist_h(cur, keep_end, L))
                return fail("peer %u: its device consumers have read, or may read, past the last entry it shares with me "
                            "(idx %llu, next idx %llu): no log adjustment", (unsigned)peer, (unsigned long long)j,
                            (unsigned long long)nidx);
            /* entries past what it holds after the resend have stale index words: the record may not name them */
            if (rec[1] > mine) { rec[1] = mine; rewrite_rec = true; }
        } else if (fc.cons_seeded && fh.end == L && fc.acked == 0) {
            /* a replacement whose consumers were seeded at the mark of a snapshot of some consumer's state
             * (apus_consume_seed): it goes on from there if that position is one of my consumer positions in
             * [head, commit].  A mark behind my head belongs to a snapshot older than my live log: take a newer one */
            uint64_t hidx;
            if (head_idx(r, mh, mine, &hidx) != APUS_OK) return APUS_ERROR;
            if (nidx < hidx) {
                snprintf(g_err, sizeof g_err, "peer %u was seeded at next idx %llu, behind my head (idx %llu): its snapshot "
                         "is older than my log, seed it from a newer one", (unsigned)peer, (unsigned long long)nidx,
                         (unsigned long long)hidx);
                return APUS_RETRY;
            }
            if (nidx > mc.committed + 1 || ring_dist_h(mh.head, cur, L) > ring_dist_h(mh.head, mh.commit, L))
                return fail("peer %u was seeded at offset %llu, next idx %llu, past my commit (offset %llu, %llu entries) "
                            "or outside my log: no log adjustment", (unsigned)peer, (unsigned long long)cur,
                            (unsigned long long)nidx, (unsigned long long)mh.commit, (unsigned long long)mc.committed);
            bool ok;
            if (consumer_boundary(r, cur, nidx, mh.commit, mc.committed, &ok) != APUS_OK) return APUS_ERROR;
            if (!ok)
                return fail("peer %u was seeded at offset %llu, next idx %llu: no consumer of my log stands there (entry "
                            "%llu does not start there, nor behind a wrap gap there): no log adjustment", (unsigned)peer,
                            (unsigned long long)cur, (unsigned long long)nidx, (unsigned long long)nidx);
            rec[0] = cur; rec[1] = nidx - 1; rewrite_rec = true; seeded = true;
        } else {
            /* it shares nothing with me and was not seeded: its consumers can go on only from my head */
            uint64_t hidx;
            if (head_idx(r, mh, mine, &hidx) != APUS_OK) return APUS_ERROR;
            if (cur != mh.head || nidx != hidx)
                return fail("peer %u shares no entry with me and its device consumers stand at offset %llu, next idx %llu, "
                            "not at my head (offset %llu, idx %llu): no log adjustment", (unsigned)peer,
                            (unsigned long long)cur, (unsigned long long)nidx, (unsigned long long)mh.head,
                            (unsigned long long)hidx);
            rec[0] = cur; rec[1] = nidx - 1; rewrite_rec = true;                /* nothing of its old log */
        }
    }
    /* the record first, so that no consume call that runs during the resend trusts the old one (one 16 B copy) */
    if (rewrite_rec && peer_write(r, peer, offsetof(apus_ctrl_t, cons_rec), rec, 16) != APUS_OK) return APUS_ERROR;
    uint64_t bytes = 0;
    if (mine > j && mh.end != L) {
        /* everything behind the shared prefix: entry bytes [keep_end, my end) -- a wrapped range is two copies, a wrap
         * gap (ghost header) travels with it -- and the offset-index words of entries j+1 .. mine */
        const uint64_t from = (j == 0) ? mh.head : keep_end;
        const uint64_t to = mh.end;
        if (to > from) { if (copy_to_peer(r, peer, r->entries_off + from, to - from) != APUS_OK) return APUS_ERROR; bytes += to - from; }
        else if (to < from || (to == from && mine > j)) {
            if (copy_to_peer(r, peer, r->entries_off + from, L - from) != APUS_OK) return APUS_ERROR;
            if (copy_to_peer(r, peer, r->entries_off, to) != APUS_OK) return APUS_ERROR;
            bytes += L - from + to;
        }
        const uint64_t cap = r->idx_cap, a = (j + 1) & (cap - 1), n = mine - j;
        if (n >= cap) { if (copy_to_peer(r, peer, APUS_INDEX_OFF, 4ull * cap) != APUS_OK) return APUS_ERROR; }
        else if (a + n <= cap) { if (copy_to_peer(r, peer, APUS_INDEX_OFF + 4ull * a, 4ull * n) != APUS_OK) return APUS_ERROR; }
        else {
            if (copy_to_peer(r, peer, APUS_INDEX_OFF + 4ull * a, 4ull * (cap - a)) != APUS_OK) return APUS_ERROR;
            if (copy_to_peer(r, peer, APUS_INDEX_OFF, 4ull * (a + n - cap)) != APUS_OK) return APUS_ERROR;
        }
        CK(cudaStreamSynchronize(r->copy_stream));
    }
    /* the follower now holds exactly my log: set its end (LR_SET_END, dare_ibv_rc.c:1396-1412) and its entry counter,
     * count it as holding everything I hold, then tell it whom to follow */
    if (j == 0) {
        /* a follower that shares nothing with me (a joiner, dare_ibv_rc.c:478-856 recover_log): it starts from my head,
         * and knows my commit offset right away */
        if (peer_write(r, peer, APUS_HDR_OFF + offsetof(apus_loghdr_t, head), &mh.head, 8) != APUS_OK) return APUS_ERROR;
        if (peer_write(r, peer, APUS_HDR_OFF + offsetof(apus_loghdr_t, commit), &mh.commit, 8) != APUS_OK) return APUS_ERROR;
    }
    const uint64_t endw[2] = { mh.end, mh.end };
    if (peer_write(r, peer, APUS_HDR_OFF + offsetof(apus_loghdr_t, end), &endw[0], 8) != APUS_OK) return APUS_ERROR;
    if (peer_write(r, peer, APUS_HDR_OFF + offsetof(apus_loghdr_t, old_end), &endw[1], 8) != APUS_OK) return APUS_ERROR;
    if (peer_write(r, peer, offsetof(apus_ctrl_t, acked), &mine, 8) != APUS_OK) return APUS_ERROR;
    const uint64_t none = L;
    if (peer_write(r, peer, offsetof(apus_ctrl_t, pend_head_end), &none, 8) != APUS_OK) return APUS_ERROR;
    /* my commit offset as a commit publish of my term: the follower's kernel follows it as far as it holds entries */
    const uint64_t pc[2] = { mh.commit, r->cfg.term };
    if (peer_write(r, peer, offsetof(apus_ctrl_t, pub_commit), pc, 16) != APUS_OK) return APUS_ERROR;
    if (own_write(r, offsetof(apus_ctrl_t, ack) + 8u * peer, &mine, 8) != APUS_OK) return APUS_ERROR;
    /* a seeded replacement's apply offset is its seed: the word still holds the lost replica's, which the pruning rule
     * would read until the replacement's kernel reports its own */
    if (seeded && own_write(r, offsetof(apus_ctrl_t, apply_off) + 8u * peer, &cur, 8) != APUS_OK) return APUS_ERROR;
    const uint64_t adj[3] = { sid, mh.end, mine };
    if (peer_write(r, peer, APUS_CTL_OFF + offsetof(apus_ctlwords_t, adj_end), &adj[1], 16) != APUS_OK) return APUS_ERROR;
    if (peer_write(r, peer, APUS_CTL_OFF + offsetof(apus_ctlwords_t, leader_sid), &adj[0], 8) != APUS_OK) return APUS_ERROR;
    if (resent) *resent = bytes;
    return APUS_OK;
}

extern "C" int apus_follower_beats(apus_replica_t *r, uint64_t out[APUS_MAX_SERVER_COUNT])
{
    if (!r || !out) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    uint64_t b[16];
    if (own_read(r, offsetof(apus_ctrl_t, fbeat), b, sizeof b) != APUS_OK) return APUS_ERROR;
    for (int i = 0; i < APUS_MAX_SERVER_COUNT; i++) out[i] = b[i];
    return APUS_OK;
}

extern "C" int apus_replica_disconnect(apus_replica_t *r, uint8_t peer_idx)
{
    if (!r || peer_idx >= APUS_MAX_SERVER_COUNT) return fail("bad argument");
    if (r->in_flight) return fail("stop the kernel first");
    /* the mapping itself is left alone (closing a handle whose exporter died is not worth the risk): nothing stores there
     * any more, and no resident fence reads there once this returns */
    if (peer_idx != r->cfg.server_idx) {
        StageLock ll(&g_live_mu);
        r->peer_ptr[peer_idx] = NULL;
        reader_forget(r, peer_idx);
    }
    return APUS_OK;
}

extern "C" int apus_replica_set_role(apus_replica_t *r, uint8_t leader_idx, uint64_t term)
{
    if (!r || leader_idx >= r->cfg.group_size) return fail("bad argument");
    if (r->sub_active)
        return fail("apus_replica_set_role: a resident submitter holds this replica's ring (apus_submitter_detach "
                    "first): an active submitter does not step down");
    if ((r->cfg.flags & APUS_F_DEVICE_APPLY) && !(r->cfg.flags & APUS_F_APPLY_ANY_ROLE))
        return fail("a replica with device consumers (APUS_F_DEVICE_APPLY) keeps its role");
    if (r->in_flight) return fail("stop the kernel first");
    DeviceGuard g(r->cfg.device);
    const bool was_leader = is_leader(r);
    r->cfg.leader_idx = leader_idx;
    r->cfg.term = term;
    /* a resident fence takes t and L from here; the take-over's release below comes after this store */
    r->rb->role = role_sid(r);
    __sync_synchronize();
    if (!is_leader(r)) {
        if (!r->peer_ptr[leader_idx]) return fail("not connected to the new leader");
        /* the leader's adjustment already set end / old_end / the entry counter (and, for a joiner, head and commit):
         * what the host sees as "committed and held" starts there, not at a stale or never-written word */
        apus_loghdr_t h;
        if (own_read(r, APUS_HDR_OFF, &h, sizeof h) != APUS_OK) return APUS_ERROR;
        r->hw->commit_off = h.commit;
        return APUS_OK;
    }
    if (was_leader) return APUS_OK;
    /* ---- a follower takes the log over as it holds it ---- */
    if (leader_ring_init(r) != APUS_OK) return APUS_ERROR;
    r->submitted = r->flushed = r->belled = 0; r->pay_head = r->pay_flushed = 0;
    r->hw->sub_tail = 0; r->hw->consumed = 0; r->hw->committed_tickets = 0;
    if (r->cfg.ring_mode == APUS_RING_DEVICE) {
        /* the device doorbell too: a replica that led before left its last value there, and the kernel does not poll
         * the stamps of a device ring.  An attached submitter is dormant here; the hand-over writes its state */
        *r->sub_tail_stage = 0;
        CK(cudaMemcpyAsync(r->sub_tail_dev, r->sub_tail_stage, 8, cudaMemcpyHostToDevice, r->copy_stream));
        CK(cudaStreamSynchronize(r->copy_stream));
    }
    apus_loghdr_t h; apus_ctrl_t c;
    if (own_read(r, APUS_HDR_OFF, &h, sizeof h) != APUS_OK || own_read(r, 0, &c, sizeof c) != APUS_OK) return APUS_ERROR;
    const uint64_t L = r->log_len, last = c.acked;
    /* adopt the largest commit offset my voters granted me (poll_vote_count, dare_server.c:1356-1362): the old leader's
     * commit pushes reach its followers at different times, so a voter may know of more committed entries than I do.
     * Every follower is then told this commit, so none of them runs ahead of mine.  Only offsets in (commit, end] by
     * ring order from my head are taken: `log_len` means "no vote", and a word left from an earlier election that lies
     * outside what I hold cannot be a commit of this log. */
    if (h.end != L) {
        uint64_t va[16];
        if (own_read(r, APUS_CTL_OFF + offsetof(apus_ctlwords_t, vote_ack), va, sizeof va) != APUS_OK) return APUS_ERROR;
        const uint64_t pe = (h.end + L - h.head) % L;
        uint64_t pc = (h.commit + L - h.head) % L;
        for (int i = 0; i < 16; i++) {
            if (i == r->cfg.server_idx || va[i] >= L) continue;
            const uint64_t pv = (va[i] + L - h.head) % L;
            if (pv > pc && pv <= pe) { pc = pv; h.commit = va[i]; }
        }
        r->hw->commit_off = h.commit;    /* what the host sees as committed until my kernel's first commit store */
    }
    /* entries between my commit offset and my end are published but not committed: count them by walking the offset
     * index backwards until an entry starts at or before the commit offset */
    uint64_t unc = 0, tail = L;
    if (h.end != L && last) {
        uint64_t off, idx, tm; uint32_t st;
        if (entry_at(r, -1, last, &off, &idx, &tm, &st) != APUS_OK) return APUS_ERROR;
        tail = off;
        uint64_t jj = last;
        const uint64_t dist_commit = (h.end >= h.commit) ? h.end - h.commit : L - (h.commit - h.end);
        while (jj > 0) {
            if (entry_at(r, -1, jj, &off, &idx, &tm, &st) != APUS_OK) return APUS_ERROR;
            const uint64_t d = (h.end >= off) ? h.end - off : L - (off - h.end);     /* bytes from this entry to my end */
            if (d > dist_commit || dist_commit == 0) break;
            unc++; jj--;
            if (unc > (1u << 20)) return fail("too many uncommitted entries to take over");
        }
    }
    c.next_idx = last + 1; c.published = last; c.pub_seen = last; c.committed = last - unc;
    c.consumed = 0; c.committed_tickets = 0;
    c.hwm = L;                       /* treat every range as written before: prefill reads the log (zeros where it was never written) */
    for (int i = 0; i < 16; i++) { c.ack[i] = 0; c.apply_off[i] = h.head; c.fbeat[i] = 0; }   /* dare_server.c:1507-1510 */
    h.tail = tail; h.old_end = h.end;
    if (own_write(r, 0, &c, offsetof(apus_ctrl_t, fin_entries)) != APUS_OK) return APUS_ERROR;
    if (r->cfg.flags & APUS_F_APPLY_ANY_ROLE) {
        /* my device consumers go on as a leader's: the record names what I now know committed -- the adopted commit
         * and the entries before it -- and my apply offset is their cursor (the commit warp keeps it so).  The consume
         * work enqueued so far runs to its end first, so that none of it sees the record change under it, and none
         * is enqueued meanwhile */
        consume_wait_release(r);                 /* a pending wait would hold the drain for its whole timeout */
        StageLock cl(&r->cons_mu);
        CK(cudaStreamSynchronize(r->cons_stream));
        const uint64_t rec[2] = { h.commit, last - unc };
        if (own_read(r, offsetof(apus_ctrl_t, cons_cur), &h.apply, 8) != APUS_OK) return APUS_ERROR;
        if (own_write(r, offsetof(apus_ctrl_t, cons_rec), rec, 16) != APUS_OK) return APUS_ERROR;
    }
    if (own_write(r, APUS_HDR_OFF, &h, sizeof h) != APUS_OK) return APUS_ERROR;
    return APUS_OK;
}

extern "C" int apus_set_head(apus_replica_t *r, uint64_t head)
{
    if (!r) return fail("null argument");
    if (head >= r->log_len) return fail("head beyond the log");
    DeviceGuard g(r->cfg.device);
    static __thread uint64_t stage;
    stage = head;
    CK(cudaMemcpyAsync(r->region + APUS_HDR_OFF + offsetof(apus_loghdr_t, head), &stage, 8,
                       cudaMemcpyHostToDevice, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    return APUS_OK;
}

extern "C" int apus_remote_apply_offsets(apus_replica_t *r, uint64_t out[APUS_MAX_SERVER_COUNT])
{
    if (!r || !out) return fail("null argument");
    DeviceGuard g(r->cfg.device);
    apus_ctrl_t c;
    CK(cudaMemcpyAsync(&c, r->region, sizeof c, cudaMemcpyDeviceToHost, r->copy_stream));
    CK(cudaStreamSynchronize(r->copy_stream));
    for (int i = 0; i < APUS_MAX_SERVER_COUNT; i++) out[i] = c.apply_off[i];
    return APUS_OK;
}
