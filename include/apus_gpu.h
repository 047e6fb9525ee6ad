/*
 * apus_gpu.h -- C ABI of the H100-native Paxos log-replication engine.
 *
 * This is the drop-in boundary for the ONE hot path of hku-systems/apus that this
 * repository accelerates (SURVEY.md s8): leader append -> replicate to every
 * follower -> majority ack -> commit.  It replaces the "lower" callee set the
 * reference's consensus thread calls into,
 *     src/include/dare/dare_ibv.h:141-201  (dare_ib_poll_tailq,
 *     dare_ib_write_remote_logs, dare_ib_send_entries_reply, ...) implemented by
 *     src/dare/dare_ibv_rc.c (RC queue pairs, RDMA WRITE/READ) and
 *     src/dare/dare_ibv_ud.c:780-790 (get_tailq_message),
 * together with the log placement of src/include/dare/dare_log.h.
 * Plain C types only: pointers, sizes, integers.  No CUDA or torch types.
 *
 * Each replica of a Paxos group is one `apus_replica_t`, bound to one GPU; its
 * consensus log (reference layout, byte for byte) and its ack / tail / commit
 * words live in that GPU's HBM.  The leader's hot loop and the followers' ack
 * loops are persistent sm_90a kernels (apus_b200/csrc/apus_kernels.cu); peers
 * are reached with P2P stores over NVLink (same process: peer access; one
 * process per replica: CUDA IPC handles exchanged with apus_replica_export /
 * apus_replica_connect -- the analogue of the raddr/rkey exchange in RC_SYN,
 * src/dare/dare_ibv_ud.c:1116-1119).
 *
 * The reference-facing "engine entry" symbols that src/proxy/proxy.c links
 * against (dare_server_init, is_leader, get_node_id, the tailhead queue) are
 * declared in apus_dare_entry.h and implemented on top of this ABI.
 *
 * Error convention follows the reference transport (dare_ibv_rc.c:27-29):
 * 0 = success, 1 = error, -1 = "retry later"; apus_last_error() gives the text.
 * There is NO CPU fallback: every entry point fails with 1 when no CUDA device
 * is usable.
 */
#ifndef APUS_GPU_H
#define APUS_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define APUS_ABI_VERSION 2

#define APUS_OK       0
#define APUS_ERROR    1
#define APUS_RETRY  (-1)

#define APUS_MAX_SERVER_COUNT 13            /* dare.h:26 */
#define APUS_LOG_SIZE (16384ull * 4096ull)  /* dare_log.h:76 LOG_SIZE */
#define APUS_ENTRY_HDR 64u                  /* sizeof(dare_log_entry_t) */

/* entry types: dare_log.h:21-24 and proxy.h:9-11 */
#define APUS_NOOP    0
#define APUS_CSM     1
#define APUS_CONFIG  2
#define APUS_HEAD    3
#define APUS_CONNECT 4
#define APUS_SEND    5
#define APUS_CLOSE   6

/* where the leader's submission ring lives */
#define APUS_RING_HOST_MAPPED 0   /* pinned host memory, read by the kernel over PCIe */
#define APUS_RING_DEVICE      1   /* HBM; the host fills it with cudaMemcpyAsync batches, or a kernel does
                                     (apus_submit_synth, apus_submit_device) */

/* apus_config_t.flags */
#define APUS_F_FENCED_ACK   0x1u  /* follower: reply bytes visible before the ack word; off = ack as soon as
                                     the tail publish is observed, reply bytes follow (default off) */
#define APUS_F_DEVICE_STATS 0x2u  /* leader: record per-batch device-side commit latency */
#define APUS_F_AUTOPRUNE    0x4u  /* leader: device-side log pruning (force_log_pruning rule,
                                     dare_server.c:2069-2122): when the ring is a quarter full the
                                     kernel appends a HEAD entry carrying min(apply offsets) */
#define APUS_F_FOLLOWER_WALK 0x8u /* follower: find entry boundaries by walking the byte stream
                                     (log_get_entry/log_entry_len, as the reference follower does)
                                     instead of reading the leader-written offset index */
#define APUS_F_HOST_APPLY   0x10u /* follower: the apply offset reported to the leader's pruning rule is the one the
                                     HOST has replayed (apus_set_applied), as apply_committed_entries advances
                                     log->apply only after do_action (dare_server.c:1939-1962); off = apply follows
                                     commit on the device (nothing replays the log on the host) */
#define APUS_F_NO_EXPRESS   0x20u /* leader: no single-warp express path, every publish is fenced (A/B switch) */
#define APUS_F_FABRIC      0x100u /* the replica's HBM region is a VMM allocation that apus_group_multicast() can bind to an
                                     NVSwitch multicast object (replicas of one process, one GPU each) */
#define APUS_F_PROFILE      0x40u /* fine-grained device timestamps in the latency path (diagnostic runs only: each is a %globaltimer read) */
#define APUS_F_DEVICE_APPLY 0x200u /* follower: the apply offset reported to the leader's pruning rule is the cursor of
                                     the device consumers (apus_consume_device), the device counterpart of
                                     APUS_F_HOST_APPLY.  Refused together with APUS_F_HOST_APPLY and on a leader
                                     (unless APUS_F_APPLY_ANY_ROLE is set too) */
#define APUS_F_APPLY_ANY_ROLE 0x400u /* with APUS_F_DEVICE_APPLY (refused without it): the device consumers work in
                                     every role, so that a group that applies in GPU memory keeps its failover.  On a
                                     leader they deliver every committed entry of its log, its own tickets included --
                                     every replica applies the same rows in the same order -- and their cursor is the
                                     leader's own apply offset in the pruning rule (a slow consumer holds the leader
                                     back instead of being overwritten).  apus_replica_set_role changes such a
                                     replica's role in both directions, and apus_ctl_adjust_follower adjusts it as long
                                     as nothing its consumers have read is rewritten */
#define APUS_F_EXPLICIT     0x80000000u /* flags are exactly as given (no defaults OR-ed in) */

typedef struct apus_replica apus_replica_t;

typedef struct apus_config {
    uint32_t struct_size;      /* sizeof(apus_config_t), for ABI growth */
    int32_t  device;           /* CUDA device ordinal hosting this replica */
    uint8_t  server_idx;       /* env server_idx (proxy.c:33-36) */
    uint8_t  group_size;       /* env group_size (proxy.c:37-40); 1..13 */
    uint8_t  leader_idx;       /* who leads in `term` (static until the control plane lands) */
    uint8_t  ring_mode;        /* APUS_RING_* (leader only) */
    uint32_t flags;            /* APUS_F_* */
    uint64_t term;             /* SID term stamped into entries (dare_server.h:53-61) */
    uint64_t log_size;         /* bytes of entries[]; 0 -> APUS_LOG_SIZE (reference) */
    uint32_t ring_slots;       /* submission descriptors, power of two; 0 -> default */
    uint32_t ring_bytes;       /* payload ring bytes, multiple of 4096; 0 -> default */
    uint32_t leader_ctas;      /* leader: worker CTAs (SMs) building tiles in parallel; 0 -> default */
    uint32_t reserved;
    /* ---- ABI 2 (struct_size tells which fields exist) ---- */
    uint32_t hb_period_us;     /* leader: heartbeat period, microseconds (hb_period of the config file,
                                  dare_server.c:763-791); 0 = no heartbeats */
    uint32_t hb_timeout_us;    /* follower: silence after which the leader is suspected (hb_timeout); 0 = never */
} apus_config_t;
#define APUS_CONFIG_SIZE_V1 48u

/* Opaque blob a replica publishes so that peers can map its HBM region.
 * Same process: carries the pointer; other process: a cudaIpcMemHandle_t. */
typedef struct apus_peer_handle {
    uint8_t bytes[128];
} apus_peer_handle_t;

/* the offsets of dare_log_t (dare_log.h:77-103) as this replica holds them */
typedef struct apus_log_offsets {
    uint64_t head, apply, commit, end, tail, old_end, old_commit, len;
} apus_log_offsets_t;

typedef struct apus_stats {
    uint64_t tickets_submitted;   /* requests accepted by apus_submit* */
    uint64_t tickets_consumed;    /* appended to the leader log by the kernel */
    uint64_t tickets_committed;   /* committed (majority acked), in log order */
    uint64_t entries_acked;       /* follower: entries acked to the leader */
    uint64_t bytes_replicated;    /* leader: sum over followers of entry bytes stored */
    uint64_t batches;             /* leader: replicate steps (tail publishes) */
    uint64_t kernel_launches;     /* launches of apus kernels that included this replica */
    uint64_t lat_samples;         /* device-side latency samples available */
    uint64_t auto_heads;          /* leader: HEAD entries appended by the device-side pruning rule */
    uint64_t entries_published;   /* leader: entries appended (tickets + auto HEAD entries) */
    uint64_t phase_ns[8];         /* leader profiling: ns waiting for requests, in T1..T6, and tile count */
    uint64_t turn_ns[8];          /* worker 0: [0..2] ns waiting for the claim lock / place turn / publish turn,
                                     [3] fast placements, [4] slow placements, [7] ns holding the place turn */
} apus_stats_t;

/* ---- library ------------------------------------------------------------------- */
int         apus_abi_version(void);
const char *apus_last_error(void);
int         apus_device_count(void);
/* NUMA node of the host memory next to a GPU, -1 if unknown: run the submitting threads (and allocate) there */
int         apus_device_numa_node(int device);

/* ---- replica life cycle --------------------------------------------------------- */
/* Allocates the HBM region (log header + entries + ctrl words), zeroed like
 * log_new() (dare_log.h:120-137: end = tail = old_end = len). */
int  apus_replica_create(const apus_config_t *cfg, apus_replica_t **out);
void apus_replica_destroy(apus_replica_t *r);

/* replaces the RC_SYN/SYNACK exchange of raddr+rkey (dare_ibv_ud.c:1116-1119) */
int  apus_replica_export(apus_replica_t *r, apus_peer_handle_t *out);
int  apus_replica_connect(apus_replica_t *r, uint8_t peer_idx, const apus_peer_handle_t *peer);

/* Replicas of ONE group, hosted by this process on pairwise different GPUs and created with APUS_F_FABRIC: bind their
 * regions to an NVSwitch multicast object.  The leader's replicate step then issues one `multimem.st` per 16 B chunk
 * (the switch fans it out to every replica, the leader's own copy included) instead of one store per replica. */
int  apus_group_multicast(apus_replica_t **rs, int n);

/* Launch the persistent kernel(s) for `n` replicas that live on the SAME device
 * in ONE fused launch (one CTA group per replica role).  The kernels return when
 * the cumulative ticket target is reached -- leader: that many requests committed;
 * follower: that many entries acked and applied -- or when apus_replicas_stop()
 * is called.  target_tickets == UINT64_MAX runs until stopped (service mode).
 * A leader with a dormant resident submitter hands its ring over to it first
 * (apus_submitter_attach): the host's submissions so far come before the
 * submitter's first ticket, and the host paths are refused from then on.
 * Asynchronous: returns after the launch. */
int  apus_replicas_launch(apus_replica_t **rs, int n, uint64_t target_tickets);
/* Wait for the launch that included `r` to finish; timeout_ms < 0 waits forever.
 * APUS_RETRY on timeout. */
int  apus_replica_wait(apus_replica_t *r, int64_t timeout_ms);
/* device time of the last finished launch that included r, in milliseconds (CUDA events) */
int  apus_replica_last_launch_ms(apus_replica_t *r, float *ms);
int  apus_replicas_stop(apus_replica_t **rs, int n);

/* ---- leader admission: the fields of tailq_entry_t (message.h:11-17) ------------- */
/* One request; `cmd` has `len` bytes (sm_cmd_t.cmd).  For APUS_CONFIG pass the
 * 16-byte dare_cid_t, for APUS_HEAD the 8-byte head offset, for APUS_NOOP nothing.
 * *ticket (optional) receives the 1-based position in the leader's append order.
 * APUS_RETRY when the submission ring is full. */
int  apus_submit(apus_replica_t *leader, uint8_t type, uint16_t connection_id, uint64_t req_id,
                 const void *cmd, uint16_t len, uint64_t *ticket);
/* n requests; payload k is payloads + k*stride (len[k] bytes).  conn/req arrays of n. */
int  apus_submit_batch(apus_replica_t *leader, uint32_t n, const uint8_t *types,
                       const uint16_t *connection_ids, const uint64_t *req_ids,
                       const uint16_t *lens, const void *payloads, size_t stride,
                       uint64_t *first_ticket);
/* n requests of ONE shape (type, connection, len; req_id = first_req_id + k; payload k at payloads + k*stride):
 * the bulk form of proxy.c:108-161's enqueue, filled by several host threads (env apus_submit_threads, default 8). */
int  apus_submit_uniform(apus_replica_t *leader, uint32_t n, uint8_t type, uint16_t connection_id,
                         uint64_t first_req_id, uint16_t len, const void *payloads, size_t stride,
                         uint64_t *first_ticket);
/* Device-generated requests (APUS_RING_DEVICE only): a fill kernel writes n SEND-like requests straight into the
 * HBM submission ring -- payload byte k of request req_id is apus_synth_byte(seed, req_id, k) -- so that a
 * benchmark can have its whole input resident in HBM without a host copy (SURVEY.md s8d, H6). */
int  apus_submit_synth(apus_replica_t *leader, uint32_t n, uint8_t type, uint16_t connection_id,
                       uint64_t first_req_id, uint16_t len, uint32_t seed, uint64_t *first_ticket);
uint8_t apus_synth_byte(uint32_t seed, uint64_t req_id, uint32_t k);
/* Requests in device memory (APUS_RING_DEVICE only), packed into the HBM submission ring by a kernel in stream order.
 * The five arrays are device memory on the leader's GPU; payload k is at payloads + k*stride (payloads may be NULL
 * when stride is 0).  `stream` is a cudaStream_t (NULL = the legacy default stream).  Returns once the work is
 * enqueued, without synchronising the host:
 *   - tickets are decided here: *first_ticket .. *first_ticket + n - 1, in log order like every other submit;
 *   - the payload ring reserves the worst case, n * round16(2 + stride) bytes (nothing when 2 + stride <= 80), and
 *     frees it when the whole batch has been consumed;
 *   - the packing runs after everything enqueued on `stream` before the call, and `stream` waits for the packing, so
 *     the arrays may be overwritten or freed in stream order as soon as the call returns;
 *   - host submissions that follow are ordered behind the packing, so their own synchronisation now also waits for
 *     whatever the caller's stream ran before the batch;
 *   - unless apus_submit_defer is on, the doorbell is raised to *first_ticket + n - 1 after the packing.
 * A request whose type is not CSM, CONNECT, SEND or CLOSE, or whose len exceeds stride, is written as the NOOP that
 * apus_submit(APUS_NOOP, conn, req_id, NULL, 0) would write at its ticket, and counted (apus_device_submit_status).
 * APUS_RETRY, with nothing reserved, when the slot ring or the payload ring has no room now; APUS_ERROR on a follower,
 * without a device ring, for a null array, or for a batch that could never fit (n > ring_slots, or a reservation
 * larger than ring_bytes). */
int  apus_submit_device(apus_replica_t *leader, uint32_t n, const uint8_t *types, const uint16_t *connection_ids,
                        const uint64_t *req_ids, const uint16_t *lens, const void *payloads, size_t stride,
                        void *stream, uint64_t *first_ticket);
/* Requests in device memory in the packed (jagged) layout: request k's cmd is values[offsets[k], offsets[k + 1]),
 * as in torch's jagged layout (values + offsets[n + 1]); offsets[0] need not be 0, so a slice of a larger buffer may be
 * passed.  The arrays are device memory on the leader's GPU; offsets and req_ids must be 8 B aligned, connection_ids
 * 2 B, values may have any alignment (and be NULL when values_bytes is 0).  Stream order, tickets, the doorbell, the
 * rejection of a type that is not CSM, CONNECT, SEND or CLOSE, APUS_RETRY and APUS_ERROR: as apus_submit_device, except:
 *   - the payload ring reserves min(n * round16(2 + 65535), round16(values_bytes + 17 n)) bytes (slot_packed_reserve),
 *     decided from n and values_bytes alone: pass only the slice of values the batch uses;
 *   - a cmd longer than 65535 B is written as a NOOP and counted;
 *   - if any offsets[k] > offsets[k + 1], or offsets[n] > values_bytes, EVERY request of the batch is written as a NOOP
 *     and counted: nothing is read outside values[0, values_bytes) and nothing written outside the reservation.
 * The packing reads offsets in more than one pass: they, like the other arrays, must not change until `stream` has
 * passed the call (a caller that rewrites them outside stream order races with the packing). */
int  apus_submit_device_packed(apus_replica_t *leader, uint32_t n, const uint8_t *types,
                               const uint16_t *connection_ids, const uint64_t *req_ids, const uint64_t *offsets,
                               const void *values, uint64_t values_bytes, void *stream, uint64_t *first_ticket);
/* requests of device batches rejected so far (written as NOOPs) and the ticket of the first of them (0 = none); a
 * batch is counted once its packing has run (e.g. after synchronising the stream it was submitted on) */
int  apus_device_submit_status(apus_replica_t *leader, uint64_t *rejected, uint64_t *first_rejected_ticket);
/* make everything submitted so far visible to the kernel (doorbell); apus_submit*
 * ring it themselves unless the replica was put in deferred mode */
int  apus_submit_defer(apus_replica_t *leader, int defer);
int  apus_submit_flush(apus_replica_t *leader);
/* ring the doorbell only up to `ticket` (<= submitted): requests beyond it stay resident but unseen */
int  apus_submit_release(apus_replica_t *leader, uint64_t ticket);

/* ---- commit observation (what update_state / do_action hang off) ---------------- */
uint64_t apus_committed_tickets(apus_replica_t *leader);
/* No CUDA call, just the pinned words the kernels keep up to date.  Leader: *offset = commit
 * offset, *count = tickets committed.  Follower: *offset = apply offset (everything before it
 * is committed and held by this replica -- what apply_committed_entries walks,
 * dare_server.c:1815-1974), *count = entries acked. */
int  apus_progress(apus_replica_t *r, uint64_t *offset, uint64_t *count);
/* spin until ticket is committed; APUS_RETRY on timeout */
int  apus_wait_committed(apus_replica_t *leader, uint64_t ticket, int64_t timeout_us);
/* Make `stream` (a cudaStream_t on the leader's GPU) wait, without the host, until `ticket` is committed: one
 * cuStreamWaitValue64 (>=) on the committed-tickets word the commit warp keeps in pinned, mapped memory.  Needs
 * CU_DEVICE_ATTRIBUTE_CAN_USE_64_BIT_STREAM_MEM_OPS (APUS_ERROR without it; there is no spin-kernel fallback).  A wait
 * on a ticket that never commits while the replica lives stays pending.  apus_replica_destroy releases pending waits
 * before it frees the word: it stops the kernels, raises the word to at least every ticket waited on and waits for the
 * streams to pass their waits.  The word cannot tell such a release from a commit; the caller knows it destroyed the
 * replica. */
int  apus_stream_wait_committed(apus_replica_t *leader, uint64_t ticket, void *stream);
/* device-visible address of that word (tickets committed; pinned and mapped, so the same address works in host and
 * device code), for kernels that look at the commit count themselves */
const volatile uint64_t *apus_committed_word(apus_replica_t *leader);

/* n requests of payload_len bytes, ONE in flight at a time: submit, spin until committed
 * (what a proxy thread does, proxy.c:108-161); lat_ns[i] = host-clock nanoseconds of request i */
int  apus_closed_loop(apus_replica_t *leader, uint32_t n, uint16_t payload_len, uint16_t connection_id,
                      uint64_t first_req_id, uint32_t *lat_ns);

/* ---- inspection (parity tests, snapshots) --------------------------------------- */
int  apus_log_offsets(apus_replica_t *r, apus_log_offsets_t *out);
/* copy entries[off, off+len) of this replica's log image to host memory */
int  apus_log_read(apus_replica_t *r, uint64_t off, uint64_t len, void *dst);
int  apus_get_stats(apus_replica_t *r, apus_stats_t *out);
/* device-side commit latencies (ns), newest `max` samples; returns count in *n */
int  apus_latency_samples(apus_replica_t *r, uint32_t *dst_ns, uint32_t max, uint32_t *n);

/* follower, APUS_F_HOST_APPLY: the application has replayed the log up to `offset` (do_action done) */
int  apus_set_applied(apus_replica_t *r, uint64_t offset);
/* copy the committed-and-held range [from, to) of the circular log (it may wrap) into dst (capacity cap);
 * *got = bytes copied.  One or two device->host copies through a pinned buffer. */
int  apus_log_read_range(apus_replica_t *r, uint64_t from, uint64_t to, void *dst, uint64_t cap, uint64_t *got);
/* Follower, APUS_F_DEVICE_APPLY (any role with APUS_F_APPLY_ANY_ROLE): deliver committed entries straight into device
 * memory, in stream order.  The arrays are device memory on the replica's GPU, element types as apus_submit_device's
 * plus idx; row k's cmd goes to
 * payloads + k*stride (payloads may be NULL when stride is 0).  `stream` is a cudaStream_t (NULL = the legacy default
 * stream).  Returns once the work is enqueued, without synchronising the host:
 *   - the work runs after everything enqueued on `stream` before the call, and `stream` waits for it; every call on
 *     one replica runs on one engine-owned stream, so calls run in call order whatever streams they come from;
 *   - it examines the next committed entries from the consumer cursor on, at most max_n of them, and writes the
 *     CSM-like ones (CSM, CONNECT, SEND, CLOSE: what do_action replays) as consecutive rows: idx, type, clt_id,
 *     req_id, cmd length and the cmd bytes (bytes of a row beyond its length are left untouched).  NOOP, CONFIG and
 *     HEAD entries are skipped; the idx of the rows shows them.  *count receives the number of rows;
 *   - the examination stops before the first CSM-like entry whose cmd exceeds `stride` (apus_consume_status tells the
 *     stride it needs: nothing is truncated or lost) and before an entry that does not carry the idx its index word
 *     promises (APUS_CONSUME_BAD_IDX, sticky: nothing more is delivered);
 *   - the cursor moves past every examined entry only after every read of their bytes has completed: the leader may
 *     prune, then overwrite, everything behind it (the follower's kernel reports it on its idle passes; a leader's
 *     commit warp takes it as its own apply offset on its idle passes);
 *   - on a leader (APUS_F_APPLY_ANY_ROLE) the rows are every committed entry of its log, its own tickets and the
 *     entries of earlier terms it took over alike: the same rows, in the same order, as every follower's.
 * It never waits for commits: it delivers what is committed when it runs, which may be nothing (apus_consume_wait,
 * enqueued before it, waits in stream order until enough is committed).  APUS_ERROR on a
 * leader without APUS_F_APPLY_ANY_ROLE, on a replica without APUS_F_DEVICE_APPLY, for a null array, for an array not
 * aligned to its element size
 * (idx and req_ids 8 B, count 4 B, connection_ids and lens 2 B; payloads may have any alignment), or for max_n == 0. */
int  apus_consume_device(apus_replica_t *follower, uint32_t max_n, uint64_t *idx, uint8_t *types,
                         uint16_t *connection_ids, uint64_t *req_ids, uint16_t *lens, void *payloads, size_t stride,
                         uint32_t *count, void *stream);
/* apus_consume_device with packed output: row r's cmd goes to values + offsets[r], contiguous and unpadded, with
 * offsets[0] = 0 and offsets[r + 1] = offsets[r] + its length for the *count rows written (offsets has max_n + 1
 * words; neither offsets past *count nor bytes of values past offsets[*count] are written).  Everything else as
 * apus_consume_device, except the stop: the examination stops just before the first CSM-like entry whose cmd would end
 * past values_cap.  When that entry would be the call's first row, apus_consume_status's need_stride reports its length
 * (a buffer of at least that many bytes delivers it); a stop after rows were delivered is not an error, the next call
 * continues there.  idx, req_ids and offsets must be 8 B aligned, count 4 B, connection_ids 2 B; values may have any
 * alignment (and be NULL when values_cap is 0). */
int  apus_consume_device_packed(apus_replica_t *follower, uint32_t max_n, uint64_t *idx, uint8_t *types,
                                uint16_t *connection_ids, uint64_t *req_ids, uint64_t *offsets, void *values,
                                uint64_t values_cap, uint32_t *count, void *stream);
#define APUS_CONSUME_BAD_IDX 1   /* an entry at an index word does not carry the expected idx */
/* the pinned words the consume work writes: the cursor and the idx of the next entry after the latest call that ran,
 * the stride the entry that stopped it needs (0 = it did not stop on a long entry), APUS_CONSUME_* (0 = none) */
int  apus_consume_status(apus_replica_t *follower, uint64_t *cursor_offset, uint64_t *next_idx, uint64_t *need_stride,
                         uint64_t *error);
/* outcomes of apus_consume_wait */
#define APUS_WAIT_READY      0u  /* at least min_entries committed entries lie past the consumer's cursor */
#define APUS_WAIT_TIMED_OUT  1u
#define APUS_WAIT_RELEASED   2u  /* ended by apus_consume_wait_release, apus_replicas_stop, apus_replica_set_role or destroy
                                    (of this replica, or of a peer it maps while it has a read fence pending) */
/* Make the consumers wait, in stream order and without the host, until at least min_entries committed entries lie past
 * the consumer's cursor (entries, not rows: NOOP, CONFIG and HEAD entries count), so that an application can enqueue
 * wait -> consume -> its own apply kernel many times ahead and synchronise only when it wants to.  Accepted in the roles
 * the consume calls accept.  `stream` is a cudaStream_t (NULL = the legacy default stream):
 *   - the wait runs on the engine-owned consume stream, in call order with every consume call on this replica; it runs
 *     after everything enqueued on `stream` before the call, and `stream` waits for it.  So a consume call of
 *     max_n >= min_entries made after a READY wait examines at least min_entries entries, unless it stops on a long cmd
 *     or on capacity as it always does;
 *   - the wait ends on whichever comes first: ready; a release (apus_consume_wait_release, apus_replicas_stop,
 *     apus_replica_set_role when a follower takes over, apus_replica_destroy: each ends every wait enqueued before it,
 *     none enqueued after it; the destroy of a peer this replica maps too, while a read fence is pending here); or
 *     timeout_us, counted from when the wait begins to run on the stream;
 *   - it then writes its APUS_WAIT_* outcome to `outcome` (optional: a 4 B-aligned device word on the replica's GPU, for
 *     device code downstream to branch on) and to the status words (apus_consume_wait_status);
 *   - a consumer stopped for good by APUS_CONSUME_BAD_IDX gets no outcome of its own: its wait ends as the counts say,
 *     and the consume after it delivers nothing and reports the error.
 * A pending wait occupies the hardware queue of the consume stream until it ends: work of other streams that shares
 * that queue (CUDA_DEVICE_MAX_CONNECTIONS) waits behind it, and if that work is what commits the entries (a leader's
 * device batches on the same GPU), the wait runs to its timeout.  APUS_ERROR, with nothing enqueued, where the consume
 * calls refuse the replica, for min_entries 0 or above the index ring's capacity, for timeout_us 0 or above 60 s, and
 * for an `outcome` not aligned to 4 B. */
int  apus_consume_wait(apus_replica_t *r, uint32_t min_entries, uint32_t timeout_us, uint32_t *outcome, void *stream);
/* end every consume wait enqueued on this replica before the call (they report APUS_WAIT_RELEASED); later waits are
 * not affected.  Returns without waiting for them to end. */
int  apus_consume_wait_release(apus_replica_t *r);
/* the pinned words the latest consume wait that ran wrote: its APUS_WAIT_* outcome (UINT64_MAX before any wait has
 * run) and the committed entries past the cursor when it ended */
int  apus_consume_wait_status(apus_replica_t *r, uint64_t *outcome, uint64_t *available);
/* Snapshots of device consumers: what replaces a lost replica of a group that applies in GPU memory.  The application
 * owns its state and copies it (device to device, CUDA IPC, or through the host); the engine names the log position
 * that state corresponds to, and starts a replacement's consumers there.
 * apus_consume_mark writes the consumer position {cursor offset, idx of the next entry}, as the consume calls enqueued
 * before it left it, into `mark`: 16 B of device memory on the replica's GPU, 16 B aligned.  `stream` is a cudaStream_t
 * (NULL = the legacy default stream), ordered exactly as for apus_consume_wait: the mark runs on the consume stream in
 * call order with the consume calls, after everything enqueued on `stream` before the call, and `stream` waits for it.
 * So a copy of the state enqueued on `stream` right behind the mark is the state at the marked position, and the group
 * keeps running while it is taken.  A consumer stopped for good by APUS_CONSUME_BAD_IDX marks next idx 0, which no seed
 * accepts.  The mark writes nothing the replica kernels read.  APUS_ERROR, with nothing enqueued, where the consume
 * calls refuse the replica and for a null or misaligned `mark`. */
int  apus_consume_mark(apus_replica_t *r, uint64_t *mark, void *stream);
/* Start the consumers of a replacement at a mark: cursor and next idx := the mark, and the consumer record names
 * nothing held past it (apus_consume_status reports the seed at once).  The leader's apus_ctl_adjust_follower then
 * accepts this replica, although it shares no entry, if the mark is a consumer position of the leader's log between its
 * head and its commit: the offset where entry next_idx starts, or where the wrap gap before it starts, or the commit
 * offset with next_idx one past the committed entries.  The adjustment resends the live log, and the leader counts the
 * seed as the replacement's apply offset in its pruning rule until the replacement's kernel reports its own; it returns
 * APUS_RETRY, with nothing written, for a mark behind the leader's head (the snapshot is older than the live log: take a
 * newer one), and APUS_ERROR, with nothing written, for a mark past its commit or at no consumer position.  APUS_ERROR,
 * with nothing written, unless the replica was created with APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE, is a follower
 * whose kernel is stopped, holds no entry (empty log, nothing acked), has had no consume call, wait or mark enqueued,
 * and unless cursor_offset < the log size and next_idx >= 1. */
int  apus_consume_seed(apus_replica_t *r, uint64_t cursor_offset, uint64_t next_idx);
/* outcome of apus_read_fence besides the three above: the leader this replica knew could not be confirmed -- a majority
 * of the group's SIDs carries a newer term, the leader is not connected, or it publishes no current consumer record */
#define APUS_WAIT_NOT_LEADER 3u  /* a fence's outcome only: apus_consume_wait never ends with it */
/* Read fences: linearizable reads from any replica's device state (Raft's read index, section 6.4), for a group that
 * applies in GPU memory on every replica (APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE).  Let t and L be the term and the
 * leader this replica knew when the fence was enqueued, N the group size.  The fence, in stream order:
 *   1. takes K, the entries-committed word of L's consumer record (L's commit warp publishes it only under
 *      APUS_F_APPLY_ANY_ROLE: no such record ends NOT_LEADER);
 *   2. after that, reads the SID of every member this replica maps, itself included, and ends NOT_LEADER unless at
 *      least N/2 + 1 of them are at term <= t.  This relies on the control plane moving a voter's SID to the
 *      candidate's term BEFORE it acks the vote, as dare_entry.c's elect does: a control plane that acks votes without
 *      moving the SID gets no guarantee from a fence;
 *   3. waits until this replica holds committed entries through K, and the last of them carries a term >= t (a new
 *      leader's commit may lag what an earlier leader committed until its blank CONFIG commits), then ends READY with
 *      the read index F := the entries committed and held here.
 * What F covers: every entry that L's consumer record named before the fence began to run (and every entry of an
 * earlier term committed before then, through the own-term entry), and this replica holds the committed entries through
 * F.  L's commit warp makes each commit advance visible elsewhere first: it stores the commit into every follower and
 * the committed-tickets word (apus_committed_tickets, apus_wait_committed, apus_stream_wait_committed) a few stores
 * before the consumer record, and for longer if L's context is descheduled in between.  A fence that begins in that
 * window may end READY with F below a write whose commit was already seen that way.  For read-your-writes, the
 * application compares F with its write's idx (rows carry idx and req_id) and enqueues another fence while F is short:
 * the record follows within the same commit advance.  A consume call enqueued after a READY fence delivers through F
 * (given a max_n that reaches it, and unless it stops on a long cmd or on capacity as it always may), and a state that
 * has applied through F answers a read that is linearizable with respect to the commits L's record has published: the
 * application compares its applied idx, which the rows carry, with F in its own read kernel.  A group that has
 * committed nothing yet keeps a fence waiting.
 * Runs exactly as apus_consume_wait does: on the consume stream under the same lock, in call order with the consume
 * calls, waits and marks, after everything enqueued on `stream` (a cudaStream_t, NULL = the legacy default stream)
 * before the call, and `stream` waits for it; it ends RELEASED at the same release points, TIMED_OUT after timeout_us
 * from when it begins to run.  It then writes F to `index` (an 8 B-aligned device word on the replica's GPU; READY only,
 * untouched otherwise), the outcome to `outcome` (optional, 4 B aligned) and both to the status words.
 * Fences read other replicas' regions, so they are for groups hosted in one process: apus_replica_destroy(p) first
 * unmaps p from every replica of the process that maps it (as apus_replica_disconnect would; a fence enqueued later
 * counts p as not connected), and on each of them that has a fence pending it ends the consume waits and fences
 * (APUS_WAIT_RELEASED) and waits for that fence.  APUS_ERROR, with nothing enqueued, for a replica without
 * APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE, a timeout_us of 0 or above 60 s, a null or misaligned `index`, a
 * misaligned `outcome`, and a replica that maps any peer through CUDA IPC. */
int  apus_read_fence(apus_replica_t *r, uint32_t timeout_us, uint64_t *index, uint32_t *outcome, void *stream);
/* the pinned words the latest fence that ran wrote: its outcome (UINT64_MAX before any fence has run) and its read
 * index (0 unless it ended READY) */
int  apus_read_fence_status(apus_replica_t *r, uint64_t *outcome, uint64_t *index);
/* Resident consumers: an application's own persistent kernel applies committed entries in place, from the log, beside
 * the replica kernels (include/apus_consumer.cuh is its device API).  The view holds the device addresses that API
 * needs; the application passes it to its kernel by value. */
typedef struct apus_consumer_view {
    const uint8_t  *entries;      /* the log ring (device memory) ... */
    uint64_t        log_len;      /* ... and its length in bytes */
    const uint32_t *index;        /* the offset index: the offset of entry idx is index[idx & idx_mask] (high bit: HEAD) */
    uint32_t        idx_mask;
    uint32_t        pad;
    const uint64_t *rec;          /* consumer record {committed-and-held offset, entries held}: 16 B, acquired */
    uint64_t       *cur;          /* cursor {offset, idx of the next entry}: 16 B, stored with a release */
    uint64_t       *error;        /* sticky APUS_CONSUME_BAD_IDX of the consume state (device memory) */
    uint64_t       *status;       /* the pinned words apus_consume_status reads: cursor, next idx, need_stride, error */
    const uint64_t *stop;         /* pinned stop word: the consumer ends once it no longer holds stop_epoch */
    uint64_t        stop_epoch;
} apus_consumer_view_t;
/* Attach a resident consumer to a replica the consume calls accept (APUS_F_DEVICE_APPLY on a follower; any role with
 * APUS_F_APPLY_ANY_ROLE).  It synchronises the consume stream, so that consume work enqueued before it has run and the
 * cursor stands where that work left it, then fills *out.  `stream` (a cudaStream_t on the replica's GPU, NULL = the
 * legacy default stream) is the stream the application launches its consumer kernel on.  While attached:
 *   - the resident consumer alone moves the cursor: apus_consume_device*, apus_consume_wait and apus_consume_mark
 *     return APUS_ERROR with nothing enqueued (apus_read_fence stays accepted; it never moves the cursor);
 *   - apus_replicas_stop, apus_replica_set_role and the release points of consume waits do not stop it: it keeps
 *     polling its record through a take-over;
 *   - a snapshot takes the position from apus_consumer_position in the application's own kernel, at a point where its
 *     state is consistent; apus_consume_seed accepts it as it accepts a mark.
 * APUS_ERROR where the consume calls refuse the replica, for a null `out`, and when a consumer is attached already. */
int  apus_consumer_attach(apus_replica_t *r, void *stream, apus_consumer_view_t *out);
/* Ask the resident consumer to end (its stop word moves) and synchronise the stream it was attached with.  Consume
 * calls, waits and marks are accepted again and continue from the cursor it left.  APUS_ERROR when none is attached.
 * apus_replica_destroy does the same for an attached replica before it frees anything: a consumer kernel that ignored
 * the stop word would keep both calls waiting. */
int  apus_consumer_detach(apus_replica_t *r);
/* Resident submitters: an application's own persistent kernel, on the leader's GPU, reserves tickets, writes slots and
 * payload images straight into the leader's HBM submission ring and rings the doorbell, without a host call
 * (include/apus_submitter.cuh is its device API; the slot format is include/apus_slot_format.h).  The submitter's state
 * lives in device memory: reservations take tickets and payload space in one order under its lock. */
typedef struct apus_submitter_state {
    uint64_t lock;                /* 0 = free; taken with a CAS by the reserving thread; APUS_SUBMITTER_HOST_HELD while
                                     dormant: the host holds it, and releases it last in the hand-over */
    uint64_t submitted;           /* tickets handed out (reserved) so far */
    uint64_t pay_head;            /* payload bytes handed out so far (monotone; position = % ring_bytes) */
    uint64_t wrap_next;           /* 1: the next external image carries APUS_SLOT_WRAP */
    uint64_t consumed;            /* the leader's consumed tickets as last read over PCIe (a lower bound) */
    uint64_t rejected;            /* requests written as NOOPs ... */
    uint64_t first_rejected;      /* ... and the lowest ticket among them (UINT64_MAX = none) */
    uint64_t lead_term;           /* the term the submitter holds the ring in (APUS_SUBMITTER_DORMANT until then) */
} apus_submitter_state_t;
#define APUS_SUBMITTER_HOST_HELD 2ull
#define APUS_SUBMITTER_DORMANT (~0ull)
typedef struct apus_submitter_view {
    uint8_t        *slots;        /* the leader's HBM slot ring: ring_slots slots of 128 B (apus_slot_t) */
    uint8_t        *pay;          /* ... and its payload ring of ring_bytes bytes */
    uint64_t       *doorbell;     /* the device doorbell the leader kernel reads: tickets readable so far */
    uint32_t        ring_slots;   /* power of two */
    uint32_t        ring_bytes;
    apus_submitter_state_t *state;
    uint64_t       *pay_end;      /* [ticket % ring_slots]: the payload counter after that ticket (device memory) */
    const uint64_t *consumed;     /* pinned: tickets the leader kernel has taken from the ring */
    const uint64_t *committed;    /* pinned: tickets committed (the word apus_committed_word gives) */
    const uint64_t *stop;         /* pinned stop word: the submitter ends once it no longer holds stop_epoch */
    uint64_t        stop_epoch;
} apus_submitter_view_t;
/* Attach a resident submitter to a replica created with APUS_RING_DEVICE, leader or follower, and fill *out.  `stream`
 * (a cudaStream_t on the replica's GPU, NULL = the legacy default stream) is the stream the application launches its
 * submitter on.  Attach allocates the replica's submission ring if it has none yet, so that the view stays valid through
 * any number of take-overs.  A submitter is dormant or active:
 *   - on a follower it starts dormant: apus_submitter_reserve returns APUS_SUBMITTER_NOT_LEADER at once and writes
 *     nothing, apus_replica_set_role is accepted, and the host paths behave as with no submitter attached (a winner
 *     submits its blank CONFIG through them before its first launch);
 *   - it becomes active by the hand-over: everything the host has submitted is pushed and rung, the ring accounting
 *     (tickets handed out, the payload counter, pay_end of the unconsumed tickets) is copied into its device state,
 *     and then the term it holds the ring in.  On a leader attach makes the hand-over; a dormant submitter gets it from
 *     the first apus_replicas_launch that runs its replica as leader, before that launch.
 * While active:
 *   - the submitter alone writes the ring: apus_submit, apus_submit_batch, _uniform, _synth, _device, _device_packed,
 *     apus_submit_defer, _flush, _release and apus_closed_loop return APUS_ERROR with nothing written;
 *   - apus_replica_set_role on this replica returns APUS_ERROR: an active submitter does not step down (detach first;
 *     the replica may attach again once it follows, dormant; include/apus_submitter.cuh says why);
 *   - apus_replicas_stop leaves it attached: its reservations and commit waits then end at their timeouts;
 *   - reads stay accepted: apus_committed_tickets, apus_wait_committed, apus_stream_wait_committed, apus_get_stats
 *     (tickets_submitted counts the published device tickets) and apus_device_submit_status (which counts the requests
 *     the submitter wrote as NOOPs).
 * APUS_ERROR for a null replica or `out`, on a host-mapped ring (leader or follower), for a stream of another device,
 * and when a submitter is attached already. */
int  apus_submitter_attach(apus_replica_t *leader, void *stream, apus_submitter_view_t *out);
/* Ask the resident submitter to end (its stop word moves), synchronise the stream it was attached with, and, if it is
 * active, hand the ring back to the host: what was published -- the doorbell P -- becomes the host's count of submitted tickets, the
 * payload counter becomes the one after ticket P, and the next host image carries APUS_SLOT_WRAP.  Reservations past P
 * were never visible to the leader: they are dropped, and the host hands their ticket numbers out again (P + 1 is the
 * next ticket).  A dropped reservation's requests that were written as NOOPs stay counted.  A dormant submitter hands
 * nothing back.  apus_replica_destroy does the same stop before it frees anything.  APUS_ERROR when none is attached. */
int  apus_submitter_detach(apus_replica_t *leader);
/* Resident readers: read fences that an application's own persistent kernel runs, with no host call per fence
 * (include/apus_reader.cuh is its device API).  What a stream fence takes from the host when it is enqueued -- the term
 * and leader, the peers' regions -- the reader reads from a pinned block the host keeps current: `role` holds the SID
 * this replica knows (term << 9 | 1 << 8 | leader idx: one 8 B word, so that no fence sees a torn pair), `member[i]` the
 * region of member i as this replica maps it (its own at its own index; 0 = not connected), and `busy[s]` is the
 * sequence word of fencing slot s, odd while a fence of that slot reads other replicas' regions.  A fence runs in one
 * slot at a time: fences that run at once use distinct slots. */
#define APUS_READER_SLOTS 32
typedef struct apus_reader_view {
    const uint8_t  *entries;      /* this replica's log ring (device memory) ... */
    uint64_t        log_len;      /* ... and its length in bytes */
    const uint32_t *index;        /* the offset index (apus_consumer_view_t.index) */
    uint32_t        idx_mask;
    uint32_t        pad;
    const uint64_t *rec;          /* this replica's consumer record {committed-and-held offset, entries held} */
    const uint64_t *role;         /* pinned: the SID this replica knows (see above) */
    uint64_t       *busy;         /* pinned: APUS_READER_SLOTS sequence words */
    const uint64_t *member;       /* pinned: APUS_MAX_SERVER_COUNT region addresses */
    uint32_t        n;            /* the group size */
    uint32_t        own;          /* this replica's index */
    uint32_t        on_off;       /* byte offsets inside a region: the consumer flag (2 = a record in every role), */
    uint32_t        rec_off;      /* ... the consumer record */
    uint32_t        sid_off;      /* ... and the SID word */
    uint32_t        pad2;
    const uint64_t *release;      /* pinned: the release epoch of consume waits and fences */
    const uint64_t *stop;         /* pinned stop word: the reader ends once it no longer holds stop_epoch */
    uint64_t        stop_epoch;
} apus_reader_view_t;
/* Attach a resident reader to a replica that stream fences accept (APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE) and fill
 * *out.  `stream` (a cudaStream_t on the replica's GPU, NULL = the legacy default stream) is the stream the application
 * launches its reader kernel on.  A resident fence has the contract of apus_read_fence, except that t and L are what the
 * role word holds when the fence begins, and that the reader's stop word ends it RELEASED too; it ends RELEASED at the
 * release points of stream fences (apus_consume_wait_release, apus_replicas_stop, a take-over's apus_replica_set_role,
 * destroy) and writes nothing to the status words apus_read_fence_status reads.  While attached:
 *   - apus_replica_connect of a peer of another process (CUDA IPC) returns APUS_ERROR;
 *   - stream fences, the consume calls and a resident consumer stay accepted: a reader never moves the cursor;
 *   - apus_replica_set_role, stops and wait releases leave it attached, and set_role rewrites the role word first;
 *   - apus_replica_disconnect and the destroy of a peer clear the peer's member word, then wait until no fence that
 *     may have read the old word is still reading that peer's region.
 * APUS_ERROR, with nothing written, where apus_read_fence refuses the replica, for a null `out`, a replica that maps a
 * peer through CUDA IPC, a stream of another device, and when a reader is attached already. */
int  apus_reader_attach(apus_replica_t *r, void *stream, apus_reader_view_t *out);
/* Ask the resident reader to end (its stop word moves) and synchronise the stream it was attached with.
 * apus_replica_destroy does the same before it frees anything.  APUS_ERROR when none is attached. */
int  apus_reader_detach(apus_replica_t *r);
/* failure detector: 0 while the leader's heartbeats arrive, else 1 + the term whose leader fell silent */
uint64_t apus_leader_suspect(apus_replica_t *follower);
/* %globaltimer (ns) of the leader kernel's latest commit (device clock; step timing of resident kernels) */
uint64_t apus_last_commit_ns(apus_replica_t *leader);

/* ---- control plane on NVLink words (election, votes, log adjustment; SURVEY.md s8f N1) ---------------------
 * Transport only: WHO votes for whom and when is decided by the caller (libapus_dare.so restates dare_server.c's
 * start_election / poll_vote_requests / poll_vote_count on top of these).  The words live in every replica's HBM
 * region next to its ack / tail slots (apus_layout.h: apus_ctlwords_t, the needed part of ctrl_data_t,
 * dare_server.h:121-138); a peer's words are written with a host-initiated copy through the same mapping the
 * kernels store through.  Replaces dare_ib_send_vote_request / replicate_vote / send_vote_ack
 * (dare_ibv_rc.c:969-1170), log_adjustment (dare_ibv_rc.c:1292-1451) and recover_log. */
typedef struct apus_ctl_view {
    uint64_t sid, leader_sid, adj_end, adj_count;
    uint64_t vote_ack[APUS_MAX_SERVER_COUNT];          /* commit offsets granted to me (log size = no vote) */
    struct { uint64_t sid, index, term, cid[2]; } vote_req[APUS_MAX_SERVER_COUNT];
} apus_ctl_view_t;
int  apus_ctl_read(apus_replica_t *r, apus_ctl_view_t *out);
int  apus_ctl_set_sid(apus_replica_t *r, uint64_t sid);
int  apus_ctl_reset_votes(apus_replica_t *r);                                  /* start_election: vote_ack[] := none */
int  apus_ctl_clear_vote_request(apus_replica_t *r, uint8_t from_idx);
int  apus_ctl_send_vote_request(apus_replica_t *r, uint8_t peer_idx, uint64_t sid, uint64_t index, uint64_t term,
                                const void *cid16);
int  apus_ctl_send_vote_ack(apus_replica_t *r, uint8_t candidate_idx, uint64_t commit);
/* follower: the heartbeat word the leader's kernel last wrote into this replica's region (term << 48 | beat counter;
 * dare_ibv_rc.c:868-958 writes the leader's SID into ctrl_data.hb[]).  The leader writes it whether or not this replica's
 * kernel runs, so a host that has stopped its kernel on a suspicion can tell a dead leader (the word stands still) from a
 * false positive (it moves) -- the reference's "false possitive => increase recomputed timeout", dare_server.c:781-796. */
int  apus_ctl_heartbeat(apus_replica_t *r, uint64_t *word);
/* idx and term of the last entry this replica holds (0,0 when the log is empty), its commit and end offsets; the
 * replica's kernel must be stopped (exclusive access, as dare_ib_revoke_log_access gives the reference) */
int  apus_ctl_last_entry(apus_replica_t *r, uint64_t *idx, uint64_t *term, uint64_t *commit, uint64_t *end);
/* elected leader, kernels stopped: bring follower `peer_idx` to my log -- find the last entry we share from its
 * commit offset on (log_find_remote_end_offset, dare_log.h:362-394), copy everything behind it (entry bytes and
 * offset index) peer to peer, and tell it to follow `sid` from there.  *resent = bytes copied.  A peer whose device
 * consumers run in any role (APUS_F_APPLY_ANY_ROLE) is refused, with nothing written, when its consumers have read
 * past the last entry it shares with me, or when it shares nothing with me and its consumers do not stand exactly at
 * my head -- unless they were seeded at a snapshot's mark (apus_consume_seed, which says when such a peer is accepted);
 * its consumer record is left naming no entry beyond what its offset index holds after the resend. */
int  apus_ctl_adjust_follower(apus_replica_t *leader, uint8_t peer_idx, uint64_t sid, uint64_t *resent);
/* role and term for the next launch.  Becoming leader takes over the log as this replica holds it (entry counters,
 * tail, submission ring); becoming follower adopts what the new leader's adjustment left (apus_ctl_view.adj_*).  With
 * APUS_F_APPLY_ANY_ROLE a new leader's device consumers go on from their cursor: the consume work enqueued before the
 * call runs first, then they may read up to the commit offset the leader adopted (the entries of earlier terms
 * committed with it).  A new leader's submission ring starts empty and its device doorbell at 0, however often it
 * led before.  A dormant resident submitter stays attached and dormant; with an active one the call is refused
 * (apus_submitter_attach). */
int  apus_replica_set_role(apus_replica_t *r, uint8_t leader_idx, uint64_t term);
/* leader: liveness counters of the followers (their kernels bump them while polling); a counter that stands still
 * is a follower that is gone (HB replies, dare_ibv_rc.c:912-958 -> fail_count -> check_failure_count) */
int  apus_follower_beats(apus_replica_t *leader, uint64_t out[APUS_MAX_SERVER_COUNT]);
/* stop storing into a peer that is gone (dare_ib_disconnect_server, dare_server.c:1200) */
int  apus_replica_disconnect(apus_replica_t *r, uint8_t peer_idx);

/* control plane hooks used by pruning (log_pruning, dare_server.c:1996-2067).  apus_set_head writes the header word a
 * LAUNCH starts from; while kernels are resident the head moves the way the reference moves it: with the HEAD entry that
 * carries the new offset (submit APUS_HEAD with the 8-byte offset; the leader adopts it when it places the entry). */
int  apus_set_head(apus_replica_t *r, uint64_t head);
int  apus_remote_apply_offsets(apus_replica_t *leader, uint64_t out[APUS_MAX_SERVER_COUNT]);

#ifdef __cplusplus
}
#endif
#endif /* APUS_GPU_H */
