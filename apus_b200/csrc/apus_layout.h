/*
 * apus_layout.h -- HBM layout of one replica and the structures shared between
 * the host engine (apus_engine.cu) and the kernels (the replica kernel of
 * apus_kernels.cu, the batch kernels of apus_batch.cu).
 *
 * One cudaMalloc'd REGION per replica (one IPC handle maps all of it in a peer):
 *
 *   +0        apus_ctrl_t   4 KiB   words written by REMOTE peers and kernel state
 *   +4096     apus_seq_t + publish ring   leader only: the sequencer words its worker CTAs
 *                                   share (claim / place / publish turns) and the ring of
 *                                   publishes awaiting a majority (60 KiB)
 *   +65536    apus_loghdr_t         mirror of dare_log_t up to entries[]
 *                                   (dare_log.h:77-103: head 0, apply 8, commit 16,
 *                                   end 24, tail 32, old_end 40, old_commit 48, len 56,
 *                                   nc_buf 64 .. 319656), padded to 320 KiB
 *   +APUS_INDEX_OFF    u32 index[idx_cap]  entry-offset ring: offset of the c-th entry
 *                                   ever appended at index[c & (idx_cap-1)], written by
 *                                   the leader next to the entry bytes so that a follower
 *                                   can ack without re-parsing the byte stream; idx_cap =
 *                                   pow2 >= log_len/64, so it can never be overrun while
 *                                   the log itself is not (head <= every apply offset)
 *   +entries_off       entries[log_len]   the reference's circular byte log
 *
 * entries[] starts 4 KiB-aligned so that a log offset and its address agree
 * modulo 16 (vectorised 16 B peer stores need that).
 *
 * Who writes what (all cross-GPU traffic is stores; nothing on the hot path reads
 * over NVLink):
 *   leader  -> follower.entries[range]       entry bytes           (replaces RDMA WRITE dare_ibv_rc.c:1606)
 *   leader  -> follower.index[..]            entry offsets, 4 B per entry
 *   leader  -> follower.ctrl.pub_{end,cum}   tail publish, 16 B    (dare_ibv_rc.c:1549-1573)
 *   leader  -> follower.ctrl.pub_commit      commit publish {offset, term}, 16 B (dare_ibv_rc.c:1810)
 *   follower-> leader.entries[e+28+idx]      reply byte, 1 B       (dare_ibv_rc.c:1833-1854)
 *   follower-> leader.ctrl.ack[idx]          ack word, 8 B         (the word the quorum ballot polls)
 *   follower-> leader.ctrl.apply_off[idx]    apply offset, 8 B     (push form of rc_get_remote_apply_offsets :1970)
 */
#ifndef APUS_LAYOUT_H
#define APUS_LAYOUT_H

#include <stddef.h>
#include <stdint.h>

#include "../../include/apus_slot_format.h"

#define APUS_MAX_SERVERS      13
#define APUS_HDR_BYTES        64u
#define APUS_CTRL_BYTES       4096u
#define APUS_LOGHDR_REF_BYTES 319656u                 /* offsetof(dare_log_t, entries) */
#define APUS_LOGHDR_BYTES     (320u * 1024u)
#define APUS_SEQ_OFF          4096u
#define APUS_PUBRING_OFF      8192u
#define APUS_PUBRING_RECORDS  256u                    /* 128 B each; power of two */
#define APUS_HDR_OFF          65536u
#define APUS_INDEX_OFF        (APUS_HDR_OFF + APUS_LOGHDR_BYTES)
#define APUS_IDX_HEAD_FLAG    0x80000000u             /* index word: the entry is a HEAD entry */

/* entry field offsets (dare_log.h:33-48) */
#define E_IDX     0
#define E_TERM    8
#define E_REQID  16
#define E_CLTID  24
#define E_TYPE   26
#define E_SENDER 27
#define E_REPLY  28
#define E_DATA   48
#define E_CMD    50

#define T_NOOP   0
#define T_CONFIG 2
#define T_HEAD   3

/* dare_log_t header mirror (first 64 bytes; nc_buf follows, unused on the hot path) */
typedef struct apus_loghdr {
    uint64_t head, apply, commit, end, tail, old_end, old_commit, len;
} apus_loghdr_t;

#define APUS_PUB_RING 1024u     /* leader: publishes in flight (power of two) */
#define APUS_LAT_RING 65536u    /* device-side latency samples (power of two) */

/* ctrl block: remote-written words first, each group on its own 128 B line */
typedef struct apus_ctrl {
    /* --- written by remote followers into the LEADER's region --- */
    uint64_t ack[16];            /* [i] = entries follower i has acked (monotone count) */
    uint64_t apply_off[16];      /* [i] = follower i's apply offset */
    uint64_t fbeat[16];          /* [i] = follower i's liveness counter (its kernel bumps it while it polls): what the
                                    leader's failure detector watches (the HB replies of dare_ibv_rc.c:912-958) */
    /* --- kernel-owned state that survives between launches --- */
    uint64_t next_idx;           /* leader: idx of the next entry (last.idx + 1) */
    uint64_t consumed;           /* leader: tickets taken from the submission ring */
    uint64_t published;          /* leader: entries whose tail has been published */
    uint64_t committed;          /* leader: entries committed */
    uint64_t committed_tickets;  /* leader: tickets committed */
    uint64_t hwm;                /* leader: high-water mark of bytes ever written (fresh beyond) */
    uint64_t bytes_replicated;
    uint64_t batches;
    uint64_t acked;              /* follower: entries acked */
    uint64_t lat_count;          /* leader: latency samples written */
    uint64_t auto_heads;         /* leader: HEAD entries appended by the device-side pruning rule */
    uint64_t pend_head_val;      /* follower: head carried by the last HEAD entry seen ... */
    uint64_t pend_head_end;      /* ... and the offset right after that entry (len = none) */
    uint64_t pub_seen;           /* leader: entries published as the commit warp has seen them (stats only; `published`
                                    follows the commit) */
    uint64_t pad0[2];
    /* --- written by the LEADER into each follower's region --- */
    uint64_t fin_entries;        /* end of a launch: entries the leader has published in total */
    uint64_t fin_target;         /* ... and the launch (its ticket target) this refers to */
    uint64_t pad1[14];
    uint64_t pub_end;            /* tail publish: the follower's new `end` (dare_ibv_rc.c:1549-1573) | APUS_PUB_CERT ... */
    uint64_t pub_cum;            /* ... and the entries that exist up to it | term << 48; one 16 B store */
    uint64_t pub_csum;           /* self-certifying publish (APUS_PUB_CERT): checksum of the bytes [start, end), keyed
                                    with pub_cum ... */
    uint64_t pub_start;          /* ... and the offset of the (single) entry; one 16 B store, NO fence before either */
    uint64_t pub_commit[2];      /* commit publish {leader's commit offset, term}: one 16 B store.  The follower drops
                                    other terms, clamps the offset to what it holds (I4) and keeps the result in its
                                    own header's `commit` */
    uint64_t pad2[2];
    uint64_t hb;                 /* leader -> follower heartbeat: term << 48 | beat counter (dare_ibv_rc.c:868-958 writes
                                    the leader's SID into ctrl_data.hb[]); its own 64 B half line */
    uint64_t pad3[7];
    /* --- leader profiling (APUS_F_DEVICE_STATS): ns spent per phase of the tile loop --- */
    uint64_t phase_ns[8];        /* [0] wait for requests, [1..6] T1..T6, [7] tiles */
    uint64_t turn_ns[8];         /* worker 0: [0] claim-lock wait, [1] place-turn wait, [2] publish-turn wait (ns),
                                    [3] fast placements, [4] slow placements, [7] place-turn hold (ns) */
    /* --- device consumers (APUS_F_DEVICE_APPLY, follower): one writer each, on this replica's own GPU --- */
    uint64_t cons_rec[2];        /* follower kernel -> consume work: {committed-and-held offset, entries held}, one 16 B
                                    release store per commit advance (cons_publish / cons_read) */
    uint64_t cons_cur[2];        /* consume work -> follower kernel: {cursor offset, idx of the next entry}; the cursor is
                                    the apply offset the follower reports to the leader's pruning rule */
    uint64_t cons_on;            /* 1: this replica was created with APUS_F_DEVICE_APPLY (the control plane refuses it);
                                    2: ... with APUS_F_APPLY_ANY_ROLE too (log adjustment guards its consumers) */
    uint64_t cons_seeded;        /* 1: apus_consume_seed started the consumers on an empty log at a snapshot's mark, and
                                    a leader's adjustment may accept this replica from there; host-written only */
    uint64_t pad4[10];
} apus_ctrl_t;

/* Control-plane words (N1: election, votes, log adjustment), at APUS_CTL_OFF inside the ctrl block -- the part of the
 * reference's ctrl_data_t (dare_server.h:121-138: sid, vote_req[], vote_ack[], prv_data) this engine needs.  Written by
 * HOST-initiated copies over NVLink (peers' blocks) and read by the host; the kernels never touch them. */
#define APUS_CTL_OFF 1024u
typedef struct apus_vote_req {       /* vote_req_t, dare_server.h:97-103 */
    uint64_t sid, index, term;
    uint64_t cid[2];                 /* dare_cid_t */
    uint64_t pad[3];
} apus_vote_req_t;
typedef struct apus_ctlwords {
    uint64_t sid;                    /* this replica's SID [TERM|L|IDX] (dare_server.h:46-61); voting = moving it (prv_data_t.vote_sid) */
    uint64_t leader_sid;             /* written by an elected leader once it has adjusted this replica's log: "follow me" */
    uint64_t adj_end;                /* ... the end offset ... */
    uint64_t adj_count;              /* ... and the entry count (== idx of the last entry) it left this replica at */
    uint64_t pad[4];
    uint64_t vote_ack[16];           /* written by voters into the CANDIDATE's block: their commit offset (log_len = no vote) */
    apus_vote_req_t vote_req[APUS_MAX_SERVERS];   /* [i] written by candidate i into everybody's block */
} apus_ctlwords_t;

/* the words a read fence reads in another replica's region, as byte offsets (apus_reader_view_t carries them) */
#define APUS_REGION_CONS_ON  ((uint32_t)offsetof(apus_ctrl_t, cons_on))
#define APUS_REGION_CONS_REC ((uint32_t)offsetof(apus_ctrl_t, cons_rec))
#define APUS_REGION_SID      ((uint32_t)(APUS_CTL_OFF + offsetof(apus_ctlwords_t, sid)))

/* Resident readers (apus_reader_attach): one pinned, mapped block per replica, kept current by the host (apus_gpu.h,
 * include/apus_reader.cuh).  The busy words have a 128 B line to themselves, away from the words the host writes. */
typedef struct apus_reader_block {
    volatile uint64_t role;                           /* the SID this replica knows: term << 9 | 1 << 8 | leader idx */
    uint64_t pad0[15];
    volatile uint64_t member[APUS_MAX_SERVERS];       /* [i]: member i's region as mapped here (own at own idx; 0 = none) */
    uint64_t pad1[3];
    volatile uint64_t busy[32];                       /* [s]: odd while a fence of slot s reads other regions */
} apus_reader_block_t;

/* Sequencer shared by the leader's worker CTAs (device memory, gpu-scope atomics).
 * A worker CLAIMS the next slots of the submission ring (one compare-and-swap), builds its
 * tile in parallel with the others, but PLACES it in the log and PUBLISHES its tail strictly
 * in slot order -- log order == submission order.  The turns are stamped with slot numbers. */
typedef struct apus_seq {
    uint64_t claimed_slots;      /* slots handed to workers so far (>= ctrl.consumed); compare-and-swap */
    uint64_t pad_c[15];
    uint64_t pub_turn[2];    uint64_t pad_e[14];   /* {next claim allowed to publish, next record number}: one 16 B word */
    uint64_t pub_tail;       uint64_t pad_g[15];   /* publish ring: next record the commit warp reads */
    uint64_t workers_done;
    uint64_t abort_flag;
    uint64_t ready_epoch;        /* == devctx.epoch once worker 0 has reset the block */
    uint64_t pad_h[13];
    /* placement state handed from claim to claim: four 16 B {stamp, value} pairs, each written
     * with ONE 16 B store and read with one 16 B load.  stamp == the claim sequence number whose
     * turn it is: the hand-over needs no fence (a system/gpu fence is expensive and the turn is
     * the only serialized part of the leader) */
    uint64_t rec_placed[2];      /* {stamp, entries placed so far} */
    uint64_t rec_end[2];         /* {stamp, end offset after the last placed entry (len = empty log)} */
    uint64_t rec_tail[2];        /* {stamp, tail offset | APUS_REC_PREV_HEAD | APUS_REC_WRAPPED} */
    uint64_t rec_head[2];        /* {stamp, head offset} (only the turn holder moves the head) */
    uint64_t avg_es, avg_xb;     /* log / staged bytes per entry of the latest claim (sizes the next claims;
                                    kept across launches) */
    uint64_t doorbell;           /* device-memory mirror of a host-mapped doorbell, kept by ONE relay warp so that
                                    idle workers do not all poll over PCIe */
    uint64_t w0_idle;            /* worker 0 is polling the next slot: it takes lone requests (express path) */
    uint64_t pad_i[4];
} apus_seq_t;
#define APUS_REC_PREV_HEAD (1ull << 62)   /* the last placed entry is a HEAD entry of the pruning rule */
#define APUS_REC_WRAPPED   (1ull << 63)   /* the ring has wrapped at least once (no fresh bytes left) */

/* One record per published tile, consumed in order by the commit warp.  Eight 16 B {stamp, value}
 * pairs, each written with one 16 B store (stamp = record number + 1): a record is valid when all
 * eight stamps match, no fence needed.  The commit warp also does the leader's bookkeeping from it. */
#define PR_CUM     0   /* entries published up to and including this tile */
#define PR_END     1   /* `end` after this tile */
#define PR_TICKETS 2   /* tickets consumed up to and including this tile */
#define PR_T0      3   /* dequeue timestamp (ns) */
#define PR_TAIL    4   /* offset of the last entry */
#define PR_HWM     5   /* high-water mark of bytes ever written */
#define PR_NEXTIDX 6   /* idx of the next entry */
#define PR_BYTES   7   /* bytes replicated by this tile, summed over followers */
typedef struct apus_pubrec {
    uint64_t w[16];
} apus_pubrec_t;

/* the submission slot (apus_slot_t, APUS_SLOT_*): include/apus_slot_format.h */
#define APUS_CSLOT_BYTES  96u     /* a slot as the leader keeps it in shared memory: descriptor + inline image */
/* the same slot without its stamp chunks (shared memory of the leader) */
typedef struct apus_cslot {
    uint64_t req_id;
    uint32_t type_off;
    uint16_t len;
    uint16_t clt_id;
    uint8_t  inl[APUS_SLOT_INLINE];
} apus_cslot_t;

/* words in pinned, mapped host memory shared with the kernels */
typedef struct apus_hostwords {
    volatile uint64_t sub_tail;          /* host -> kernel doorbell (RING_HOST_MAPPED) */
    uint64_t pad0[15];
    volatile uint64_t commit_off;        /* kernel -> host: {commit offset, committed tickets} is ONE 16 B store, */
    volatile uint64_t committed_tickets; /* ... so a 16 B host load sees a consistent pair */
    volatile uint64_t consumed;          /* kernel -> host (ring space) */
    volatile uint64_t last_commit_ns;    /* kernel -> host: %globaltimer of the latest commit */
    volatile uint64_t dev_rejected;      /* packing kernel -> host: requests of device batches written as NOOPs ... */
    volatile uint64_t dev_first_rejected;/* ... and the ticket of the first of them (0 = none) */
    volatile uint64_t cons_cursor;       /* consume work -> host (APUS_F_DEVICE_APPLY): the cursor after the latest call, */
    volatile uint64_t cons_next_idx;     /* ... the idx of the next entry, */
    volatile uint64_t cons_need_stride;  /* ... the stride the entry that stopped it needs (0 = none), */
    volatile uint64_t cons_error;        /* ... and APUS_CONSUME_BAD_IDX (apus_gpu.h; 0 = none; sticky) */
    volatile uint64_t cons_wait_epoch;   /* host -> consume waits: apus_consume_wait_release bumps it; a wait enqueued
                                            under an older value ends as APUS_WAIT_RELEASED */
    volatile uint64_t cons_wait_outcome; /* consume wait -> host: APUS_WAIT_* of the latest wait that ran (UINT64_MAX:
                                            none has run yet) ... */
    volatile uint64_t cons_wait_avail;   /* ... and the committed entries past the cursor when it ended */
    volatile uint64_t fence_outcome;     /* read fence -> host: APUS_WAIT_* / APUS_WAIT_NOT_LEADER of the latest fence that
                                            ran (UINT64_MAX: none has run yet) ... */
    volatile uint64_t fence_index;       /* ... and its read index (0 unless it ended READY) */
    uint64_t pad1[1];
    volatile uint32_t stop;              /* host -> kernel */
    uint32_t pad2[31];
    volatile uint64_t host_apply;        /* host -> follower kernel (APUS_FLAG_HOST_APPLY): offset up to which the
                                            application has replayed the log (dare_server.c:1939-1962) */
    volatile uint64_t consumer_stop;     /* host -> resident consumer (apus_consumer_attach): detach and destroy bump it;
                                            the consumer ends once it differs from the value it was attached under */
    volatile uint64_t submitter_stop;    /* host -> resident submitter (apus_submitter_attach): detach and destroy bump
                                            it, the same way */
    volatile uint64_t reader_stop;       /* host -> resident reader (apus_reader_attach): detach and destroy bump it */
    uint64_t pad3[12];
    volatile uint64_t heartbeat;         /* kernel liveness (debug) */
    volatile uint64_t error;             /* kernel-detected protocol error code */
    volatile uint64_t leader_suspect;    /* follower kernel -> host: 1 + term whose leader stopped sending heartbeats */
    volatile uint64_t hb_seen;           /* follower kernel -> host: last heartbeat word observed */
} apus_hostwords_t;
#ifdef __cplusplus
static_assert(offsetof(apus_hostwords_t, stop) == 256 && offsetof(apus_hostwords_t, host_apply) == 384 &&
              offsetof(apus_hostwords_t, consumer_stop) == 392 && offsetof(apus_hostwords_t, submitter_stop) == 400 &&
              offsetof(apus_hostwords_t, reader_stop) == 408 && offsetof(apus_hostwords_t, heartbeat) == 512 && sizeof(apus_hostwords_t) == 544,
              "the stop words of resident consumers, submitters and readers take spare words: no offset moves");
#endif

#define APUS_FLAG_FENCED_ACK 0x1u
#define APUS_FLAG_STATS      0x2u
#define APUS_FLAG_AUTOPRUNE  0x4u
#define APUS_FLAG_WALK       0x8u   /* follower parses the byte stream itself (reference behaviour) */
#define APUS_FLAG_HOST_APPLY 0x10u  /* follower: the apply offset it reports is the one the HOST has replayed */
#define APUS_FLAG_NO_EXPRESS 0x20u  /* leader: no single-warp express path / self-certifying publishes */
#define APUS_FLAG_PROFILE    0x40u  /* %globaltimer stamps inside the express path and the follower's verification (the reads
                                       lengthen the path: kept out of measured runs) */

#define APUS_FLAG_DEVICE_APPLY 0x200u /* follower: the apply offset it reports is the device consumers' cursor */
#define APUS_FLAG_APPLY_ANY_ROLE 0x400u /* with DEVICE_APPLY, on a leader: the commit warp publishes the consumer record,
                                           and the consumers' cursor is the leader's apply offset */

#define APUS_PUB_CERT      (1ull << 63)         /* pub_end: this publish is self-certifying (no writer fence) */
#define APUS_PUB_TERM_SHIFT 48                   /* pub_cum / hb: term in the top 16 bits */
#define APUS_PUB_CUM_MASK  ((1ull << 48) - 1)

#define APUS_ROLE_NONE     0
#define APUS_ROLE_LEADER   1
#define APUS_ROLE_FOLLOWER 2

/* everything a kernel role needs; lives in device memory, written by the host
 * before each launch */
typedef struct apus_devctx {
    uint8_t  idx, group_size, leader_idx, quorum;
    uint32_t flags;
    uint64_t term;
    uint64_t log_len;
    uint64_t entries_off;                 /* byte offset of entries[] inside a region */
    uint32_t idx_mask;                    /* index ring capacity - 1 */
    uint32_t pad_i;
    uint64_t target;                      /* cumulative ticket / entry target of this launch */
    uint32_t n_workers;                   /* leader CTAs of this launch */
    uint32_t doorbell_relay;              /* 1: workers poll seq.doorbell, a relay warp polls the host word */
    uint32_t slot_poll;                   /* 1: worker 0 polls the next slot itself (host-mapped ring) */
    uint32_t epoch;                       /* launch counter (sequencer reset handshake) */
    uint64_t hb_period_ns;                /* leader: heartbeat period (0 = no heartbeats) */
    uint64_t hb_timeout_ns;               /* follower: silence after which the leader is suspected (0 = never) */
    uint8_t *region;                      /* own region */
    uint8_t *mc_region;                   /* leader, fabric mode: NVSwitch multicast mapping of the group's regions (else NULL) */
    uint8_t *peer[APUS_MAX_SERVERS];      /* peers' regions as mapped here (NULL = absent) */
    /* leader submission ring */
    const apus_slot_t *sub_slots;
    const uint8_t     *sub_pay;
    uint32_t           sub_mask;          /* slots - 1 */
    uint32_t           pad;
    const volatile uint64_t *sub_tail;    /* doorbell word (host-mapped or device) */
    apus_hostwords_t  *hw;                /* host-mapped words */
    uint32_t          *lat_ns;            /* device latency ring (APUS_LAT_RING) or NULL */
} apus_devctx_t;

typedef struct apus_role {
    uint32_t       kind;
    uint32_t       worker;                /* leader: worker CTA index */
    apus_devctx_t *ctx;
} apus_role_t;

/* Device consumers (apus_consume_device, apus_consume_device_packed): the state of one replica's consume work, in
 * device memory ahead of APUS_CONS_BLK_WORDS words per consume block ({rows, then their exclusive scan; stop; cmd
 * bytes of those rows, then their exclusive scan (packed calls)}).  The cursor itself is apus_ctrl_t.cons_cur. */
typedef struct apus_cons_state {
    uint64_t cursor, next_idx, committed, m;  /* this call: the cursor and the record it starts from, entries to look at */
    uint64_t rows, n_exam, new_cursor, need_stride;   /* ... and what it found */
    uint64_t error;                           /* sticky APUS_CONSUME_BAD_IDX */
    uint64_t bytes;                           /* packed calls: cmd bytes of the rows written (offsets[rows]) */
    uint64_t pad[6];
} apus_cons_state_t;
#define APUS_CONS_THREADS 256u                /* entries per consume block */
#define APUS_CONS_BLK_WORDS 3u

/* one consume call as the consume kernels see it: the strided layout (lens and payloads + row * stride) or, when
 * offsets is set, the packed one (row r's cmd at payloads + offsets[r], at most values_cap bytes in all; lens NULL) */
typedef struct apus_consume_args {
    uint8_t  *region;                         /* the follower's region (ctrl block, index, entries) */
    uint64_t  entries_off, log_len, stride;
    uint32_t  idx_mask, max_n;                /* max_n <= the index ring's capacity */
    uint32_t  nblk, pad;
    apus_cons_state_t *st;                    /* followed by APUS_CONS_BLK_WORDS * nblk words */
    apus_hostwords_t  *hw;                    /* status words (device address of the pinned page) */
    uint64_t *idx;
    uint8_t  *types;
    uint16_t *conns;
    uint64_t *req_ids;
    uint16_t *lens;
    uint8_t  *payloads;
    uint32_t *count;
    uint64_t *offsets;                        /* packed: max_n + 1 words */
    uint64_t  values_cap;
} apus_consume_args_t;

/* one read fence (apus_read_fence) as its kernel sees it: the group's regions as this replica maps them when the fence is
 * enqueued (NULL = not connected, or a peer destroyed since), its own, and the term and leader it knew then */
typedef struct apus_fence_args {
    const uint8_t *member[APUS_MAX_SERVERS];  /* [i < n]: member i's region; [own idx] = region */
    const uint8_t *region;                    /* this replica's region (ctrl block, index, entries) */
    apus_hostwords_t *hw;                     /* status words and the release epoch (device address of the pinned page) */
    uint64_t  epoch;                          /* the release epoch the fence was enqueued under */
    uint64_t  term;                           /* t */
    uint64_t  entries_off, log_len;
    uint64_t  timeout_ns;
    uint64_t *index;                          /* receives F on READY */
    uint32_t *outcome;                        /* optional */
    uint32_t  idx_mask;
    uint8_t   n, leader, pad[2];
} apus_fence_args_t;

/* Device batches (apus_submit_device, apus_submit_device_packed): one batch as the packing kernels see it, in either
 * layout.  A packing block has as many threads as a consume block (the two share one block scan). */
#define APUS_PACK_THREADS 256u     /* requests per packing block */
/* words per packing block: external bytes (-> their exclusive scan), rejected, first rejected, and the packed layout's
 * verdict: the block saw offsets that decrease or end past values_bytes (-> the whole batch's verdict) */
#define APUS_PACK_BLK_WORDS 4u
static inline uint32_t apus_pack_blocks(uint64_t n) { return (uint32_t)((n + APUS_PACK_THREADS - 1) / APUS_PACK_THREADS); }
typedef struct apus_pack_args {
    apus_slot_t *ring;
    uint8_t *pay;
    uint64_t *blk;                /* APUS_PACK_BLK_WORDS per block, see above */
    const uint8_t *types;
    const uint16_t *conns;
    const uint64_t *req_ids;
    const uint16_t *lens;         /* strided layout (apus_submit_device): cmd k is payloads[k * stride, + lens[k]) */
    const uint64_t *offsets;      /* packed layout (apus_submit_device_packed, lens NULL): cmd k is
                                     payloads[offsets[k], offsets[k + 1]), inside [0, values_bytes) */
    const uint8_t *payloads;
    uint64_t stride, values_bytes;
    uint64_t first_slot;          /* submitted count before the batch: request k gets ticket first_slot + k + 1 */
    uint64_t res_pos;             /* ring position of the batch's payload reservation */
    uint32_t n, mask;
} apus_pack_args_t;

#define APUS_KERNEL_THREADS    512
#define APUS_MAX_TILE_ENTRIES  512u             /* slots fetched per tile (48 KiB of shared memory) */
#define APUS_LEADER_IMG_BYTES  (80u * 1024u)    /* log bytes composed per tile (>= one maximal entry) */
#define APUS_LEADER_EXT_BYTES  (66u * 1024u)    /* payload-ring bytes staged per tile (>= one maximal image) */
#define APUS_FOLLOWER_WIN_BYTES (96u * 1024u)   /* log bytes a follower walks per window */

#endif /* APUS_LAYOUT_H */
