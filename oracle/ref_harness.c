/*
 * oracle/ref_harness.c -- the REFERENCE's own log code as a shared library
 * (oracle/_ref/libapus_ref.so).  TEST INFRASTRUCTURE ONLY (see orc_log.h).
 *
 * This file #includes /root/reference/src/include/dare/dare_log.h UNMODIFIED
 * (header-only, static functions; -I points at the read-only reference tree,
 * no reference source is copied into this repository) and exposes it through
 * the same flat API as oracle_port.c, so tests can drive the compiled reference
 * and the restatement with identical inputs and compare every byte.  The
 * replicate/ack/commit/apply steps come from cluster_sim.inc (the files holding
 * them in the reference need libibverbs/libev and cannot be compiled here) but
 * run on the reference's log_append_entry / log_get_entry / log_fit_entry /
 * log_entry_len / log_offset_end_distance / log_is_offset_larger / log_get_tail, and log adjustment on its
 * log_entries_to_nc_buf / log_find_remote_end_offset.
 *
 * Built only where /root/reference exists (oracle/Makefile target `ref`); the
 * resulting .so travels to the GPU box, the reference tree does not.
 */
#include <stdio.h>
#include <stddef.h>
#include <stdint.h>
#include <dare/dare_log.h>

FILE *log_fp;                 /* debug.h:108 expects the embedding program to define it */
int prev_log_entry_head;      /* dare_log.h:27 */

_Static_assert(sizeof(dare_log_entry_t) == 64, "entry header");
_Static_assert(offsetof(dare_log_entry_t, idx) == 0, "idx");
_Static_assert(offsetof(dare_log_entry_t, term) == 8, "term");
_Static_assert(offsetof(dare_log_entry_t, req_id) == 16, "req_id");
_Static_assert(offsetof(dare_log_entry_t, clt_id) == 24, "clt_id");
_Static_assert(offsetof(dare_log_entry_t, type) == 26, "type");
_Static_assert(offsetof(dare_log_entry_t, sender) == 27, "sender");
_Static_assert(offsetof(dare_log_entry_t, reply) == 28, "reply");
_Static_assert(offsetof(dare_log_entry_t, data) == 48, "data");
_Static_assert(offsetof(dare_log_t, head) == 0 && offsetof(dare_log_t, apply) == 8 &&
               offsetof(dare_log_t, commit) == 16 && offsetof(dare_log_t, end) == 24 &&
               offsetof(dare_log_t, tail) == 32 && offsetof(dare_log_t, old_end) == 40 &&
               offsetof(dare_log_t, old_commit) == 48 && offsetof(dare_log_t, len) == 56 &&
               offsetof(dare_log_t, nc_buf) == 64, "log header");
_Static_assert(offsetof(dare_log_t, entries) == 319656, "entries");
_Static_assert(sizeof(dare_cid_t) == 16, "cid");

static void ref_init(void) { if (!log_fp) log_fp = stderr; }

/* log_new() is hard-wired to LOG_SIZE; for other lengths repeat its
 * initialisation (dare_log.h:120-137) on a buffer of the requested size. */
static dare_log_t *ref_new_len(uint64_t len)
{
    ref_init();
    if (len == (uint64_t)(LOG_SIZE)) return log_new();
    dare_log_t *log = (dare_log_t *)calloc(1, sizeof(dare_log_t) + len);
    if (!log) return NULL;
    log->len = len; log->end = len; log->tail = len; log->old_end = len;
    return log;
}

/* ---- single-log API ----------------------------------------------------------- */
dare_log_t *ref_log_create(uint64_t len) { return ref_new_len(len); }
void ref_log_destroy(dare_log_t *l) { log_free(l); }
uint64_t ref_log_append(dare_log_t *l, uint64_t term, uint64_t req_id, uint16_t clt_id,
                        uint8_t type, const void *data)
{
    return log_append_entry(l, term, req_id, clt_id, type, (void *)data);
}
void ref_log_offsets(dare_log_t *l, uint64_t out[8])
{
    out[0] = l->head; out[1] = l->apply; out[2] = l->commit; out[3] = l->end;
    out[4] = l->tail; out[5] = l->old_end; out[6] = l->old_commit; out[7] = l->len;
}
void ref_log_set_offsets(dare_log_t *l, const uint64_t in[8])
{
    l->head = in[0]; l->apply = in[1]; l->commit = in[2]; l->end = in[3];
    l->tail = in[4]; l->old_end = in[5]; l->old_commit = in[6];
}
uint8_t *ref_log_entries(dare_log_t *l) { return l->entries; }
uint64_t ref_log_end_distance(dare_log_t *l, uint64_t off) { return log_offset_end_distance(l, off); }
int ref_log_is_offset_larger(dare_log_t *l, uint64_t a, uint64_t b) { return log_is_offset_larger(l, a, b); }
uint64_t ref_log_get_tail(dare_log_t *l) { return log_get_tail(l); }
uint32_t ref_sizeof_entry(void) { return (uint32_t)sizeof(dare_log_entry_t); }
uint64_t ref_sizeof_log(void) { return (uint64_t)sizeof(dare_log_t); }
uint64_t ref_log_size(void) { return (uint64_t)(LOG_SIZE); }

/* ---- cluster simulation bound to the reference header ------------------------- */
#define SIM(name) ref_##name
#define L_T dare_log_t
#define L_NEW(len) ref_new_len(len)
#define L_FREE(l) log_free(l)
#define L_APPEND(l, term, req, clt, type, data) \
    log_append_entry((l), (term), (req), (clt), (type), (void *)(data))
#define L_GET_ENTRY(l, poff) ((uint8_t *)log_get_entry((l), (poff)))
#define L_FIT_ENTRY(l, off, e) log_fit_entry((l), (off), (dare_log_entry_t *)(e))
#define L_ENTRY_LEN(e) log_entry_len((dare_log_entry_t *)(e))
#define L_END_DISTANCE(l, off) log_offset_end_distance((l), (off))
#define L_IS_LARGER(l, a, b) log_is_offset_larger((l), (a), (b))
#define L_GET_TAIL(l) log_get_tail(l)
#define L_PREV_HEAD(l) prev_log_entry_head
#define L_NORM(l, off) (off)
/* log adjustment: the follower builds the list in its own log (server_to_follower); the leader reads it into its
 * nc_buf[i] (LR_GET_NCE) -- here built straight into the leader's slot, which holds the same bytes */
#define L_NC_MAX MAX_NC_ENTRIES
#define L_NC_BUILD(l, f, i) (log_entries_to_nc_buf((f), &(l)->nc_buf[i]), (l)->nc_buf[i].len)
#define L_FIND_REMOTE_END(l, i) log_find_remote_end_offset((l), &(l)->nc_buf[i])
#include "cluster_sim.inc"
#include "cpu_bench.inc"
