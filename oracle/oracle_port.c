/*
 * oracle/oracle_port.c -- the restated oracle as a shared library
 * (oracle/liboracle_port.so).  TEST INFRASTRUCTURE ONLY (see orc_log.h).
 *
 * Exports, for ctypes:
 *   orc_log_*       single-log API over orc_log.h (restates dare_log.h)
 *   orc_cluster_*   replicate/ack/commit/apply steps (cluster_sim.inc)
 *   orc_bench_*     multi-threaded CPU run of the same steps (cpu_bench.inc)
 * A `rules` argument selects ORC_RULES_REFERENCE (bit-for-bit the reference,
 * bugs included) or ORC_RULES_ENGINE (divergences E1/E2, see orc_log.h).
 */
#include "orc_log.h"

static int g_rules = ORC_RULES_REFERENCE;
void orc_set_rules(int rules) { g_rules = rules; }
int  orc_get_rules(void) { return g_rules; }

/* ---- single-log API ----------------------------------------------------------- */
orc_log_t *orc_log_create(uint64_t len) { return orc_log_new(len, g_rules); }
void orc_log_destroy(orc_log_t *l) { orc_log_free(l); }
uint64_t orc_log_append(orc_log_t *l, uint64_t term, uint64_t req_id, uint16_t clt_id,
                        uint8_t type, const void *data)
{
    return orc_append(l, term, req_id, clt_id, type, data);
}
void orc_log_offsets(orc_log_t *l, uint64_t out[8])
{
    out[0] = l->head; out[1] = l->apply; out[2] = l->commit; out[3] = l->end;
    out[4] = l->tail; out[5] = l->old_end; out[6] = l->old_commit; out[7] = l->len;
}
void orc_log_set_offsets(orc_log_t *l, const uint64_t in[8])
{
    l->head = in[0]; l->apply = in[1]; l->commit = in[2]; l->end = in[3];
    l->tail = in[4]; l->old_end = in[5]; l->old_commit = in[6];
}
uint8_t *orc_log_entries(orc_log_t *l) { return l->entries; }
uint64_t orc_log_fnv(orc_log_t *l, uint64_t from, uint64_t to) { return orc_fnv1a(l->entries + from, to - from); }
uint64_t orc_log_end_distance(orc_log_t *l, uint64_t off) { return orc_end_distance(l, off); }
int orc_log_is_offset_larger(orc_log_t *l, uint64_t a, uint64_t b) { return orc_is_offset_larger(l, a, b); }
uint64_t orc_log_get_tail(orc_log_t *l) { return orc_get_tail(l); }
uint32_t orc_sizeof_entry(void) { return ORC_HDR; }

/* ---- cluster simulation bound to the restatement ------------------------------ */
#define SIM(name) orc_##name
#define L_T orc_log_t
#define L_NEW(len) orc_log_new((len), g_rules)
#define L_FREE(l) orc_log_free(l)
#define L_APPEND(l, term, req, clt, type, data) orc_append((l), (term), (req), (clt), (type), (data))
#define L_GET_ENTRY(l, poff) orc_get_entry((l), (poff))
#define L_FIT_ENTRY(l, off, e) orc_fit_entry((l), (off), (e))
#define L_ENTRY_LEN(e) orc_entry_len(e)
#define L_END_DISTANCE(l, off) orc_end_distance((l), (off))
#define L_IS_LARGER(l, a, b) orc_is_offset_larger((l), (a), (b))
#define L_GET_TAIL(l) orc_get_tail(l)
#define L_PREV_HEAD(l) ((l)->prev_head)
#define L_NORM(l, off) (((l)->rules == ORC_RULES_ENGINE && (off) == (l)->len) ? 0 : (off))
static orc_nc_buf_t g_nc[ORC_MAX_SERVER_COUNT];   /* the leader's nc_buf[i] (dare_log.h:99) */
#define L_NC_MAX ORC_NC_MAX
#define L_NC_BUILD(l, f, i) (orc_entries_to_nc_buf((f), &g_nc[i]), g_nc[i].len)
#define L_FIND_REMOTE_END(l, i) orc_find_remote_end_offset((l), &g_nc[i])
#include "cluster_sim.inc"
#include "cpu_bench.inc"
