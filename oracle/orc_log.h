/*
 * oracle/orc_log.h -- CPU restatement of the APUS/DARE consensus log.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product path:
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may build, load or call it.  The product (apus_b200/csrc) never
 * links or falls back to this code.
 *
 * What it restates (reference = /root/reference, hku-systems/apus):
 *   src/include/dare/dare_log.h   the circular log: layout, append, walkers, and the
 *                                 not-committed-entry list of log adjustment
 * Every function cites the reference lines it follows.  The restatement is an
 * independent re-write working on explicit byte offsets (no struct overlay), so
 * it also documents the byte layout the CUDA engine must reproduce:
 *
 *   entry header, 64 B (dare_log.h:33-48; offsets measured in SURVEY.md s8):
 *     +0  idx u64 | +8 term u64 | +16 req_id u64 | +24 clt_id u16 | +26 type u8
 *     +27 sender u8 | +28 reply[13] | +41..47 padding (never written)
 *     +48 data union: sm_cmd_t{u16 len; u8 cmd[]} | dare_cid_t (16 B) | u64 head
 *   entry stride: 64 for NOOP/CONFIG/HEAD, 64 + cmd.len otherwise (:228-234)
 *
 * Parity status: the reference has no tests or golden vectors for this path
 * (SURVEY.md s4, s8c), so parity is pinned differently: oracle/ref_harness.c
 * compiles the reference's own dare_log.h unmodified into oracle/_ref/ and
 * tests/test_oracle_vs_ref.py checks this restatement against it bit for bit;
 * tests/golden/ holds vectors generated from that compiled reference header.
 *
 * rules == ORC_RULES_REFERENCE reproduces the reference bit for bit, including
 * its wrap bugs (SURVEY.md H11 iii/iv).  rules == ORC_RULES_ENGINE applies the
 * two documented divergences of the CUDA engine (DESIGN.md s"Divergences"):
 *   E1  an append that makes end == len stores end = 0 instead (the reference's
 *       value doubles as the "log is empty" sentinel and makes the entry vanish);
 *   E2  an append that does not fit before `head` is refused with NO state
 *       change (the engine back-pressures; the reference corrupts `end`).
 */
#ifndef ORC_LOG_H
#define ORC_LOG_H

#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_NOOP   0
#define ORC_CSM    1
#define ORC_CONFIG 2
#define ORC_HEAD   3
/* proxy entry types (src/include/proxy/proxy.h:9-11) -- all take the CSM path */
#define ORC_P_CONNECT 4
#define ORC_P_SEND    5
#define ORC_P_CLOSE   6

#define ORC_MAX_SERVER_COUNT 13                 /* dare.h:26 */
#define ORC_HDR   64u                           /* sizeof(dare_log_entry_t) */
#define ORC_LOG_SIZE (16384ull * 4096ull)       /* dare_log.h:76 */

#define ORC_OFF_IDX     0
#define ORC_OFF_TERM    8
#define ORC_OFF_REQID  16
#define ORC_OFF_CLTID  24
#define ORC_OFF_TYPE   26
#define ORC_OFF_SENDER 27
#define ORC_OFF_REPLY  28
#define ORC_OFF_DATA   48
#define ORC_OFF_CMD    50

#define ORC_RULES_REFERENCE 0
#define ORC_RULES_ENGINE    1

typedef struct orc_log {
    uint64_t head, apply, commit, end, tail, old_end, old_commit, len;
    int      prev_head;   /* the reference's global prev_log_entry_head */
    int      rules;
    uint8_t *entries;
} orc_log_t;

static inline uint64_t orc_ld64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static inline uint16_t orc_ld16(const uint8_t *p) { uint16_t v; memcpy(&v, p, 2); return v; }
static inline void orc_st64(uint8_t *p, uint64_t v) { memcpy(p, &v, 8); }
static inline void orc_st16(uint8_t *p, uint16_t v) { memcpy(p, &v, 2); }

/* dare_log.h:120-137 log_new (len generalised; the reference hard-wires LOG_SIZE) */
static orc_log_t *orc_log_new(uint64_t len, int rules)
{
    orc_log_t *l = (orc_log_t *)calloc(1, sizeof(*l));
    if (!l) return NULL;
    l->entries = (uint8_t *)calloc(1, len);
    if (!l->entries) { free(l); return NULL; }
    l->len = len;
    l->end = len;
    l->tail = len;
    l->old_end = len;
    l->rules = rules;
    return l;
}

static void orc_log_free(orc_log_t *l)
{
    if (l) { free(l->entries); free(l); }
}

/* dare_log.h:158-162 */
static inline int orc_is_empty(const orc_log_t *l) { return l->end == l->len; }
/* dare_log.h:168-172 */
static inline int orc_is_full(const orc_log_t *l) { return l->end == l->head; }
/* dare_log.h:201-205 */
static inline int orc_fit_header(const orc_log_t *l, uint64_t off) { return l->len - off >= ORC_HDR; }

/* dare_log.h:228-234 */
static inline uint32_t orc_entry_len(const uint8_t *e)
{
    uint8_t t = e[ORC_OFF_TYPE];
    if (t == ORC_NOOP || t == ORC_CONFIG || t == ORC_HEAD) return ORC_HDR;
    return ORC_HDR + orc_ld16(e + ORC_OFF_DATA);
}

/* dare_log.h:241-247 */
static inline int orc_fit_entry(const orc_log_t *l, uint64_t off, const uint8_t *e)
{
    return l->len - off >= orc_entry_len(e);
}

/* dare_log.h:255-262 */
static inline uint64_t orc_end_distance(const orc_log_t *l, uint64_t off)
{
    uint64_t end = l->end;
    if (end == l->len) return 0;
    if (end >= off) return end - off;
    return l->len - (off - end);
}

/* dare_log.h:269-282: "larger" == closer to end */
static inline int orc_is_offset_larger(const orc_log_t *l, uint64_t lo, uint64_t ro)
{
    return orc_end_distance(l, lo) < orc_end_distance(l, ro);
}

/* dare_log.h:316-332 */
static uint8_t *orc_get_entry(orc_log_t *l, uint64_t *off)
{
    if (orc_is_empty(l)) return NULL;
    if (0 == orc_end_distance(l, *off)) return NULL;
    if (!orc_fit_header(l, *off)) *off = 0;
    return l->entries + *off;
}

/* one step of the walk every reference loop performs
 * (dare_log.h:346-357, dare_server.c:1795-1808, dare_ibv_rc.c:1726-1745) */
static inline void orc_walk_next(orc_log_t *l, uint64_t *off, const uint8_t *e)
{
    if (!orc_fit_entry(l, *off, e)) *off = 0;
    *off += orc_entry_len(e);
}

/* dare_log.h:402-457 */
static uint64_t orc_get_tail(orc_log_t *l)
{
    if (l->tail != l->len) return l->tail;
    if (orc_is_empty(l)) return l->len;
    uint64_t starts[3] = { l->commit, l->apply, l->head };
    uint64_t tail = l->len;
    for (int s = 0; s < 3; s++) {
        uint64_t off = starts[s];
        uint8_t *e;
        while ((e = orc_get_entry(l, &off)) != NULL) {
            tail = off;
            orc_walk_next(l, &off, e);
        }
        if (tail != l->len && s < 2) return tail;
    }
    return tail;
}

/* dare_log.h:213-221 */
static inline uint8_t *orc_add_new_entry(orc_log_t *l)
{
    if (orc_is_full(l)) return NULL;
    if (orc_is_empty(l) || !orc_fit_header(l, l->end)) return l->entries;
    return l->entries + l->end;
}

static inline void orc_fill_header(uint8_t *e, uint64_t idx, uint64_t term, uint64_t req_id,
                                   uint16_t clt_id, uint8_t type)
{
    orc_st64(e + ORC_OFF_IDX, idx);
    orc_st64(e + ORC_OFF_TERM, term);
    orc_st64(e + ORC_OFF_REQID, req_id);
    orc_st16(e + ORC_OFF_CLTID, clt_id);
    e[ORC_OFF_TYPE] = type;
    memset(e + ORC_OFF_REPLY, 0, ORC_MAX_SERVER_COUNT);
}

/* bytes the append is going to occupy, counting the stretch skipped at the wrap;
 * used only by rule E2 (engine back-pressure) */
static uint64_t orc_append_span(const orc_log_t *l, uint32_t elen)
{
    uint64_t end = orc_is_empty(l) ? 0 : l->end;
    if (l->len - end < ORC_HDR || l->len - end < elen) return (l->len - end) + elen;
    return elen;
}

/*
 * dare_log.h:466-558 log_append_entry.
 * `data`: sm_cmd_t image {u16 len; u8 cmd[len]} for CSM-like types, dare_cid_t
 * (16 B) for CONFIG, u64 for HEAD, ignored for NOOP.
 * Returns the new idx, or 0 when the reference reports "The LOG is full".
 */
static uint64_t orc_append(orc_log_t *l, uint64_t term, uint64_t req_id, uint16_t clt_id,
                           uint8_t type, const void *data)
{
    const uint8_t *d = (const uint8_t *)data;
    uint16_t clen = 0;
    int has_cmd = !(type == ORC_NOOP || type == ORC_CONFIG || type == ORC_HEAD);
    if (has_cmd) clen = orc_ld16(d);
    uint32_t elen = ORC_HDR + (has_cmd ? clen : 0);

    if (l->rules == ORC_RULES_ENGINE) {
        /* E2: refuse (caller blocks) unless the span fits strictly before head */
        uint64_t used = orc_is_empty(l) ? 0 : orc_end_distance(l, l->head);
        if (used + orc_append_span(l, elen) >= l->len) return 0;
    }

    if (type != ORC_HEAD) l->prev_head = 0;                       /* :477-480 */

    if (l->tail == l->len) l->tail = orc_get_tail(l);             /* :483-485 */
    uint64_t off = l->tail;
    uint8_t *last = orc_get_entry(l, &off);                       /* :486-488 */
    uint64_t idx = last ? orc_ld64(last + ORC_OFF_IDX) + 1 : 1;

    uint8_t *e = orc_add_new_entry(l);                            /* :491-495 */
    if (!e) return 0;
    orc_fill_header(e, idx, term, req_id, clt_id, type);          /* :496-501 */
    if (!orc_fit_header(l, l->end)) l->end = 0;                   /* :502-504 */

    switch (type) {                                               /* :507-545 */
    case ORC_CONFIG: memcpy(e + ORC_OFF_DATA, d, 16); break;
    case ORC_HEAD:   memcpy(e + ORC_OFF_DATA, d, 8); break;
    case ORC_NOOP:   break;
    default:
        orc_st16(e + ORC_OFF_DATA, clen);
        if (!orc_fit_entry(l, l->end, e)) {
            /* the header written above stays behind as a payload-less ghost */
            l->end = 0;
            e = orc_add_new_entry(l);
            if (!e) return 0;
            orc_fill_header(e, idx, term, req_id, clt_id, type);
            orc_st16(e + ORC_OFF_DATA, clen);
        }
        if (clen) memcpy(e + ORC_OFF_CMD, d + 2, clen);
        break;
    }
    l->tail = l->end;                                             /* :547 */
    l->end += orc_entry_len(e);                                   /* :549 */
    if (l->rules == ORC_RULES_ENGINE && l->end == l->len) l->end = 0;   /* E1 */
    return idx;
}

/* dare_log.h:50-65: {idx, term, offset} of every entry that is not committed */
#define ORC_NC_MAX 1024                         /* MAX_NC_ENTRIES */
typedef struct orc_nc_buf {
    uint64_t len;
    struct { uint64_t idx, term, offset; } e[ORC_NC_MAX];
} orc_nc_buf_t;

/* dare_log.h:340-359 log_entries_to_nc_buf: walk from the commit offset to the end;
 * the offset recorded is where the walk found the header (a ghost's, for an entry
 * that continues at 0) */
static void orc_entries_to_nc_buf(orc_log_t *l, orc_nc_buf_t *nc)
{
    uint64_t off = l->commit, n = 0;
    uint8_t *e;
    while ((e = orc_get_entry(l, &off)) != NULL) {
        nc->e[n].idx = orc_ld64(e + ORC_OFF_IDX);
        nc->e[n].term = orc_ld64(e + ORC_OFF_TERM);
        nc->e[n].offset = off;
        n++;
        orc_walk_next(l, &off, e);
    }
    nc->len = n;
}

/* dare_log.h:368-394 log_find_remote_end_offset: the offset of the first listed
 * entry that this log does not hold at the same offset with the same {idx, term},
 * or the offset behind the last one */
static uint64_t orc_find_remote_end_offset(orc_log_t *l, const orc_nc_buf_t *nc)
{
    uint64_t off = 0;
    for (uint64_t i = 0; i < nc->len; i++) {
        off = nc->e[i].offset;
        uint8_t *e = orc_get_entry(l, &off);
        if (!e) return off;
        if (orc_ld64(e + ORC_OFF_IDX) != nc->e[i].idx || orc_ld64(e + ORC_OFF_TERM) != nc->e[i].term) return off;
        orc_walk_next(l, &off, e);
    }
    return off;
}

/* FNV-1a 64 over a byte range; the checksum quoted in SURVEY.md s8c */
static inline uint64_t orc_fnv1a(const uint8_t *p, uint64_t n)
{
    uint64_t h = 0xcbf29ce484222325ull;
    for (uint64_t i = 0; i < n; i++) { h ^= p[i]; h *= 0x100000001b3ull; }
    return h;
}

#endif /* ORC_LOG_H */
