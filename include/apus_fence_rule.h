/*
 * apus_fence_rule.h -- the decisions of a read fence (DESIGN.md section 2 "Read fences"), in plain C and CUDA: the
 * stream fence kernel (apus_b200/csrc/apus_batch.cu), the resident reader (apus_reader.cuh) and the CPU property test
 * (tests/hostlogic/read_fence_props.c) all take them from here.
 *
 * A fence on a replica that knew term t and leader L takes L's committed entry count K, then CONFIRMS that no leader of
 * a newer term can exist: a majority of the group's N members still carries a SID of term <= t.  That is sound only
 * because a voter moves its SID to the candidate's term BEFORE it acks the vote (dare_entry.c: elect): a newer leader
 * needs N/2 + 1 such acks, so a majority at <= t after K was read means none had been elected by then.  A control plane
 * that acks votes without moving the SID gets no guarantee from a fence.  The fence then waits until this replica's
 * committed-and-held count reaches K and the entry at that count carries a term >= t: Raft's "the leader has committed
 * an entry of its own term" (a new leader's commit may lag what an earlier leader committed until its blank CONFIG
 * commits).
 */
#ifndef APUS_FENCE_RULE_H
#define APUS_FENCE_RULE_H
#include <stdint.h>
#ifdef __CUDACC__
#define APUS_FENCE_HD __host__ __device__ __forceinline__
#else
#define APUS_FENCE_HD static inline
#endif

#define APUS_SID_TERM(sid) ((sid) >> 9)           /* SID [TERM|L|IDX] (dare_server.h:46-61) */

/* member i of the group counts towards the confirmation: its region is mapped here, and its SID is still at term <= t */
APUS_FENCE_HD uint32_t rf_member_counts(int connected, uint64_t sid, uint64_t t)
{
    return connected && APUS_SID_TERM(sid) <= t ? 1u : 0u;
}
/* the confirmation of a fence of an N-member group, from the number of members that count */
APUS_FENCE_HD int rf_confirmed(uint32_t counted, uint32_t n)
{
    return counted >= n / 2 + 1;
}
/* the READY test, polled on this replica's own consumer record: `held` committed entries held, the commit K taken from
 * the leader, and the header {idx, term} of the entry that the offset index names for idx `held` (a header whose idx is
 * not `held` is an entry of another lap: not ready, poll again).  A replica that holds no committed entry is never ready */
APUS_FENCE_HD int rf_ready(uint64_t held, uint64_t k, uint64_t entry_idx, uint64_t entry_term, uint64_t t)
{
    return held != 0 && held >= k && entry_idx == held && entry_term >= t;
}
#endif
