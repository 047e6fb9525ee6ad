"""shadow.Takeover on the device submission ring, for the GPU tests of resident submitters through take-overs
(tests/test_gpu_submit_takeover.py), with two moves those tests need beside the ones Takeover makes: the old leader may
vote and rejoin as a follower, so that one replica can lead twice; and the winner's host may submit (its blank CONFIG)
once the roles are set, before its first launch hands the ring to a dormant submitter.  Importing this module starts no
CUDA context."""
import ctypes as C

import engine_util as EU
import orc as O
import scenarios
import shadow
from apus_b200 import engine as E

u64 = C.c_uint64


class _DeviceRing:
    """the engine module, with every Group created on the device submission ring"""

    def __init__(self, eng):
        self._eng = eng

    def __getattr__(self, name):
        return getattr(self._eng, name)

    def Group(self, *a, **kw):
        return self._eng.Group(*a, ring_mode=self._eng.RING_DEVICE, **kw)


class DeviceTakeover(shadow.Takeover):
    """Takeover whose group submits through the HBM ring (APUS_RING_DEVICE)"""

    def __init__(self, eng, orc, n, L, flags, seed):
        super().__init__(_DeviceRing(eng), orc, n, L, flags, seed)

    def take_over(self, winner, voters, check_commit=True, old_votes=False, before_launch=None):
        """Takeover.take_over; `old_votes`: the old leader stays a member, stays connected and may be among the voters
        (it rejoins as a follower when it is launched again); `before_launch()` runs once the roles are set, before the
        winner's first launch"""
        launch, elect = EU.launch_each, shadow.elect

        def first_launch(*a, **kw):
            EU.launch_each = launch
            if before_launch is not None:
                before_launch()
            return launch(*a, **kw)
        EU.launch_each = first_launch
        if old_votes:
            shadow.elect = elect_keeping_old_leader
        try:
            return super().take_over(winner, voters, check_commit)
        finally:
            EU.launch_each, shadow.elect = launch, elect


def elect_keeping_old_leader(eng, g, c, survivors, winner, voters, term):
    """shadow.elect with the old leader among the survivors: it stays connected and may vote.  The engine's adjustment
    of the old leader resends from where old_leader_shares says"""
    L, dead = g.replicas[0].log_len, g.leader_idx
    survivors = sorted(set(survivors) | {dead})
    lib = eng.lib()
    rep = g.replicas
    commits = {}
    for i in survivors:
        idx, tm, commit, end = u64(), u64(), u64(), u64()
        E._ck(lib.apus_ctl_last_entry(rep[i].h, C.byref(idx), C.byref(tm), C.byref(commit), C.byref(end)),
              "apus_ctl_last_entry")
        assert (int(tm.value), int(idx.value)) == scenarios.last_entry(c, i), f"replica {i}: last (term, idx)"
        oo = c.offsets(i)
        assert (int(commit.value), int(end.value)) == (oo["commit"], oo["end"]), f"replica {i}: commit, end {oo}"
        commits[i] = int(commit.value)
    for v in voters:
        E._ck(lib.apus_ctl_send_vote_ack(rep[v].h, winner, commits[v]), "apus_ctl_send_vote_ack")
    c.take_over(winner, term, {v: commits[v] for v in voters})
    wend = c.offsets(winner)["end"]
    shared = {v: c.adjust(v) for v in voters}
    for v in voters:
        c.replicate(v)
    E._ck(lib.apus_replica_set_role(rep[winner].h, winner, term), "apus_replica_set_role (winner)")
    for i in survivors:
        if i != winner and i not in voters:
            E._ck(lib.apus_replica_disconnect(rep[winner].h, i), "apus_replica_disconnect")
    resent = {}
    for v in voters:
        got = u64()
        E._ck(lib.apus_ctl_adjust_follower(rep[winner].h, v, shadow.sid(term, 1, winner), C.byref(got)),
              "apus_ctl_adjust_follower")
        frm = old_leader_shares(c, winner, term - 1) if v == dead else shared[v]
        gap = (wend - frm) % L if wend != L else 0
        assert int(got.value) == gap, \
            f"voter {v}: resent {int(got.value)} bytes, from {frm} to the winner's end {wend} leave {gap}"
        if gap:
            resent[v] = (frm, wend)
            shadow.check_resent(rep[v], c, v, winner, frm, wend)
    for v in voters:
        E._ck(lib.apus_replica_set_role(rep[v].h, winner, term), "apus_replica_set_role (voter)")
    g.leader_idx = winner
    for r in rep:
        r.leader = winner
    g.tickets = 0
    return commits, shared, resent


def old_leader_shares(c, winner, led_in):
    """Where the engine's adjustment of the old leader, when it votes, resends from: it recognises the entries the old
    leader received as a follower, not those it appended itself in term `led_in`, so it resends those -- the same
    bytes, reply bytes aside -- from the end of the winner's last entry of an earlier term, or from the winner's head
    when there is none"""
    L, wo, wimg = c.len, c.offsets(winner), c.image(winner)
    frm = wo["head"]
    for off, stride in O.walk_entries(wimg, wo["head"], wo["end"], L) if wo["end"] != L else []:
        if int.from_bytes(wimg[off + 8:off + 16].tobytes(), "little") < led_in:
            frm = (off + stride) % L
    return frm
