"""Leader take-over and log adjustment on the engine, shadowed by the oracle (SIM(take_over), SIM(adjust)).

Everything runs in one process with one launch per replica (engine_util.launch_each), as in tests/test_gpu_quorum.py:
states are built only through the protocol, by stopping and relaunching followers while the leader streams.  Nothing is
killed: the old leader's launch is stopped once everything it published is committed (its commit warp would otherwise
wait for the rest), and every survivor disconnects it.  The control plane is then driven the way dare_entry.c's elect()
drives it: vote acks carrying each voter's commit offset, apus_ctl_last_entry on every survivor (against the oracle's
last (term, idx)), apus_replica_set_role on the winner, apus_ctl_adjust_follower for every voter (the bytes it resends
against the oracle's shared end), apus_replica_set_role on the voters, relaunch.

Mask rule for the images.  Every entry a replica holds is compared, reply bytes exactly except in two places:
  - in a voter's resent range (from the shared end to the winner's end at the adjustment), every reply byte: the engine
    resends the winner's bytes and counts the voter as holding them (it acks none), the oracle's voter acks each one;
  - on a replica that has been stopped and relaunched, the other replicas' reply bytes (tests/test_gpu_quorum.py: the
    oracle's lagging copy carries the replies that had reached the leader by then)."""
import ctypes as C
import time

import numpy as np
import pytest

import autoprune_replay as AR
import engine_util as EU
import orc as O
import scenarios
import streams as S
from test_gpu_parity import MODES, devices_for, eng  # noqa: F401
from test_gpu_quorum import QUIET_S, Pair, mask_others, wait_for

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

F_NO_EXPRESS = 0x20                  # leader: no single-warp express path, every publish fenced
F_AUTOPRUNE = 0x4                    # leader: device-side log pruning

u8, u64, vp = C.c_uint8, C.c_uint64, C.c_void_p


def ctl(eng):
    L = eng.lib()
    L.apus_ctl_send_vote_ack.argtypes = [vp, u8, u64]
    L.apus_ctl_last_entry.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.apus_replica_set_role.argtypes = [vp, u8, u64]
    L.apus_ctl_adjust_follower.argtypes = [vp, u8, u64, C.POINTER(u64)]
    L.apus_replica_disconnect.argtypes = [vp, u8]
    return L


def sid(term, leader, idx):
    return (term << 9) | ((1 if leader else 0) << 8) | idx


class Takeover(Pair):
    """Pair (tests/test_gpu_quorum.py) whose leader can change: take_over() elects a new one among the survivors."""

    def __init__(self, eng, orc, n, L, flags, seed):
        self.members = set(range(n))
        self.term = 1
        self.resent = {}                     # voter -> [first, last] idx of the entries it was last resent
        self.idx_base = 0                    # idx of the entry before the current leader's first ticket
        try:
            super().__init__(eng, orc, n, 0, L, flags, seed)
        except BaseException:
            if hasattr(self, "c"):           # the group is up and launched: leave no launch resident
                self.close()
            raise

    def close(self):
        try:
            for i in self.followers:
                if i not in self.live:
                    self.relaunch(i)
            self.leader.wait_committed(self.g.tickets, 5_000_000)
        except Exception:                                    # noqa: BLE001 - the test's own failure is the report
            pass
        try:
            EU.stop_each(self.eng, [self.rep(i) for i in sorted(self.members)])
        finally:
            self.g.close()
            self.c.close()

    def take_over(self, winner, voters, check_commit=True):
        """The old leader's launch stops (everything it published is committed) and the followers still up stop too;
        `winner` takes over with `voters`; the winner and the voters that were up before run again."""
        dead = self.lead
        was_live = set(self.live)
        assert self.leader.committed() == self.g.tickets, "the old leader must have nothing uncommitted"
        EU.stop_each(self.eng, [self.rep(i) for i in sorted(self.live | {dead})])
        self.live.clear()
        self.term += 1
        commits, shared, resent = elect(self.eng, self.g, self.c, sorted(self.members - {dead}), winner, voters, self.term)
        self.lead = winner
        self.members = {winner} | set(voters)
        wimg = self.c.image(winner)
        for v, (a, b) in resent.items():
            idxs = [int.from_bytes(wimg[o:o + 8].tobytes(), "little") for o, _ in O.walk_entries(wimg, a, b, self.L)]
            self.resent[v] = (min(idxs), max(idxs))
        self.followers = sorted(voters)
        self.idx_base = scenarios.last_entry(self.c, winner)[1]
        self.conn, self.rid = winner << 8, 1
        if check_commit:
            assert self.leader.offsets()["commit"] == self.c.offsets(winner)["commit"], \
                "the winner's commit is not the largest its voters granted"
        # run again: the winner and the voters that were up
        EU.launch_each(self.eng, [self.rep(i) for i in sorted((was_live & set(voters)) | {winner})])
        self.live = was_live & set(voters)
        self.rejoined |= set(voters) - was_live
        return commits, shared

    def wait_published(self, t):
        wait_for(lambda: self.leader.stats()["entries_published"] >= self.idx_base + t, f"ticket {t} published")

    def settle(self):
        """every live follower has acked everything published and followed the leader's commit offset (tickets restart
        at 1 with every leader; entry counts do not)"""
        t = self.g.tickets
        self.wait_published(t)
        lc = self.leader.offsets()["commit"]
        for i in self.live:
            r = self.rep(i)
            wait_for(lambda: r.stats()["entries_acked"] >= self.idx_base + t and
                     (not self.has_quorum() or r.offsets()["commit"] == lc), f"follower {i} acked ticket {t}")

    def new_term(self):
        """the blank CONFIG of the new term (dare_server.c:1412-1421) and the CONNECT of the new leader's client"""
        self.g.prologue()
        self.c.prologue()
        self.lone(1)

    def check_images(self):
        L, lead = self.L, self.lead
        lo = self.c.offsets(lead)
        limg_o = self.c.image(lead)
        ents = O.walk_entries(limg_o, lo["head"], lo["end"], L) if lo["end"] != L else []

        def resent(i):
            """the entries voter i was resent, by idx: a later lap over the same bytes is not masked"""
            if i not in self.resent:
                return []
            lo_idx, hi_idx = self.resent[i]
            return [(o, s) for o, s in ents if lo_idx <= int.from_bytes(limg_o[o:o + 8].tobytes(), "little") <= hi_idx]

        for i in sorted(self.members):
            end = self.c.offsets(i)["end"]
            ei, oi = self.rep(i).image(), self.c.image(i)
            if i in self.rejoined:
                ei, oi = mask_others(ei, ents, i), mask_others(oi, ents, i)
            r = resent(i)
            ei, oi = O.mask_replies(ei, r), O.mask_replies(oi, r)
            held = O.walk_entries(oi, self.c.offsets(i)["head"], end, L) if end != L else []
            for off, stride in held:
                d = np.nonzero(ei[off:off + stride] != oi[off:off + stride])[0]
                if len(d):
                    idx = int.from_bytes(oi[off:off + 8].tobytes(), "little")
                    raise AssertionError(f"replica {i} (leader {lead}, live {i in self.live}): entry idx {idx} at {off}: "
                                         f"{len(d)} bytes differ, first byte {off + int(d[0])} (+{int(d[0])}): engine "
                                         f"{int(ei[off + d[0]])} oracle {int(oi[off + d[0]])}")

    def check_offsets(self, keys_leader=("head", "apply", "commit", "end", "tail")):
        for i in sorted(self.members):
            eo, oo = self.rep(i).offsets(), self.c.offsets(i)
            keys = keys_leader if i == self.lead else ("head", "apply", "commit", "end")
            assert {k: eo[k] for k in keys} == {k: oo[k] for k in keys}, (i, i == self.lead, i in self.live, eo, oo)

    def check_stamps(self):
        """entries of the current term carry it and the leader as sender; the leader has published every entry it
        holds and committed every ticket"""
        lo = self.c.offsets(self.lead)
        img = self.leader.image()
        ents = O.walk_entries(img, lo["head"], lo["end"], self.L)
        last = int.from_bytes(img[ents[-1][0]:ents[-1][0] + 8].tobytes(), "little")
        assert self.leader.stats()["entries_published"] == last
        assert self.leader.committed() == self.g.tickets
        for off, _ in ents:
            if int.from_bytes(img[off + 8:off + 16].tobytes(), "little") == self.term:
                assert img[off + 27] == self.lead, f"entry at {off}: sender {img[off + 27]}, leader {self.lead}"


def _ck(rc, what):
    from apus_b200 import engine as E
    E._ck(rc, what)


def elect(eng, g, c, survivors, winner, voters, term):
    """The control plane of a take-over, driven as dare_entry.c's elect() drives it, with every replica stopped, and the
    oracle cluster `c` shadowing it.  `survivors`: every replica but the dead leader.  Returns ({survivor: commit
    offset}, {voter: shared end}, {voter: (from, to) of a non-empty resent range})."""
    L, dead = g.replicas[0].log_len, g.leader_idx
    lib = ctl(eng)
    rep = g.replicas
    for i in survivors:
        _ck(lib.apus_replica_disconnect(rep[i].h, dead), "apus_replica_disconnect")
    # what every survivor votes on, against the oracle
    commits = {}
    for i in survivors:
        idx, tm, commit, end = u64(), u64(), u64(), u64()
        _ck(lib.apus_ctl_last_entry(rep[i].h, C.byref(idx), C.byref(tm), C.byref(commit), C.byref(end)),
            "apus_ctl_last_entry")
        assert (int(tm.value), int(idx.value)) == scenarios.last_entry(c, i), f"replica {i}: last (term, idx)"
        oo = c.offsets(i)
        assert (int(commit.value), int(end.value)) == (oo["commit"], oo["end"]), f"replica {i}: commit, end {oo}"
        commits[i] = int(commit.value)
    for v in voters:
        _ck(lib.apus_ctl_send_vote_ack(rep[v].h, winner, commits[v]), "apus_ctl_send_vote_ack")
    # the oracle: adoption, then the adjustment of every voter (before the blank CONFIG, in the engine's order)
    c.take_over(winner, term, {v: commits[v] for v in voters})
    wend = c.offsets(winner)["end"]
    shared = {v: c.adjust(v) for v in voters}
    for v in voters:
        # the resend itself: a one-sided write that lands whether or not the voter runs (the engine's adjustment copies
        # the bytes at once), acked when the voter runs again
        c.replicate(v)
    # the engine
    _ck(lib.apus_replica_set_role(rep[winner].h, winner, term), "apus_replica_set_role (winner)")
    for i in survivors:
        if i != winner and i not in voters:
            _ck(lib.apus_replica_disconnect(rep[winner].h, i), "apus_replica_disconnect")
    resent = {}
    for v in voters:
        got = u64()
        _ck(lib.apus_ctl_adjust_follower(rep[winner].h, v, sid(term, 1, winner), C.byref(got)), "apus_ctl_adjust_follower")
        gap = (wend - shared[v]) % L if wend != L else 0
        assert int(got.value) == gap, \
            f"voter {v}: resent {int(got.value)} bytes, the shared end {shared[v]} and the winner's end {wend} leave {gap}"
        if gap:
            resent[v] = (shared[v], wend)
            check_resent(rep[v], c, v, winner, shared[v], wend)
    for v in voters:
        _ck(lib.apus_replica_set_role(rep[v].h, winner, term), "apus_replica_set_role (voter)")
    g.leader_idx = winner
    for r in rep:
        r.leader = winner
    g.tickets = 0
    return commits, shared, resent


def check_resent(r, c, v, winner, a, b):
    """right after the adjustment: voter v holds the winner's entries of [a, b), reply bytes aside"""
    L = c.len
    wimg = c.image(winner)
    ents = O.walk_entries(wimg, a, b, L)
    ei, oi = O.mask_replies(r.image(), ents), O.mask_replies(c.image(v), ents)
    for off, stride in ents:
        d = np.nonzero(ei[off:off + stride] != oi[off:off + stride])[0]
        if len(d):
            raise AssertionError(f"voter {v}: resent entry idx {int.from_bytes(wimg[off:off + 8].tobytes(), 'little')} at "
                                 f"{off}: {len(d)} bytes differ from the winner's, first byte {off + int(d[0])} "
                                 f"(+{int(d[0])}): engine {int(ei[off + d[0]])} oracle {int(oi[off + d[0]])}")


def watch_commits(p, secs):
    """for `secs`: no follower's header commit and no follower host's commit offset is ahead of the leader's commit
    (the ring does not lap here: ring order is plain order), and every commit only grows"""
    lead_c = p.leader.offsets()["commit"]
    last = {i: p.rep(i).offsets()["commit"] for i in p.live}
    t_end = time.time() + secs
    while time.time() < t_end:
        for i in p.live:
            fc = p.rep(i).offsets()["commit"]
            hc = p.rep(i).progress()[0]
            assert fc <= lead_c and hc <= lead_c, \
                f"follower {i}: commit {fc} (host {hc}) is ahead of leader {p.lead}'s commit {lead_c}"
            assert fc >= last[i], f"follower {i}: commit went back from {last[i]} to {fc}"
            last[i] = fc
        lc = p.leader.offsets()["commit"]
        assert lc >= lead_c, f"leader {p.lead}: commit went back from {lead_c} to {lc}"
        lead_c = lc
        time.sleep(0.002)


@pytest.mark.parametrize("mode", list(MODES))
def test_voters_commit_ahead_of_the_winners(eng, orc, mode):
    """N = 5.  Followers 2-4 stop; a burst is acked by follower 1 alone; 1 stops, 2 and 3 come back and the burst
    commits (1 never hears of it).  The leader stops.  1 wins with voters 2 and 3, whose commit offsets lie past its own.
    3 and 4 stay down, so the new term has no majority: no follower's commit -- in its header or on its host -- may run
    ahead of the new leader's, which must be the largest its voters granted (the oracle's, adopted).  Then 3 comes back:
    the old-term entries commit with the blank CONFIG, and the new term commits exactly as the oracle's."""
    p = Takeover(eng, orc, 5, 1 << 20, MODES[mode], seed=7)
    try:
        p.step(20, 2)
        for i in (2, 3, 4):
            p.stop(i)
        c0 = (p.leader.committed(), p.leader.progress(), p.leader.offsets()["commit"])
        p.burst(30)
        p.check_not_committed(*c0)
        p.stop(1)
        p.relaunch(2)
        p.relaunch(3)
        p.check_committed()
        commits, _ = p.take_over(1, [2, 3], check_commit=False)
        assert commits[2] == commits[3] > commits[1], f"the voters' commit offsets must lie past the winner's: {commits}"
        p.stop(3)                                            # 3 and 4 down: no majority in term 2
        p.g.prologue()
        p.c.prologue()
        p.wait_published(p.g.tickets)
        p.rounds()
        wait_for(lambda: p.rep(2).stats()["entries_acked"] >= p.leader.stats()["entries_published"], "follower 2 acks")
        watch_commits(p, QUIET_S * 2)
        assert p.leader.offsets()["commit"] == p.c.offsets(1)["commit"], \
            f"winner's commit {p.leader.offsets()['commit']}, the oracle's (adopted) {p.c.offsets(1)['commit']}"
        assert p.leader.committed() == 0
        p.relaunch(3)
        p.lone(1)
        p.check_committed()
        p.step(40, 3)
        p.check_stamps()
    finally:
        p.close()


LAGGING = [(3, "index_earlyack", True), (3, "walk_fenced", False), (5, "walk_earlyack", True),
           (5, "index_fenced", False), (7, "index_earlyack", False), (7, "walk_fenced", True)]


@pytest.mark.parametrize("n,mode,express", LAGGING, ids=[f"n{n}-{m}-{'express' if x else 'fenced'}" for n, m, x in LAGGING])
def test_lagging_voter_is_resent_what_it_missed(eng, orc, n, mode, express):
    """A voter stopped early misses several bursts while the majority goes on; the leader stops and the most
    up-to-date follower wins.  The adjustment resends the lagging voter exactly the bytes from its end to the winner's
    (the oracle's remote_end gap), and the new term commits on every voter as in the oracle.  Its lone requests go
    through the express path on the taken-over log (its cached placement and hole prefetch start from the log as the
    take-over left it), or, with the express path off, through fenced publishes."""
    p = Takeover(eng, orc, n, 1 << 20, MODES[mode] | (0 if express else F_NO_EXPRESS), seed=n)
    try:
        lag = n - 1
        p.step(20, 2)
        p.stop(lag)
        p.step(30, 2)
        p.step(25, 1)
        p.rounds()
        winner = 1
        voters = [i for i in range(2, n)]
        _, shared = p.take_over(winner, voters)
        assert lag in p.resent
        p.relaunch(lag)
        p.new_term()
        p.check_committed()
        p.step(30, 3)
        p.check_stamps()
    finally:
        p.close()


@pytest.mark.parametrize("mode", ["index_earlyack", "walk_fenced"])
def test_winner_commits_old_term_entries_with_its_config(eng, orc, mode):
    """N = 5.  Followers 2-4 stop; a burst is acked by follower 1 alone; 1 stops, 2 comes back and the burst commits
    (1 acked it, but never hears of the commit).  The leader stops.  1 wins with voters 3 and 4, which know no more
    than it does: the burst is published but not committed on the winner, and the adjustment resends it to both.  With
    only the winner up, then with one voter, nothing commits -- the burst has no reply bytes on the winner and the
    CONFIG no majority; with both voters the burst commits as a prefix of the CONFIG, exactly as in the oracle."""
    p = Takeover(eng, orc, 5, 1 << 20, MODES[mode], seed=11)
    try:
        p.step(20, 2)
        for i in (2, 3, 4):
            p.stop(i)
        c0 = (p.leader.committed(), p.leader.progress(), p.leader.offsets()["commit"])
        p.burst(30)
        p.check_not_committed(*c0)
        p.stop(1)
        p.relaunch(2)
        p.check_committed()
        commits, shared = p.take_over(1, [3, 4])
        wc = p.leader.offsets()["commit"]
        assert commits[3] == commits[4] == commits[1] == wc < p.leader.offsets()["end"], commits
        assert set(p.resent) == {3, 4}
        p.g.prologue()
        p.c.prologue()
        p.wait_published(p.g.tickets)
        p.rounds()
        for live in ((), (3,)):
            for i in live:
                p.relaunch(i)
            p.settle()
            p.rounds()
            t_end = time.time() + QUIET_S
            while time.time() < t_end:
                assert p.leader.offsets()["commit"] == wc and p.leader.committed() == 0, (live, p.leader.offsets())
                time.sleep(0.005)
            assert p.c.offsets(1)["commit"] == wc
            p.check_offsets(keys_leader=("head", "apply", "commit"))
        p.relaunch(4)
        p.lone(2)
        p.check_committed()
        p.step(30, 2)
        p.check_stamps()
    finally:
        p.close()


def lap_stream(n_req, conn, seed):
    """one CONNECT, then SENDs of 0..100 B with one of 700..1500 B every 20th: some 400 entries a lap of 64 KiB, so the
    offset index (1024 words) wraps every few laps, and ghost headers where a long one meets the ring's end"""
    rng = np.random.default_rng(seed)
    out = [(S.CONNECT, conn, 1, b"")]
    for i in range(n_req):
        ln = int(rng.integers(700, 1501)) if i % 20 == 19 else int(rng.integers(0, 101))
        out.append((S.SEND, conn, 2 + i, rng.integers(0, 256, ln, dtype=np.uint8).tobytes()))
    return out


def test_lapped_resend_on_a_pruning_ring(eng, orc):
    """N = 3 on a 64 KiB ring with device-side pruning (APUS_F_AUTOPRUNE), launches under a third of a lap, HEAD entries
    replayed into the oracle (tests/autoprune_replay.py).  Two laps with everybody up; then follower 2 misses 0.6 of a
    lap, started where that range wraps the ring and its entries' index words wrap the offset index; the leader stops
    and 1 takes over with voter 2.  The resend is two copies across the wrap, with HEAD entries inside it, and the
    index-word copy is two copies across idx_cap.  The new term laps twice with pruning (the dead leader, disconnected,
    must not hold the head back): both survivors' heads against the oracle's poll_head after every launch, the new
    leader's pruning start (apply offsets := head), every byte and offset of both survivors at the end."""
    n, L, cap = 3, 1 << 16, (1 << 16) // 64
    old, new = lap_stream(20_000, 0, 31), lap_stream(20_000, 1 << 8, 32)
    requests = [(O.CONFIG, 0, 0, b"")]
    rp = AR.Replay(orc, n, L)
    g = eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES["index_earlyack"] | F_AUTOPRUNE)
    state = dict(prev=0, k=0, running=[])

    def run(stream, nbytes, live):
        """submit requests of `stream` worth `nbytes` ring bytes and run one launch of the leader and `live` to them"""
        part = []
        while S.stream_bytes(part) < nbytes:
            part.append(stream[state["k"]])
            state["k"] += 1
        requests.extend(part)
        g.submit_stream(part)
        reps = [g.replicas[i] for i in live] + [g.leader]
        state["running"] = reps
        EU.launch_each(eng, reps, target=g.tickets)
        for r in reps:
            r.wait(60_000)
        state["running"] = []
        end = g.leader.offsets()["end"]
        rp.launch(AR.read_launch(g.leader, state["prev"], end, L), requests, live=live)
        state["prev"] = end

    try:
        g.prologue()
        while rp.written < 2 * L:
            run(old, 0.3 * L, [1, 2])
        # on to a point where 0.6 of a lap wraps the ring and crosses a multiple of idx_cap
        while True:
            o = g.leader.offsets()
            e, last = o["end"], g.leader.stats()["entries_published"]
            # (and a head more than an eighth of a lap behind: the pruning rule, due from a quarter of a lap in use, then
            # moves it up to follower 2's apply offset with a HEAD inside the range follower 2 misses)
            if 0.42 * L < e < 0.7 * L and 20 <= cap - last % cap <= 200 and AR.dist(o["head"], e, L) > 0.14 * L:
                break
            assert rp.written < 12 * L, "no point to start the lagging range found"
            run(old, 0.04 * L, [1, 2])
        lag_start, w_lag = g.replicas[2].offsets()["end"], rp.written
        # follower 2 pins the pruning at lag_start: the leader may prune up to there, so a window below 0.85 of a lap
        # never blocks; go on past 0.6 of a lap until a HEAD lies inside it
        while rp.written - w_lag < 0.6 * L or (not [h for h in rp.heads if h.lap_pos >= w_lag] and
                                                rp.written - w_lag < 0.7 * L):
            run(old, 0.1 * L, [1])
        assert [h for h in rp.heads if h.lap_pos >= w_lag], \
            (f"no HEAD entry inside the range follower 2 missed ([{lag_start}, {rp.end()}), {rp.written - w_lag} bytes); "
             f"last HEADs {[(h.off, h.value, h.lap_pos) for h in rp.heads[-3:]]}, window from {w_lag}")
        assert g.leader.committed() == g.tickets
        first, last = g.replicas[2].stats()["entries_acked"] + 1, g.replicas[1].stats()["entries_acked"]
        _, shared, resent = elect(eng, g, rp.c, [1, 2], 1, [2], 2)
        a, b = resent[2]
        assert a == lag_start and b < a, f"the resent range [{a}, {b}) must wrap the ring"
        assert first // cap != last // cap, f"the resent entries' index words {first}..{last} must wrap idx_cap {cap}"
        head = g.replicas[1].offsets()["head"]
        assert g.replicas[1].remote_apply_offsets()[:n] == [head] * n, "set_role: every apply offset starts at head"
        # the new term: the leader is 1, its only follower 2; a CONFIG request stands for the prologue
        requests.append((O.CONFIG, 0, 0, b""))
        g.prologue()
        state["k"], w0 = 0, rp.written
        while rp.written - w0 < 2 * L:
            run(new, 0.3 * L, [2])
            check_heads([g.replicas[1], g.replicas[2]], rp, [1, 2], f"after the new term's launch ending at {rp.end()}")
        for i in (1, 2):
            eo, oo = g.replicas[i].offsets(), rp.c.offsets(i)
            keys = ("head", "apply", "commit", "end") + (("tail",) if i == 1 else ())
            assert {k: eo[k] for k in keys} == {k: oo[k] for k in keys}, (i, eo, oo)
            ei, oi = g.replicas[i].image(), rp.c.image(i)
            d = np.nonzero(ei != oi)[0]
            assert len(d) == 0, f"replica {i}: {len(d)} bytes differ, first at {int(d[0])} (engine {ei[d[0]]} " \
                                f"oracle {oi[d[0]]}); offsets {eo}"
        assert g.leader.committed() == g.tickets
    finally:
        try:
            if state["running"]:
                EU.stop_each(eng, state["running"])
        finally:
            g.close()
            rp.close()


def check_heads(reps, rp, idxs, what):
    """every survivor holds the head of the last committed HEAD entry, as the oracle's poll_head has it"""
    want = rp.last_committed_head()
    for r, i in zip(reps, idxs):
        got = r.offsets()["head"]
        assert got == want == rp.c.offsets(i)["head"], f"{what}: replica {i} head {got}, last HEAD carries {want}"
