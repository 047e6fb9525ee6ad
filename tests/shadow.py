"""An engine group shadowed by an oracle cluster, for the GPU tests of the commit rule with followers down
(tests/test_gpu_quorum.py) and of leader take-over (tests/test_gpu_takeover.py): every replica runs in its own launch
(engine_util.launch_each), so single followers can be stopped and relaunched, and the control plane of a take-over is
driven on stopped replicas the way dare_entry.c's elect() drives it.  The mask rules for the images are stated in those
two test modules."""
import ctypes as C
import time

import numpy as np

import engine_util as EU
import orc as O
import scenarios
import streams as S
from apus_b200 import engine as E

u64 = C.c_uint64


def mask_others(img, ents, me):
    """zero the reply bytes of every replica but `me`"""
    img = img.copy()
    for off, _ in ents:
        own = img[off + 28 + me]
        img[off + 28:off + 41] = 0
        img[off + 28 + me] = own
    return img


class Pair:
    """One engine group (resident, one launch per replica) and the oracle cluster that shadows it."""

    def __init__(self, eng, orc, n, lead, L, flags, seed):
        self.eng, self.n, self.lead, self.L = eng, n, lead, L
        self.quorum = n // 2 + 1
        self.followers = [i for i in range(n) if i != lead]
        self.live = set(self.followers)
        self.rejoined = set()                                # followers that have been down at least once
        self.rng = np.random.default_rng(seed)
        self.g = eng.Group(n, devices=EU.devices_for(eng, n), leader=lead, log_size=L, flags=flags)
        orc.set_rules(O.RULES_ENGINE)
        self.c = O.Cluster(orc, n, leader=lead, term=1, length=L)
        self.conn, self.rid = lead << 8, 1
        EU.launch_each(eng, self.g.replicas)
        self.g.prologue()
        self.c.prologue()
        self.lone(1)                                         # the CONNECT
        self.rounds()
        self.settle()

    def close(self):
        try:
            # (after a failure) bring the majority back first: a leader stopped with uncommitted entries waits for them
            for i in self.followers:
                if i not in self.live:
                    self.relaunch(i)
            self.leader.wait_committed(self.g.tickets, 5_000_000)
        except Exception:                                    # noqa: BLE001 - the test's own failure is the report
            pass
        try:
            self.g.stop()
        finally:
            self.g.close()
            self.c.close()

    @property
    def leader(self):
        return self.g.leader

    def rep(self, i):
        return self.g.replicas[i]

    def has_quorum(self):
        return 1 + len(self.live) >= self.quorum

    def _next(self, max_len):
        if self.rid == 1:
            req = (S.CONNECT, self.conn, 1, b"")
        else:
            ln = int(self.rng.integers(0, max_len + 1))
            req = (S.SEND, self.conn, self.rid, self.rng.integers(0, 256, size=ln, dtype=np.uint8).tobytes())
        self.rid += 1
        typ, clt, rid, payload = req
        assert self.c.submit(typ, clt, rid, O.cmd_image(payload)) != 0, f"the oracle refused request {rid}"
        return req

    def burst(self, k):
        """k requests of up to 300 B in one flush: the tile path"""
        self.g.submit_stream([self._next(300) for _ in range(k)])

    def lone(self, k):
        """k requests of up to 78 B (an inline image), one at a time: the express path.  Each waits for its commit,
        or, without a quorum, until it is published"""
        for _ in range(k):
            t = self.g.submit(*self._next(78))
            if self.has_quorum():
                self.leader.wait_committed(t, 5_000_000)
            else:
                self.wait_published(t)

    def wait_published(self, t):
        EU.wait_for(lambda: self.leader.stats()["entries_published"] >= t, f"entry {t} published")

    def rounds(self):
        self.c.round(live=self.live)
        self.c.round(live=self.live)

    def settle(self):
        """every live follower has acked everything published and followed the leader's commit offset"""
        t = self.g.tickets
        self.wait_published(t)
        lc = self.leader.offsets()["commit"]
        for i in self.live:
            r = self.rep(i)
            EU.wait_for(lambda: r.stats()["entries_acked"] >= t and (not self.has_quorum() or r.offsets()["commit"] == lc),
                        f"follower {i} acked {t}")

    def stop(self, i):
        EU.stop_each(self.eng, [self.rep(i)])
        self.live.discard(i)

    def relaunch(self, i):
        EU.launch_each(self.eng, [self.rep(i)])
        self.live.add(i)
        self.rejoined.add(i)

    def check_images(self):
        """leader exact over [0, its end); every follower over [0, its end) (the engine's leader also stores beyond a
        stopped follower's end)"""
        L, lead = self.L, self.lead
        lo = self.c.offsets(lead)
        limg_o = self.c.image(lead)
        ents = O.walk_entries(limg_o, 0, lo["end"], L)
        limg_e = self.leader.image()
        d = np.nonzero(limg_e[:lo["end"]] != limg_o[:lo["end"]])[0]
        assert len(d) == 0, f"leader: {len(d)} bytes differ, first at {int(d[0])}"
        for i in self.followers:
            end = self.c.offsets(i)["end"]
            ei, oi = self.rep(i).image(0, end), self.c.image(i, 0, end)
            if i in self.rejoined:
                fents = [(o, s) for o, s in ents if o + s <= end]
                ei, oi = mask_others(ei, fents, i), mask_others(oi, fents, i)
            d = np.nonzero(ei != oi)[0]
            assert len(d) == 0, f"follower {i} (live {i in self.live}): {len(d)} bytes differ, first at {int(d[0])}"

    def check_offsets(self, keys_leader=("head", "apply", "commit", "end", "tail")):
        for i in range(self.n):
            eo, oo = self.rep(i).offsets(), self.c.offsets(i)
            keys = keys_leader if i == self.lead else ("head", "apply", "commit", "end")
            assert {k: eo[k] for k in keys} == {k: oo[k] for k in keys}, (i, i in self.live, eo, oo)
            if i != self.lead:
                assert eo["commit"] <= eo["end"], f"I4: follower {i} commit {eo['commit']} beyond its end {eo['end']}"

    def check_committed(self):
        """a quorum is up: everything commits; exact against the oracle"""
        self.leader.wait_committed(self.g.tickets, 5_000_000)
        self.rounds()
        self.settle()
        assert self.leader.committed() == self.g.tickets, (self.leader.committed(), self.g.tickets)
        self.check_offsets()
        self.check_images()

    def check_not_committed(self, committed0, progress0, lcommit0):
        """no quorum: the new entries are published and acked by the live followers, and nothing commits"""
        self.rounds()
        self.settle()
        t_end = time.time() + EU.QUIET_S
        while time.time() < t_end:
            assert self.leader.committed() == committed0, (self.leader.committed(), committed0)
            assert self.leader.progress() == progress0, (self.leader.progress(), progress0)
            assert self.leader.offsets()["commit"] == lcommit0, (self.leader.offsets(), lcommit0)
            time.sleep(0.005)
        assert self.leader.stats()["entries_published"] == self.g.tickets, \
            (self.leader.stats()["entries_published"], self.g.tickets)
        assert self.c.offsets(self.lead)["commit"] == lcommit0, (self.c.offsets(self.lead), lcommit0)
        self.check_offsets(keys_leader=("head", "apply", "commit"))   # the leader's header `end` follows its commit
        self.check_images()

    def step(self, k_burst, k_lone):
        before = (self.leader.committed(), self.leader.progress(), self.leader.offsets()["commit"])
        self.burst(k_burst)
        self.lone(k_lone)
        if self.has_quorum():
            self.check_committed()
        else:
            self.check_not_committed(*before)


def sid(term, leader, idx):
    return (term << 9) | ((1 if leader else 0) << 8) | idx


class Takeover(Pair):
    """Pair whose leader can change: take_over() elects a new one among the survivors."""

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
        EU.wait_for(lambda: self.leader.stats()["entries_published"] >= self.idx_base + t, f"ticket {t} published")

    def settle(self):
        """every live follower has acked everything published and followed the leader's commit offset (tickets restart
        at 1 with every leader; entry counts do not)"""
        t = self.g.tickets
        self.wait_published(t)
        lc = self.leader.offsets()["commit"]
        for i in self.live:
            r = self.rep(i)
            EU.wait_for(lambda: r.stats()["entries_acked"] >= self.idx_base + t and
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
        assert self.leader.stats()["entries_published"] == last, (self.leader.stats()["entries_published"], last)
        assert self.leader.committed() == self.g.tickets, (self.leader.committed(), self.g.tickets)
        for off, _ in ents:
            if int.from_bytes(img[off + 8:off + 16].tobytes(), "little") == self.term:
                assert img[off + 27] == self.lead, f"entry at {off}: sender {img[off + 27]}, leader {self.lead}"


def elect(eng, g, c, survivors, winner, voters, term):
    """The control plane of a take-over, driven as dare_entry.c's elect() drives it, with every replica stopped, and the
    oracle cluster `c` shadowing it.  `survivors`: every replica but the dead leader.  Returns ({survivor: commit
    offset}, {voter: shared end}, {voter: (from, to) of a non-empty resent range})."""
    L, dead = g.replicas[0].log_len, g.leader_idx
    lib = eng.lib()
    rep = g.replicas
    for i in survivors:
        E._ck(lib.apus_replica_disconnect(rep[i].h, dead), "apus_replica_disconnect")
    # what every survivor votes on, against the oracle
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
    # the oracle: adoption, then the adjustment of every voter (before the blank CONFIG, in the engine's order)
    c.take_over(winner, term, {v: commits[v] for v in voters})
    wend = c.offsets(winner)["end"]
    shared = {v: c.adjust(v) for v in voters}
    for v in voters:
        # the resend itself: a one-sided write that lands whether or not the voter runs (the engine's adjustment copies
        # the bytes at once), acked when the voter runs again
        c.replicate(v)
    # the engine
    E._ck(lib.apus_replica_set_role(rep[winner].h, winner, term), "apus_replica_set_role (winner)")
    for i in survivors:
        if i != winner and i not in voters:
            E._ck(lib.apus_replica_disconnect(rep[winner].h, i), "apus_replica_disconnect")
    resent = {}
    for v in voters:
        got = u64()
        E._ck(lib.apus_ctl_adjust_follower(rep[winner].h, v, sid(term, 1, winner), C.byref(got)),
              "apus_ctl_adjust_follower")
        gap = (wend - shared[v]) % L if wend != L else 0
        assert int(got.value) == gap, \
            f"voter {v}: resent {int(got.value)} bytes, the shared end {shared[v]} and the winner's end {wend} leave {gap}"
        if gap:
            resent[v] = (shared[v], wend)
            check_resent(rep[v], c, v, winner, shared[v], wend)
    for v in voters:
        E._ck(lib.apus_replica_set_role(rep[v].h, winner, term), "apus_replica_set_role (voter)")
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


def lap_stream(n_req, conn, seed):
    """one CONNECT, then SENDs of 0..100 B with one of 700..1500 B every 20th: some 400 entries a lap of 64 KiB, so the
    offset index (1024 words) wraps every few laps, and ghost headers where a long one meets the ring's end"""
    rng = np.random.default_rng(seed)
    out = [(S.CONNECT, conn, 1, b"")]
    for i in range(n_req):
        ln = int(rng.integers(700, 1501)) if i % 20 == 19 else int(rng.integers(0, 101))
        out.append((S.SEND, conn, 2 + i, rng.integers(0, 256, ln, dtype=np.uint8).tobytes()))
    return out


def check_heads(reps, rp, what, idxs=None):
    """every replica of `reps` (the oracle's replicas `idxs`, by default 0, 1, ...) holds the head of the last committed
    HEAD entry, as the oracle's poll_head has it: the leader holds it, the followers adopted it (poll_config_entries)"""
    want = rp.last_committed_head()
    for r, i in zip(reps, range(len(reps)) if idxs is None else idxs):
        got = r.offsets()["head"]
        assert got == want == rp.c.offsets(i)["head"], f"{what}: replica {i} head {got}, last HEAD carries {want}"
