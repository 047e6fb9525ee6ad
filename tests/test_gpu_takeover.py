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
import time

import numpy as np
import pytest

import autoprune_replay as AR
import engine_util as EU
import orc as O
import streams as S
from apus_b200 import engine as E
from engine_util import MODES, QUIET_S, devices_for, eng, wait_for  # noqa: F401
from shadow import Takeover, check_heads, elect, lap_stream, watch_commits

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


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
    p = Takeover(eng, orc, n, 1 << 20, MODES[mode] | (0 if express else E.F_NO_EXPRESS), seed=n)
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
    g = eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES["index_earlyack"] | E.F_AUTOPRUNE)
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
            check_heads([g.replicas[1], g.replicas[2]], rp, f"after the new term's launch ending at {rp.end()}", [1, 2])
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
