"""The commit rule with followers down, against the oracle's partial rounds (orc.Cluster.round(live=...)).

Every replica runs in its own launch (engine_util.launch_each), so single followers can be stopped and relaunched in
the same term -- what dare_entry.c does after a false suspicion (DESIGN s7).  While a follower is stopped the leader
keeps storing entry bytes, index words and publishes into its HBM; it acks nothing and its header does not move.
On relaunch it acks everything it missed.

Reply bytes: the engine pushes an entry's composed image (reply bytes zero) to every follower when it publishes it; the
reference's RDMA WRITE to a follower that lags copies the leader's bytes as they are THEN, reply bytes of the followers
that acked in the meantime included (the oracle does the same).  So on a follower that has been down, the other
replicas' reply bytes are masked; its own reply byte, and everything on the leader and on followers that never
stopped, is compared exactly."""
import threading
import time

import numpy as np
import pytest

import engine_util as EU
import streams as S
from apus_b200 import engine as E
from engine_util import MODES, devices_for, eng, wait_for  # noqa: F401
from shadow import Pair

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


# Up to 7 replicas: every replica is a launch of its own that stays resident, and a process has 8 hardware work queues
# by default (CUDA_DEVICE_MAX_CONNECTIONS); a ninth concurrent launch can queue behind a resident one and never start.
# Larger groups are covered by the oracle's own test (tests/test_oracle_quorum.py, N up to 13).
QUORUM_CASES = [(2, 0, "index_earlyack"), (3, 0, "walk_fenced"), (4, 0, "index_earlyack"), (5, 0, "walk_earlyack"),
                (6, 0, "index_fenced"), (7, 0, "walk_fenced"),
                (5, 3, "index_earlyack"), (6, 5, "walk_fenced")]


@pytest.mark.parametrize("n,lead,mode", QUORUM_CASES, ids=[f"n{n}-leader{ld}-{m}" for n, ld, m in QUORUM_CASES])
def test_no_commit_without_a_majority(eng, orc, n, lead, mode):
    """Followers stop one at a time, each at a quiescent point and at a different depth of the stream; after every
    stop a bulk burst and a few lone requests.  While a majority (size/2+1, the leader included) is up everything
    commits and every replica is exact against the oracle; below it nothing commits for QUIET_S, while the leader's
    reply bytes show exactly who acked what.  Then the followers come back in reverse order: the commit resumes when,
    and only when, the majority is back."""
    p = Pair(eng, orc, n, lead, 1 << 20, MODES[mode], seed=100 * n + lead)
    try:
        order = [int(x) for x in p.rng.permutation(p.followers)]
        for i in order:
            p.step(int(p.rng.integers(10, 40)), 0)           # a different depth for every stop
            p.stop(i)
            p.step(int(p.rng.integers(20, 60)), 3)
        for i in reversed(order):
            before = (p.leader.committed(), p.leader.progress(), p.leader.offsets()["commit"])
            p.relaunch(i)
            if p.has_quorum():
                p.check_committed()
            else:
                p.check_not_committed(*before)
        p.step(30, 3)                                        # everybody up: the oracle has run full rounds
        p.g.stop()
        p.check_offsets()
        p.check_images()
    finally:
        p.close()


@pytest.mark.parametrize("mode", ["index_earlyack", "walk_fenced"])
@pytest.mark.parametrize("n", [3, 5])
def test_express_with_a_lagging_follower(eng, orc, n, mode):
    """A stopped follower misses lone requests.  The first one after the stop finds every follower caught up and goes
    out self-certified: the stopped follower verifies it against its own HBM after the relaunch.  With k > 1 it lags,
    the publishes are fenced, and it takes the k entries in one step.  The express path runs in both phases."""
    # (APUS_F_PROFILE: followers count the self-certified publishes they verified, stats phase_ns[0])
    p = Pair(eng, orc, n, 0, 1 << 20, MODES[mode] | E.F_PROFILE, seed=n)
    try:
        f = p.followers[-1]
        for k, certs in ((1, 1), (4, 0)):
            p.lone(5)
            p.check_committed()
            p.stop(f)
            time.sleep(0.01)
            x0 = p.leader.stats()["turn_ns"][5]
            v0 = p.rep(f).stats()["phase_ns"][0]
            p.lone(k)
            # (worker 0 copies its counters to the stats block every few hundred idle polls)
            wait_for(lambda: p.leader.stats()["turn_ns"][5] > x0, "the express path to run", timeout=2.0)
            p.check_committed()
            p.relaunch(f)
            p.check_committed()
            assert p.rep(f).stats()["phase_ns"][0] - v0 == certs, (k, p.rep(f).stats()["phase_ns"])
        p.lone(3)
        p.check_committed()
    finally:
        p.close()


@pytest.mark.parametrize("n", [4, 5])
def test_commit_invariants_under_follower_churn(eng, orc, n):
    """One thread streams requests while followers stop and come back on a seeded schedule, never below a majority.
    Sampled: the committed count never decreases and never passes what a majority holds (read after it: the counts
    only grow); no follower's commit is ahead of its end (I4).  Without pruning the final images do not depend on the
    interleaving: they equal the oracle's full run."""
    L = 1 << 21
    quorum = n // 2 + 1
    g = eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES["index_earlyack"])
    stream = S.ragged_stream(4000, 200, conns=3, seed=n)
    rng = np.random.default_rng(n)
    err = {}
    done, quit_ = threading.Event(), threading.Event()

    def feed():
        try:
            k = 0
            while k < len(stream) and not quit_.is_set():
                m = int(rng.integers(1, 40))
                t = g.submit_stream(stream[k:k + m]) if m > 1 else g.submit(*stream[k])
                k += m
                g.leader.wait_committed(t, 10_000_000)
                time.sleep(float(rng.uniform(0.002, 0.006)))       # a stream that outlasts many stops and relaunches
        except Exception as ex:                              # noqa: BLE001 - surfaced by the test
            err["feed"] = f"{type(ex).__name__}: {ex}"
        finally:
            done.set()

    th = threading.Thread(target=feed, daemon=True)
    live, down = list(range(1, n)), []
    try:
        EU.launch_each(eng, g.replicas)
        g.leader.wait_committed(g.prologue())
        th.start()
        last, samples, events = 0, 0, 0
        sched = np.random.default_rng(1000 + n)
        while not done.is_set():
            committed = g.leader.committed()
            # a follower stores its ack word into the leader before its `entries_acked` (reply bytes in between):
            # read the counts a moment later -- they only grow, so the bound stays sound
            time.sleep(0.001)
            votes = sorted([g.leader.stats()["entries_published"]] +
                           [g.replicas[i].stats()["entries_acked"] for i in range(1, n)], reverse=True)
            assert committed >= last, (last, committed)
            assert committed <= votes[quorum - 1], (committed, votes)
            last = committed
            for i in range(1, n):
                # (the ring is not lapped: ring order is plain order.)  A running follower stores `end` before the
                # `commit` that follows it, but the host's 64 B read of the header is not ordered with those stores:
                # a violation must still be there a moment later
                o = g.replicas[i].offsets()
                if o["end"] != L and o["commit"] > o["end"]:
                    time.sleep(0.002)
                    o = g.replicas[i].offsets()
                    assert o["end"] != L and o["commit"] <= o["end"], f"I4: follower {i} {o}"
            samples += 1
            if sched.random() < 0.3:
                can_stop = 1 + len(live) - 1 >= quorum
                if down and (sched.random() < 0.5 or not can_stop):
                    i = down.pop(int(sched.integers(0, len(down))))
                    EU.launch_each(eng, [g.replicas[i]])
                    live.append(i)
                    events += 1
                elif can_stop:
                    i = live.pop(int(sched.integers(0, len(live))))
                    EU.stop_each(eng, [g.replicas[i]])
                    down.append(i)
                    events += 1
            time.sleep(float(sched.uniform(0.001, 0.01)))
        th.join(timeout=30)
        assert "feed" not in err, err
        while down:
            i = down.pop()
            EU.launch_each(eng, [g.replicas[i]])
        t = g.tickets
        g.leader.wait_committed(t)
        wait_for(lambda: all(g.replicas[i].stats()["entries_acked"] >= t and
                             g.replicas[i].offsets()["commit"] == g.leader.offsets()["commit"] for i in range(1, n)),
                 "every follower caught up")
        g.stop()
        assert events >= 10 and samples >= 50, (events, samples)
        c = EU.oracle_cluster(orc, n, L, stream)
        try:
            EU.compare_group_to_oracle(g, c, exact=True)
        finally:
            c.close()
    finally:
        quit_.set()
        if th.is_alive():
            th.join(timeout=30)
        try:
            for i in down:                                   # (after a failure) everybody up before the stop
                EU.launch_each(eng, [g.replicas[i]])
            g.stop()
        except Exception:                                    # noqa: BLE001 - the test's own failure is the report
            pass
        g.close()
