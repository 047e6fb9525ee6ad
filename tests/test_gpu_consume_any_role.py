"""Device consumers on every replica, the leader included (APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE).  Every
replica's rows are checked against the request stream and the CPU oracle's log: the leader's consumer delivers every
committed entry of its log, its own tickets included.  The leader's cursor gates its own pruning rule, so a lagging
consumer on the leader must hold the leader back instead of being overwritten.  The control plane (set_role both ways,
log adjustment and its refusal) is checked on stopped replicas.

Every replica here holds a resident launch plus a copy and a consume stream, and the consumers bring torch streams of
their own: more than the 8 hardware queues a process gets by default, and consume work whose stream lands on a resident
launch's queue never runs (DESIGN.md s2, "Device paths beside resident kernels").  So each case runs in a worker
process of this file that sets CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA starts.  Marked gpu."""
import os
import sys
import threading
import time
import types as T

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":
    os.environ["CUDA_DEVICE_MAX_CONNECTIONS"] = "32"         # before anything starts CUDA
    for p in (HERE, os.path.dirname(HERE)):
        if p not in sys.path:
            sys.path.insert(0, p)

import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402
import pytest  # noqa: E402

import autoprune_replay as AR  # noqa: E402
import engine_util as EU  # noqa: E402
import orc as O  # noqa: E402
import streams as S  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consumers import (ANY, Consumer, PackedConsumer, catch_up, check_rows, close_all, consumer_group,  # noqa: E402
                       drain, heads_against_reports, idx_cap, oracle_rows, wait_forwarded_all)
from engine_util import MODES, QUIET_S, devices_for, eng, run_case, submit_all, tensors, wait_for  # noqa: E402,F401
from shadow import Takeover, check_heads, elect, lap_stream, sid, watch_commits  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

FOREVER = EU.FOREVER


# ---- the pytest side: one worker process per case ------------------------------------------------------------------
# N, follower mode, express path, consumer layout, requests from device tensors: every mode, both N, both layouts,
# both batch kinds and the express path on and off each appear with the others
LEADER_CASES = [(3, "index_earlyack", True, "strided", False), (3, "walk_fenced", False, "packed", True),
                (3, "index_fenced", True, "packed", False), (3, "walk_earlyack", False, "strided", True),
                (5, "index_earlyack", False, "packed", True), (5, "walk_fenced", True, "strided", False),
                (5, "index_fenced", False, "strided", True), (5, "walk_earlyack", True, "packed", False)]


@pytest.mark.parametrize("n,mode,express,layout,device_batch", LEADER_CASES,
                         ids=[f"n{n}-{m}-{'express' if x else 'fenced'}-{lay}-{'device' if d else 'host'}"
                              for n, m, x, lay, d in LEADER_CASES])
def test_leader_consumes(eng, n, mode, express, layout, device_batch):
    """a ragged 0..1500 B stream (host batches or one device batch) and closed-loop requests: every replica's rows,
    the leader's included, equal the stream and the oracle's log; every final cursor is the commit offset and is
    forwarded as the apply offset; the logs are byte-equal to the oracle's"""
    run_case(__file__, "leader_consumes", n=n, mode=mode, express=express, layout=layout, device_batch=device_batch)


@pytest.mark.parametrize("layout", ["strided", "packed"])
def test_leader_cursor_gates_pruning(eng, layout):
    """one launch laps a 256 KiB ring several times with APUS_F_AUTOPRUNE while the leader's own consumer lags: every
    HEAD is checked against every replica's cursor reports, the leader's among them, and at least one carries the
    leader's lagging cursor"""
    run_case(__file__, "leader_gates_pruning", layout=layout)


TAKEOVER_CASES = [("voters_ahead", 5, "index_earlyack", True), ("lagging", 3, "index_earlyack", True),
                  ("lagging", 3, "walk_fenced", False), ("lagging", 5, "walk_earlyack", True),
                  ("lagging", 5, "index_fenced", False), ("old_term", 5, "index_earlyack", True)]


@pytest.mark.parametrize("scenario,n,mode,express", TAKEOVER_CASES,
                         ids=[f"{s}-n{n}-{m}-{'express' if x else 'fenced'}" for s, n, m, x in TAKEOVER_CASES])
def test_takeover_with_consumers_everywhere(eng, scenario, n, mode, express):
    """the scenarios of test_gpu_takeover.py with device consumers on every replica, called from threads before, during
    (while the replicas are stopped and roles change) and after the take-over: every member's rows are the oracle's
    committed CSM-like entries of the winner's log in idx order, across both terms; the winner delivers the old-term
    entries it never submitted; the rows of the old leader and of replicas left out are a prefix of them; final cursors
    are the commit offsets; Takeover's image and offset checks pass"""
    run_case(__file__, "takeover", scenario=scenario, n=n, mode=mode, express=express)


def test_lapped_resend_with_consumers_everywhere(eng):
    """test_gpu_takeover.test_lapped_resend_on_a_pruning_ring with a device consumer on every replica: their cursors
    gate the pruning on both sides of the take-over, and the rows of the survivors equal the oracle's replayed log"""
    run_case(__file__, "lapped_resend")


def test_argument_checks(eng):
    """the flag needs APUS_F_DEVICE_APPLY; with it a leader consumes, set_role and adjust_follower accept the replica,
    without it they keep refusing; an adjustment of a peer that shares nothing and whose consumer stands past idx 1,
    with the leader's head pruned past it, is refused and writes nothing"""
    run_case(__file__, "argument_checks")


# ---- the worker side ---------------------------------------------------------------------------------------------
def case_leader_consumes(eng, orc, n, mode, express, layout, device_batch):
    L = 1 << 22
    stream = S.ragged_stream(1500, 1500, conns=4, seed=700 + n, close_every=40)
    nlone, ln = 200, 40
    pl = bytes((k * 131 + 7) & 0xFF for k in range(ln))
    lone = [(S.SEND, 9, 1 + i, pl) for i in range(nlone)]
    base = MODES[mode] | (0 if express else E.F_NO_EXPRESS)
    reps = consumer_group(eng, n, L, base, leader_flags=ANY, follower_flags=[ANY] * (n - 1),
                          ring_mode=E.RING_DEVICE if device_batch else E.RING_HOST_MAPPED)
    try:
        allreq = stream + lone
        if layout == "strided":
            cons = [Consumer(r, 1500, 4096) for r in reps]
        else:
            cons = [PackedConsumer(r, [len(p) for *_, p in allreq], seed=30 + k) for k, r in enumerate(reps)]
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)))
        if device_batch:
            t0 = lead.submit_device(*tensors(stream, lead.device, 1500))
            t = t0 + len(stream) - 1
        else:
            t = submit_all(lead, stream)
        lead.wait_committed(t, 60_000_000)
        lat = lead.closed_loop(nlone, ln, 9, 1)                # one in flight: the express path when it is on
        assert len(lat) == nlone
        last_idx = 1 + len(allreq)
        errs = []

        def run(cn, seed):
            try:
                drain(cn, lambda st: st.next_idx == last_idx + 1, [1, 2, 7, 64, 333, 4096], np.random.default_rng(seed))
            except Exception as e:        # noqa: BLE001 - reported below
                errs.append(e)
        th = [threading.Thread(target=run, args=(cn, 40 + k)) for k, cn in enumerate(cons)]
        for x in th:
            x.start()
        for x in th:
            x.join(300)
            assert not x.is_alive()
        assert not errs, errs
        wait_forwarded_all(reps)
        EU.stop_each(eng, reps)
        c = EU.oracle_cluster(orc, n, L, allreq)
        EU.compare_group_to_oracle(T.SimpleNamespace(n=n, replicas=reps, leader_idx=0), c, exact=True)
        for j, cn in enumerate(cons):
            check_rows(cn.rows, allreq, first_idx=2)
            assert cn.rows == oracle_rows(c, j), f"replica {j}: rows differ from the oracle's log"
            st = reps[j].consume_status()
            assert st.cursor == reps[j].offsets()["commit"] == reps[j].offsets()["apply"] == c.offsets(j)["commit"]
            assert st.next_idx == last_idx + 1 and st.error == 0
        c.close()
        print(f"leader consumed {len(cons[0].rows)} rows in {cons[0].calls} calls")
    finally:
        close_all(eng, reps)


def case_leader_gates_pruning(eng, orc, layout):
    """(test_gpu_consume_device.test_pruning_in_one_launch_replayed with the lagging consumer on the leader) follower
    1's host applies through a recorder, which gives the replay the leader's append sequence; followers 2 and 3 and the
    leader consume on the device, the leader with small max_n and pauses"""
    n, L, ctas = 4, 1 << 18, 2
    stream = S.ragged_stream(int(6.5 * 1.15 * L / 814) + 1, 1500, conns=3, seed=197, close_every=20)
    stride = 1500
    requests = [(O.CONFIG, 0, 0, b"")] + stream
    reps = consumer_group(eng, n, L, leader_flags=E.F_AUTOPRUNE | ANY, ring_slots=1 << 14, ring_bytes=1 << 17, ctas=ctas,
                          follower_flags=[E.F_HOST_APPLY, ANY, ANY])
    rec = AR.Recorder(reps[1], 1, L)
    rp = AR.Replay(orc, n, L)
    lagging = 0
    try:
        who = [0, 2, 3]
        if layout == "strided":
            cons = {i: Consumer(reps[i], stride, 256) for i in who}
        else:
            cons = {i: PackedConsumer(reps[i], [len(p) for *_, p in stream], max_n_cap=256, cap_max=1 << 20, seed=90 + i)
                    for i in who}
        errs, total = [], {}

        def run(cn, lag, seed):
            rng = np.random.default_rng(seed)
            try:
                drain(cn, lambda st: "t" in total and st.next_idx > total["t"] + total["heads"](),
                      [1, 2, 3] if lag else [16, 256], rng, pause=0.002 if lag else 0.0)
            except Exception as e:        # noqa: BLE001 - reported below
                errs.append(e)
        total["heads"] = lambda: reps[0].stats()["auto_heads"]
        th = [threading.Thread(target=run, args=(cons[i], i == lagging, 90 + i)) for i in who]
        rec.start()
        for x in th:
            x.start()
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = submit_all(lead, stream)
        deadline = time.time() + 400
        while lead.committed() < t:
            rec.check()
            assert not errs, errs
            assert time.time() < deadline, f"committed {lead.committed()} of {t}; leader {lead.offsets()}"
            time.sleep(0.005)
        total["t"] = t
        final = lead.offsets()["end"]
        rec.finish(final)
        for x in th:
            x.join(400)
            assert not x.is_alive()
        assert not errs, errs
        wait_forwarded_all([reps[0], reps[2], reps[3]])
        EU.stop_each(eng, reps)

        pieces, flat, src, gaps = AR.recording_pieces([rec.rec], L)
        assert gaps[1] is None, gaps
        hits = []
        on_head = heads_against_reports(L, rec.rec.segs, {1: rec.rec.reports, **{i: cons[i].reports for i in who}},
                                        lagging, hits)
        for c0, lc in pieces:
            rp.launch(lc, requests, replica=src, on_head=on_head)
            for s, b, _ in rec.rec.segs:
                if s + len(b) == c0 + len(lc.buf):
                    AR.compare_read(rp, 1, s, b, flat)
        assert rp.pos == len(requests)
        assert rp.written >= 6 * L, rp.written / L
        assert hits, "no HEAD carried the leader's lagging cursor: the test never gated the pruning rule"
        for cn in cons.values():
            assert cn.at == rp.written
        for i, r in enumerate(reps):
            eo, oo = r.offsets(), rp.c.offsets(i)
            for key in ("end", "commit", "head"):
                assert eo[key] == oo[key], (i, key, eo, oo)
            assert eo["apply"] == final, (i, eo)
            ei, oi = r.image(), rp.c.image(i)
            d = np.nonzero(ei != oi)[0]
            assert len(d) == 0, f"replica {i}: {len(d)} bytes differ, first at {int(d[0])}"
        st = lead.stats()
        assert st["auto_heads"] == len(rp.heads) >= int(rp.written / L), (st["auto_heads"], len(rp.heads))
        AR.assert_heads_have_teeth(rp, rp.c.image(0))
        for cn in cons.values():
            check_rows(cn.rows, stream, first_idx=2)
            st_ = cn.rep.consume_status()
            assert st_.next_idx == t + st["auto_heads"] + 1 and st_.error == 0
        print(f"{rp.written / L:.2f} laps, {len(rp.heads)} HEAD entries, {len(hits)} carried the leader's lagging "
              f"cursor, {cons[lagging].calls} calls of the leader's consumer")
    finally:
        rec.stop.set()
        try:
            EU.stop_each(eng, reps)
        finally:
            for r in reps:
                r.close()
            rp.close()


class AnyTakeover(Takeover):
    """Takeover (shadow.py) with a device consumer on every replica, each called from its own thread with
    max_n from 1 up, whatever the replicas are doing: running, stopped, changing roles"""

    def __init__(self, eng, orc, n, L, flags, seed):
        # the consumers (and their torch streams) must exist before the group's first launch: torch's stream pool,
        # created while replica kernels are resident, waits for them; created after the replicas' own streams, its
        # streams also stay off the queues of the launches (as in case_leader_consumes)
        self.cons = None
        launch = EU.launch_each

        def first_launch(eng_, reps, *a, **kw):
            if self.cons is None:
                self.cons = [Consumer(r, 300, 512) for r in sorted(reps, key=lambda r: r.idx)]
            return launch(eng_, reps, *a, **kw)
        EU.launch_each = first_launch
        try:
            super().__init__(eng, orc, n, L, flags | ANY, seed)
        finally:
            EU.launch_each = launch
        self.halt = threading.Event()
        self.errs = []
        self.threads = [threading.Thread(target=self._run, args=(cn, 50 + k)) for k, cn in enumerate(self.cons)]
        for x in self.threads:
            x.start()

    def _run(self, cn, seed):
        rng = np.random.default_rng(seed)
        try:
            while not self.halt.is_set():
                cn.step(int(rng.choice([1, 2, 5, 64, 512])))
                time.sleep(0.0005)
        except Exception as e:        # noqa: BLE001 - reported by finish()
            self.errs.append(e)

    def check_offsets(self, keys_leader=("head", "apply", "commit", "end", "tail")):
        """the oracle's apply offsets follow the commit; here they are the consumers' cursors (checked by finish())"""
        keys_leader = tuple(k for k in keys_leader if k != "apply")
        for i in sorted(self.members):
            eo, oo = self.rep(i).offsets(), self.c.offsets(i)
            keys = keys_leader if i == self.lead else ("head", "commit", "end")
            assert {k: eo[k] for k in keys} == {k: oo[k] for k in keys}, (i, i == self.lead, i in self.live, eo, oo)

    def halt_consumers(self):
        self.halt.set()
        for x in self.threads:
            x.join(60)
            assert not x.is_alive()

    def finish(self, old_lead):
        """every member catches up to its commit offset; rows against the oracle's winner log"""
        self.halt_consumers()
        assert not self.errs, self.errs
        check_consumers(self.c, self.lead, self.members, self.cons, old_lead)

    def close(self):
        if hasattr(self, "threads"):
            self.halt.set()
            for x in self.threads:
                x.join(60)
        super().close()


def check_consumers(c, lead, members, cons, old_lead, want=None):
    """every member's rows are `want` (default: the oracle's CSM-like entries of the winner's log), with strictly
    increasing idx; every other replica's rows are a prefix of them; the winner delivered the old term's rows"""
    want = oracle_rows(c, lead) if want is None else want
    for i in sorted(members):
        st = catch_up(cons[i])
        rows = cons[i].rows
        first = next((q for q, (a, b) in enumerate(zip(rows, want)) if a != b), None)
        assert rows == want, f"replica {i} (leader {lead}): {len(rows)} rows, want {len(want)}; first difference {first}"
        assert all(rows[q][0] < rows[q + 1][0] for q in range(len(rows) - 1)), f"replica {i}: idx not increasing"
        assert st.error == 0 and st.cursor == cons[i].rep.offsets()["commit"]
    for i in range(len(cons)):
        if i not in members:
            rows = cons[i].rows
            assert rows == want[:len(rows)], f"replica {i}: its rows are not a prefix of the winner's"
    old = [x for x in want if x[2] == (old_lead << 8)]
    assert old and [x for x in cons[lead].rows if x[2] == (old_lead << 8)] == old, \
        "the winner's consumer did not deliver the old term's entries"
    print({i: len(cn.rows) for i, cn in enumerate(cons)}, "rows;", {i: cn.calls for i, cn in enumerate(cons)}, "calls",
          flush=True)


def case_takeover(eng, orc, scenario, n, mode, express):
    flags = MODES[mode] | (0 if express else E.F_NO_EXPRESS)
    p = AnyTakeover(eng, orc, n, 1 << 20, flags, seed=n + 100)
    try:
        if scenario == "voters_ahead":           # test_voters_commit_ahead_of_the_winners
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
            assert commits[2] == commits[3] > commits[1], commits
            p.stop(3)
            p.g.prologue()
            p.c.prologue()
            p.wait_published(p.g.tickets)
            p.rounds()
            wait_for(lambda: p.rep(2).stats()["entries_acked"] >= p.leader.stats()["entries_published"], "follower 2")
            watch_commits(p, QUIET_S * 2)
            assert p.leader.offsets()["commit"] == p.c.offsets(1)["commit"]
            p.relaunch(3)
            p.lone(1)
            p.check_committed()
            p.step(40, 3)
            p.check_stamps()
        elif scenario == "lagging":              # test_lagging_voter_is_resent_what_it_missed
            lag = n - 1
            p.step(20, 2)
            p.stop(lag)
            p.step(30, 2)
            p.step(25, 1)
            p.rounds()
            p.take_over(1, list(range(2, n)))
            assert lag in p.resent
            p.relaunch(lag)
            p.new_term()
            p.check_committed()
            p.step(30, 3)
            p.check_stamps()
        else:                                    # test_winner_commits_old_term_entries_with_its_config
            p.step(20, 2)
            for i in (2, 3, 4):
                p.stop(i)
            c0 = (p.leader.committed(), p.leader.progress(), p.leader.offsets()["commit"])
            p.burst(30)
            p.check_not_committed(*c0)
            p.stop(1)
            p.relaunch(2)
            p.check_committed()
            commits, _ = p.take_over(1, [3, 4])
            wc = p.leader.offsets()["commit"]
            assert commits[3] == commits[4] == commits[1] == wc < p.leader.offsets()["end"], commits
            p.g.prologue()
            p.c.prologue()
            p.wait_published(p.g.tickets)
            p.rounds()
            p.relaunch(3)
            p.settle()
            p.rounds()
            assert p.leader.offsets()["commit"] == wc and p.leader.committed() == 0
            p.relaunch(4)
            p.lone(2)
            p.check_committed()
            p.step(30, 2)
            p.check_stamps()
        p.finish(0)
    finally:
        p.close()


def case_lapped_resend(eng, orc):
    """(test_gpu_takeover.test_lapped_resend_on_a_pruning_ring) N = 3 on a 64 KiB ring with pruning, launches under a
    third of a lap, a device consumer on every replica from its own thread: follower 2 misses 0.6 to 0.7 of a lap, 1
    takes over with voter 2 (a resend across the ring's wrap and the offset index's), and the new term laps twice.  The consumers
    gate the pruning on both sides; the survivors' rows equal the requests of both terms in order"""
    n, L = 3, 1 << 16
    old, new = lap_stream(20_000, 0, 31), lap_stream(20_000, 1 << 8, 32)
    requests = [(O.CONFIG, 0, 0, b"")]
    rp = AR.Replay(orc, n, L)
    g = E.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES["index_earlyack"] | E.F_AUTOPRUNE | ANY)
    cons = [Consumer(r, 1500, 512) for r in g.replicas]
    halt, errs = threading.Event(), []
    state = dict(prev=0, k=0, running=[])

    def consume(cn, seed):
        rng = np.random.default_rng(seed)
        try:
            while not halt.is_set():
                cn.step(int(rng.choice([1, 7, 64, 512])))
                time.sleep(0.0005)
        except Exception as e:        # noqa: BLE001 - reported below
            errs.append(e)
    th = [threading.Thread(target=consume, args=(cn, 60 + k)) for k, cn in enumerate(cons)]

    def run(stream, nbytes, live):
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
            r.wait(120_000)
        state["running"] = []
        assert not errs, errs
        end = g.leader.offsets()["end"]
        rp.launch(AR.read_launch(g.leader, state["prev"], end, L), requests, live=live)
        state["prev"] = end

    try:
        for x in th:
            x.start()
        g.prologue()
        while rp.written < 2 * L:
            run(old, 0.3 * L, [1, 2])
        cap = idx_cap(L)
        while True:
            o = g.leader.offsets()
            e, last = o["end"], g.leader.stats()["entries_published"]
            if 0.42 * L < e < 0.7 * L and 20 <= cap - last % cap <= 200 and AR.dist(o["head"], e, L) > 0.14 * L:
                break
            assert rp.written < 12 * L, "no point to start the lagging range found"
            run(old, 0.04 * L, [1, 2])
        lag_start, w_lag = g.replicas[2].offsets()["end"], rp.written
        # follower 2 pins the pruning at lag_start, so that the window below never blocks (as in test_gpu_takeover's
        # case).  A bounded launch ends without waiting for the consumers, and a follower forwards its consumer's cursor
        # only every few hundred polls, so the cursor the leader holds may lie a launch or more behind: let follower 2
        # alone run until it has forwarded its consumer's cursor at lag_start
        state["running"] = [g.replicas[2]]
        EU.launch_each(eng, state["running"], FOREVER)
        wait_for(lambda: g.leader.remote_apply_offsets()[2] == lag_start, f"follower 2 to forward its cursor {lag_start}")
        EU.stop_each(eng, state["running"])
        state["running"] = []
        while rp.written - w_lag < 0.6 * L or (not [h for h in rp.heads if h.lap_pos >= w_lag] and
                                                rp.written - w_lag < 0.7 * L):
            run(old, 0.1 * L, [1])
        # (unlike test_gpu_takeover's case, a HEAD inside the missed range is not required: follower 2's apply offset
        # is its consumer's cursor as its kernel last forwarded it, which the head may already have reached)
        assert g.leader.committed() == g.tickets
        first, last = g.replicas[2].stats()["entries_acked"] + 1, g.replicas[1].stats()["entries_acked"]
        _, shared, resent = elect(eng, g, rp.c, [1, 2], 1, [2], 2)
        a, b = resent[2]
        assert a == lag_start and b < a, f"the resent range [{a}, {b}) must wrap the ring"
        assert first // cap != last // cap, f"the resent entries' index words {first}..{last} must wrap idx_cap {cap}"
        requests.append((O.CONFIG, 0, 0, b""))
        g.prologue()
        state["k"], w0 = 0, rp.written
        while rp.written - w0 < 2 * L:
            # (heads are compared at the end, not after each launch: the voter adopts the head of a HEAD entry it was
            # resent only with the next HEAD it acks, and here the consumers' cursors decide when that comes)
            run(new, 0.3 * L, [2])
        check_heads([g.replicas[1], g.replicas[2]], rp, f"after the new term's last launch, ending at {rp.end()}",
                    [1, 2])
        halt.set()
        for x in th:
            x.join(60)
            assert not x.is_alive()
        assert not errs, errs
        for i in (1, 2):
            eo, oo = g.replicas[i].offsets(), rp.c.offsets(i)
            keys = ("head", "commit", "end") + (("tail",) if i == 1 else ())
            assert {k: eo[k] for k in keys} == {k: oo[k] for k in keys}, (i, eo, oo)
            ei, oi = g.replicas[i].image(), rp.c.image(i)
            d = np.nonzero(ei != oi)[0]
            assert len(d) == 0, f"replica {i}: {len(d)} bytes differ, first at {int(d[0])}"
        # rows: the CSM-like requests of both terms in submission order, on both survivors; the old leader's a prefix
        want = [(t, c_ & 0xFFFF, r_, bytes(p_)) for t, c_, r_, p_ in requests if t not in (O.NOOP, O.CONFIG, O.HEAD)]
        for i in (1, 2):
            catch_up(cons[i])
            check_rows(cons[i].rows, want, first_idx=2)
            assert cons[i].rows == cons[1].rows
            assert cons[i].rep.consume_status().error == 0
        assert cons[0].rows == cons[1].rows[:len(cons[0].rows)]
        assert [x for x in cons[1].rows if x[2] == 0], "the winner delivered no row of the old term"
        print({i: len(cn.rows) for i, cn in enumerate(cons)}, "rows", flush=True)
    finally:
        halt.set()
        for x in th:
            x.join(60)
        try:
            if state["running"]:
                EU.stop_each(eng, state["running"])
        finally:
            g.close()
            rp.close()


INDEX_OFF = 65536 + 320 * 1024          # apus_layout.h APUS_INDEX_OFF: the offset index follows the log header


def region_bytes(rep, off, n):
    """bytes [off, off + n) of a replica's HBM region (control block, header, offset index), read through the region
    pointer its peer handle carries in this process"""
    try:
        rt = C.CDLL("libcudart.so.12")
    except OSError:
        import nvidia.cuda_runtime as ncr
        rt = C.CDLL(os.path.join(list(ncr.__path__)[0], "lib", "libcudart.so.12"))
    ptr = int.from_bytes(rep.export()[24:32], "little")          # peer_blob.ptr
    out = np.zeros(n, dtype=np.uint8)
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    assert rt.cudaMemcpy(out.ctypes.data, ptr + off, n, 2) == 0          # cudaMemcpyDeviceToHost
    return out


def case_argument_checks(eng, orc):
    lib = eng.lib()
    n, L = 3, 1 << 20
    devs = devices_for(eng, n)
    for i in (0, 1):
        with pytest.raises(E.ApusError, match="needs APUS_F_DEVICE_APPLY"):
            E.Replica(devs[i], i, n, 0, 1, L, flags=E.F_APPLY_ANY_ROLE)
    with pytest.raises(E.ApusError, match="needs APUS_F_DEVICE_APPLY"):
        E.Replica(devs[1], 1, n, 0, 1, L, flags=E.F_APPLY_ANY_ROLE | E.F_HOST_APPLY)
    plain = consumer_group(eng, n, L)                       # device consumers on the followers only
    a = consumer_group(eng, n, L, leader_flags=ANY, follower_flags=[ANY, ANY])
    b = []
    got = u64()
    try:
        out = a[0].consume_device(4, 16)                    # a leader with the flag consumes (nothing committed yet)
        a[0].consume_device_packed(4, 64)
        import torch
        torch.cuda.synchronize(a[0].device)
        assert int(out[6].cpu()[0]) == 0 and a[0].consume_status().error == 0
        with pytest.raises(E.ApusError, match="follower"):
            plain[0].consume_device(4, 16)
        with pytest.raises(E.ApusError, match="keeps its role"):
            E._ck(lib.apus_replica_set_role(plain[1].h, 1, 2), "apus_replica_set_role")
        with pytest.raises(E.ApusError, match="consumes on the device"):
            E._ck(lib.apus_ctl_adjust_follower(plain[0].h, 1, sid(1, 1, 0), C.byref(got)), "apus_ctl_adjust_follower")
        # group a: 40 requests, every consumer reads them all (cursor past idx 1)
        lead = a[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = submit_all(lead, [(S.CONNECT, 1, 1, b"")] + [(S.SEND, 1, 2 + k, b"a" * (k % 60)) for k in range(40)])
        EU.launch_each(eng, a, t)
        for r in a:
            r.wait(60_000)
        for r in a:
            cn = Consumer(r, 64, 64)
            k, st = cn.step(64)
            assert k == 41 and st.next_idx == 43 and st.cursor == r.offsets()["commit"], (k, st)
        # group b (term 5): a log that shares nothing with a's, its head moved past idx 43; once its launch is over,
        # its leader is connected to a's replica 2 as its own peer 2
        b = [E.Replica(devs[i], i, n, 0, 5, L, flags=MODES["index_earlyack"] | ANY) for i in (0, 1)]
        b[0].connect(1, b[1].export())
        b[1].connect(0, b[0].export())
        lb = b[0]
        lb.submit(O.CONFIG, 0, 0, O.cid_image(n))
        tb = submit_all(lb, [(S.CONNECT, 2, 1, b"")] + [(S.SEND, 2, 2 + k, b"b" * (k % 50)) for k in range(100)])
        EU.launch_each(eng, b, tb)
        for r in b:
            r.wait(60_000)
        img = lb.image()
        ents = O.walk_entries(img, 0, lb.offsets()["end"], L)
        at = [o for o, _ in ents if int.from_bytes(img[o:o + 8].tobytes(), "little") == 60][0]
        lb.set_head(at)
        b[0].connect(2, a[2].export())
        # the peer's whole region but its entries: control block (consumer record and cursor among it), log header and
        # offset index; and the entries, offsets, consume status and stats
        raw = (0, 4096), (65536, 64), (INDEX_OFF, 4 * idx_cap(L))
        before = ([region_bytes(a[2], o, k) for o, k in raw], a[2].image(), a[2].offsets(), tuple(a[2].consume_status()),
                  a[2].stats())
        with pytest.raises(E.ApusError, match="shares no entry"):
            E._ck(lib.apus_ctl_adjust_follower(lb.h, 2, sid(5, 1, 0), C.byref(got)), "apus_ctl_adjust_follower")
        after = ([region_bytes(a[2], o, k) for o, k in raw], a[2].image(), a[2].offsets(), tuple(a[2].consume_status()),
                 a[2].stats())
        for (o, k), x, y in zip(raw, before[0], after[0]):
            d = np.nonzero(x != y)[0]
            assert len(d) == 0, f"the refused adjustment wrote region bytes {o}+{int(d[0])}.. of the peer"
        assert np.array_equal(before[1], after[1]) and before[2:] == after[2:], "the refused adjustment wrote to the peer"
        # the flag lets the control plane work: an adjustment of a follower that shares its log, and role changes both
        # ways on stopped replicas
        E._ck(lib.apus_ctl_adjust_follower(a[0].h, 1, sid(1, 1, 0), C.byref(got)), "apus_ctl_adjust_follower")
        assert int(got.value) == 0
        E._ck(lib.apus_replica_set_role(a[1].h, 1, 2), "apus_replica_set_role (to leader)")
        assert a[1].offsets()["apply"] == a[1].consume_status().cursor
        E._ck(lib.apus_replica_set_role(a[1].h, 0, 2), "apus_replica_set_role (back to follower)")
        assert a[1].consume_status().error == 0
    finally:
        for g in (b, a, plain):
            for r in g:
                r.close()


u64 = C.c_uint64

if __name__ == "__main__":
    EU.worker_main(globals())
