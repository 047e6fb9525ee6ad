"""Resident consumers (apus_consumer_attach, include/apus_consumer.cuh): an application's own persistent kernel --
tests/devicelogic/resident_rows.cu, which includes only the public header -- applies committed entries from the log in
place, beside the replica kernels.  Its rows are checked against the request stream and the CPU oracle's log, as the
stream-ordered consumers' are; its cursor gates the pruning rule; it hands over to and from the stream-ordered calls
without a gap; it stays attached through a take-over; its position seeds a replacement; read fences work beside it; and
every refusal, detach and destroy ends where it should.

Each replica holds a resident launch plus its own streams, and the resident consumers bring one stream each: more than
the 8 hardware queues a process gets by default, and a stream that shares a queue with a resident launch waits behind it
(DESIGN.md s2).  So each case runs in a worker process of this file that sets CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA
starts.  Marked gpu."""
import ctypes as C
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

import numpy as np  # noqa: E402
import pytest  # noqa: E402

import autoprune_replay as AR  # noqa: E402
import engine_util as EU  # noqa: E402
import orc as O  # noqa: E402
import resident as R  # noqa: E402
import streams as S  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consumers import (ANY, Consumer, check_rows, close_all, consumer_group, heads_against_reports,  # noqa: E402
                       idx_cap, new_stream, oracle_rows, wait_forwarded, wait_forwarded_all)
from engine_util import MODES, QUIET_S, devices_for, eng, run_case, submit_all, tensors, wait_for  # noqa: E402,F401
from shadow import Takeover, check_heads, elect, lap_stream, watch_commits  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

FOREVER = EU.FOREVER


# ---- the pytest side: one worker process per case ------------------------------------------------------------------
# N, follower mode, express path, batch kind: every mode, both N, the express path on and off and all three batch kinds
# each appear with the others
ROWS_CASES = [(3, "index_earlyack", True, "host"), (3, "walk_fenced", False, "strided"),
              (3, "index_fenced", True, "packed"), (3, "walk_earlyack", False, "host"),
              (5, "index_earlyack", False, "strided"), (5, "walk_fenced", True, "packed"),
              (5, "index_fenced", False, "host"), (5, "walk_earlyack", True, "strided")]


@pytest.mark.parametrize("n,mode,express,batch", ROWS_CASES,
                         ids=[f"n{n}-{m}-{'express' if x else 'fenced'}-{b}" for n, m, x, b in ROWS_CASES])
def test_resident_rows(eng, n, mode, express, batch):
    """a ragged stream (host batches, one strided or one packed device batch) and closed-loop requests, with a resident
    consumer on every follower: every follower's rows equal the stream and the oracle's log; every final cursor is the
    commit offset and is forwarded as the apply offset"""
    run_case(__file__, "rows", n=n, mode=mode, express=express, batch=batch)


def test_resident_cursor_gates_pruning(eng):
    """one launch laps a 256 KiB ring with APUS_F_AUTOPRUNE while one follower's resident consumer lags: every row
    equals the stream, every HEAD carries a position some consumer logged (or the tail once all had caught up), and at
    least one carries the lagging consumer's"""
    run_case(__file__, "pruning")


def test_resident_hand_over(eng):
    """stream-ordered consume calls, then a resident consumer, then stream-ordered calls again: no gap, no duplicate,
    idx strictly increasing, and the consume call enqueued just before attach delivers before the first resident row"""
    run_case(__file__, "hand_over")


def test_resident_read_fence(eng):
    """a fence on a replica with an attached consumer ends READY with F, and that consumer's rows reach F; a fence
    that ends short of the committed-tickets word is followed by one that covers it"""
    run_case(__file__, "read_fence")


TAKEOVER_CASES = [("voters_ahead", 5, "index_earlyack", True), ("lagging", 3, "index_earlyack", True),
                  ("lagging", 3, "walk_fenced", False), ("lagging", 5, "walk_earlyack", True),
                  ("lagging", 5, "index_fenced", False), ("old_term", 5, "index_earlyack", True)]


@pytest.mark.parametrize("scenario,n,mode,express", TAKEOVER_CASES,
                         ids=[f"{s}-n{n}-{m}-{'express' if x else 'fenced'}" for s, n, m, x in TAKEOVER_CASES])
def test_resident_takeover(eng, scenario, n, mode, express):
    """the take-over scenarios of test_gpu_consume_any_role.py with a resident consumer on every replica, the leader
    included, attached throughout: every member's rows are the oracle's CSM-like entries of the winner's log across
    both terms, the winner's including the old term's; the final cursors are the commit offsets"""
    run_case(__file__, "takeover", scenario=scenario, n=n, mode=mode, express=express)


def test_resident_lapped_resend(eng):
    """the lapped resend on a pruning ring with a resident consumer on every replica: their cursors gate the pruning on
    both sides of the take-over, and the survivors' rows equal the requests of both terms"""
    run_case(__file__, "lapped_resend")


def test_resident_replacement(eng):
    """a resident consumer writes its position beside a copy of its state; a fresh replica seeded there and adjusted in
    runs its own resident consumer, and every replica ends with the same state"""
    run_case(__file__, "replacement")


def test_resident_refusals_and_lifetime(eng):
    """attach is refused without the flags, on a leader without APUS_F_APPLY_ANY_ROLE and when attached already;
    consume, wait and mark are refused while attached and accepted after detach; detach returns once the kernel has
    ended; destroy of an attached replica ends its running consumer through the stop word and returns"""
    run_case(__file__, "refusals")


# ---- the worker side ---------------------------------------------------------------------------------------------
def _submit(lead, stream, batch):
    """the requests, through the host or as one device batch in either layout; returns the last ticket"""
    if batch == "host":
        return submit_all(lead, stream)
    import torch
    if batch == "strided":
        t0 = lead.submit_device(*tensors(stream, lead.device, 1500))
    else:
        dev = torch.device("cuda", lead.device)
        ty, co, rq, _, _ = tensors(stream, lead.device, 1500)
        offs = np.concatenate([[0], np.cumsum([len(p) for *_, p in stream])]).astype(np.int64)
        vals = np.frombuffer(b"".join(p for *_, p in stream) or b"\0", dtype=np.uint8).copy()
        t0 = lead.submit_device_packed(ty, co, rq, torch.from_numpy(offs).to(dev), torch.from_numpy(vals).to(dev))
    return t0 + len(stream) - 1


def _residents(reps, **kw):
    return [R.Resident(r, new_stream(r.device), **kw) for r in reps]


def case_rows(eng, orc, n, mode, express, batch):
    L = 1 << 22
    stream = S.ragged_stream(1500, 1500, conns=4, seed=900 + n, close_every=40)
    nlone, ln = 200, 40
    pl = bytes((k * 131 + 7) & 0xFF for k in range(ln))
    lone = [(S.SEND, 9, 1 + i, pl) for i in range(nlone)]
    base = MODES[mode] | (0 if express else E.F_NO_EXPRESS)
    reps = consumer_group(eng, n, L, base, ring_mode=E.RING_HOST_MAPPED if batch == "host" else E.RING_DEVICE)
    R.lib()
    res = []
    try:
        allreq = stream + lone
        res = [x.start() for x in _residents(reps[1:], max_pass=97)]
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)))
        lead.wait_committed(_submit(lead, stream, batch), 60_000_000)
        assert len(lead.closed_loop(nlone, ln, 9, 1)) == nlone
        for x in res:
            x.wait_rows(len(allreq))
        wait_forwarded(reps)
        for x in res:
            why, k, _ = x.detach()
            assert why == R.END_STOP and k == len(allreq), (why, k)
        EU.stop_each(eng, reps)
        c = EU.oracle_cluster(orc, n, L, allreq)
        EU.compare_group_to_oracle(T.SimpleNamespace(n=n, replicas=reps, leader_idx=0), c, exact=True)
        for j, x in enumerate(res, start=1):
            rows = x.rows()
            check_rows(rows, allreq, first_idx=2)
            assert rows == oracle_rows(c, j), f"replica {j}: rows differ from the oracle's log"
            st = reps[j].consume_status()
            assert st.cursor == reps[j].offsets()["commit"] == reps[j].offsets()["apply"] == c.offsets(j)["commit"]
            assert st.next_idx == len(allreq) + 2 and st.error == 0, st
        c.close()
    finally:
        close_all(eng, reps)


def case_pruning(eng, orc):
    """(test_gpu_consume_any_role.test_leader_cursor_gates_pruning with resident consumers on the followers) follower
    1's host applies through a recorder, which gives the replay the leader's append sequence; followers 2 and 3 consume
    with resident consumers, follower 2 lagging by a delay per pass and a per-pass limit of 3 entries"""
    n, L, ctas = 4, 1 << 18, 2
    stream = S.ragged_stream(int(6.5 * 1.15 * L / 814) + 1, 1500, conns=3, seed=297, close_every=20)
    requests = [(O.CONFIG, 0, 0, b"")] + stream
    reps = consumer_group(eng, n, L, leader_flags=E.F_AUTOPRUNE, ring_slots=1 << 14, ring_bytes=1 << 17, ctas=ctas,
                          follower_flags=[E.F_HOST_APPLY, E.F_DEVICE_APPLY, E.F_DEVICE_APPLY])
    rec = AR.Recorder(reps[1], 1, L)
    rp = AR.Replay(orc, n, L)
    lagging = 2
    R.lib()
    try:
        cap = len(stream) + 8
        res = {2: R.Resident(reps[2], new_stream(reps[2].device), max_pass=3, delay_ns=2_000_000, row_cap=cap,
                             log_cap=cap),
               3: R.Resident(reps[3], new_stream(reps[3].device), max_pass=64, row_cap=cap, log_cap=cap)}
        for x in res.values():
            x.start()
        rec.start()
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        # the kernels' %globaltimer onto the host clock: the CONFIG commits after h0, so a device time d maps to at most
        # the host time it happened at (a report never looks later than it was)
        h0 = time.perf_counter()
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)))
        to_host = h0 - lead.last_commit_ns() * 1e-9
        t = submit_all(lead, stream)
        deadline = time.time() + 400
        while lead.committed() < t:
            rec.check()
            assert time.time() < deadline, f"committed {lead.committed()} of {t}; leader {lead.offsets()}"
            time.sleep(0.005)
        for x in res.values():
            x.wait_rows(len(stream), timeout=300)
        final = lead.offsets()["end"]
        rec.finish(final)
        wait_forwarded_all([reps[2], reps[3]])
        EU.stop_each(eng, reps)
        reports = {1: rec.rec.reports}
        for j, x in res.items():
            why, k, lg = x.detach()
            assert why == R.END_STOP and k == len(stream), (j, why, k)
            check_rows(x.rows(), stream, first_idx=2)
            at, prev, rs = 0, 0, []
            for cur, _, ns in lg:
                adv = (cur - prev) % L
                prev = cur
                if adv:
                    at += adv
                    rs.append((at, ns * 1e-9 + to_host))
            reports[j] = rs
        pieces, flat, src, gaps = AR.recording_pieces([rec.rec], L)
        assert gaps[1] is None, gaps
        hits = []
        on_head = heads_against_reports(L, rec.rec.segs, reports, lagging, hits)
        for c0, lc in pieces:
            rp.launch(lc, requests, replica=src, on_head=on_head)
            for s_, b, _ in rec.rec.segs:
                if s_ + len(b) == c0 + len(lc.buf):
                    AR.compare_read(rp, 1, s_, b, flat)
        assert rp.pos == len(requests)
        assert rp.written >= 6 * L, rp.written / L
        assert hits, "no HEAD carried the lagging resident consumer's cursor: the test never gated the pruning rule"
        for j in res:
            assert reports[j][-1][0] == rp.written, (j, reports[j][-1], rp.written)
        for i, r in enumerate(reps):
            eo, oo = r.offsets(), rp.c.offsets(i)
            for key in ("end", "commit", "head"):
                assert eo[key] == oo[key], (i, key, eo, oo)
        AR.assert_heads_have_teeth(rp, rp.c.image(0))
    finally:
        close_all(eng, reps)


def case_hand_over(eng, orc):
    n, L = 3, 1 << 22
    parts = [S.ragged_stream(300, 600, conns=3, seed=40 + k, close_every=50) for k in range(3)]
    reps = consumer_group(eng, n, L)
    R.lib()
    try:
        lead, fol = reps[0], reps[1]
        stream = new_stream(fol.device)
        cn = Consumer(fol, 600, 0, stream=stream)
        x = R.Resident(fol, stream)
        EU.launch_each(eng, reps, FOREVER)
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)))
        lead.wait_committed(submit_all(lead, parts[0]))
        k, _ = cn.step(100)                                   # stream-ordered rows: part of the first part
        assert k > 0
        # a call enqueued right before attach, never synchronised: its rows come before the first resident row
        last = fol.consume_device(4096, 600, stream=stream)
        x.start()
        got_last = int(last[6].cpu()[0])
        idx, ty, co, rq, ln, pl = (t[:got_last].cpu().numpy() for t in last[:6])
        cn.rows += [(int(idx[q]), int(ty[q]), int(co[q]) & 0xFFFF, int(rq[q]), pl[q, :int(ln[q]) & 0xFFFF].tobytes())
                    for q in range(got_last)]
        lead.wait_committed(submit_all(lead, parts[1]))
        x.wait_rows(len(parts[0]) + len(parts[1]) - len(cn.rows))
        why, nres, _ = x.detach()
        assert why == R.END_STOP
        res_rows = x.rows()
        assert res_rows and res_rows[0][0] > cn.rows[-1][0], (res_rows[:1], cn.rows[-1:])
        lead.wait_committed(submit_all(lead, parts[2]))
        mid = len(cn.rows)
        cn.rows += res_rows
        while len(cn.rows) < sum(len(p) for p in parts):
            cn.step(256)
        assert len(cn.rows) - mid - len(res_rows) > 0
        check_rows(cn.rows, parts[0] + parts[1] + parts[2], first_idx=2)
        wait_forwarded(reps[:2])
    finally:
        close_all(eng, reps)


def case_read_fence(eng, orc):
    n, L = 3, 1 << 22
    reps = consumer_group(eng, n, L, leader_flags=ANY, follower_flags=[ANY, ANY])
    R.lib()
    try:
        res = _residents(reps)
        fence_streams = [new_stream(r.device) for r in reps]
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)))
        for x in res:
            x.start()
        stop = threading.Event()
        req = []

        def writer():
            rid = 1
            while not stop.is_set():
                part = [(S.SEND, 2, rid + q, bytes([(rid + q) & 0xFF]) * ((rid + q) % 90)) for q in range(50)]
                submit_all(lead, part)
                req.extend(part)
                rid += 50
                time.sleep(0.0005)
        th = threading.Thread(target=writer)
        th.start()
        try:
            for rnd in range(40):
                j = rnd % n
                r = reps[j]
                seen = lead.committed()
                s = fence_streams[j]
                index, outcome = r.read_fence(5_000_000, stream=s)
                s.synchronize()
                assert int(outcome.cpu()[0]) == E.WAIT_READY, (rnd, int(outcome.cpu()[0]))
                F = int(index.cpu()[0])
                if F < seen:                             # short of the tickets word: one more fence covers it
                    index, outcome = r.read_fence(5_000_000, stream=s)
                    s.synchronize()
                    assert int(outcome.cpu()[0]) == E.WAIT_READY
                    F = int(index.cpu()[0])
                    assert F >= seen, (rnd, F, seen)
                # the attached consumer's rows reach F: rows are CSM-like entries, idx 1 is the CONFIG
                t_end = time.time() + 30
                while True:
                    st = r.consume_status()
                    if st.next_idx > F:
                        break
                    assert time.time() < t_end, (rnd, st, F)
                    time.sleep(0.0005)
        finally:
            stop.set()
            th.join()
        t = lead.committed()
        for x in res:
            x.wait_rows(len(req))
        for x in res:
            why, k, _ = x.detach()
            assert why == R.END_STOP and k == len(req)
            check_rows(x.rows(), req, first_idx=2)
        assert t >= len(req)
    finally:
        close_all(eng, reps)


class ResidentTakeover(Takeover):
    """Takeover (shadow.py) with a resident consumer on every replica, attached before the group's first launch and
    throughout: running, stopped, changing roles"""

    def __init__(self, eng, orc, n, L, flags, seed):
        # the consumers, their streams and their kernel's module exist before the first launch: a lazy load or a
        # stream pool created beside resident replica kernels may wait for them
        self.cons = None
        launch = EU.launch_each
        R.lib()

        def first_launch(eng_, reps, *a, **kw):
            if self.cons is None:
                self.cons = [R.Resident(r, new_stream(r.device), stride=300, max_pass=int(m), log_cap=16).start()
                             for r, m in zip(sorted(reps, key=lambda r: r.idx), (1, 5, 64, 256, 17))]
            return launch(eng_, reps, *a, **kw)
        EU.launch_each = first_launch
        try:
            super().__init__(eng, orc, n, L, flags | ANY, seed)
        finally:
            EU.launch_each = launch

    def check_offsets(self, keys_leader=("head", "apply", "commit", "end", "tail")):
        """the oracle's apply offsets follow the commit; here they are the consumers' cursors (checked by finish())"""
        keys_leader = tuple(k for k in keys_leader if k != "apply")
        for i in sorted(self.members):
            eo, oo = self.rep(i).offsets(), self.c.offsets(i)
            keys = keys_leader if i == self.lead else ("head", "commit", "end")
            assert {k: eo[k] for k in keys} == {k: oo[k] for k in keys}, (i, i == self.lead, i in self.live, eo, oo)

    def finish(self, old_lead):
        """every member's consumer reaches its commit offset; rows against the oracle's winner log, across both terms"""
        for i in sorted(self.members):
            _resident_caught_up(self.cons[i])
        rows = {}
        for i, x in enumerate(self.cons):
            why, _, _ = x.detach()
            assert why == R.END_STOP, (i, why)
            rows[i] = x.rows()
        want = oracle_rows(self.c, self.lead)
        for i in sorted(self.members):
            got = rows[i]
            first = next((q for q, (a, b) in enumerate(zip(got, want)) if a != b), None)
            assert got == want, f"replica {i} (leader {self.lead}): {len(got)} rows, want {len(want)}; first diff {first}"
            st = self.rep(i).consume_status()
            assert st.error == 0 and st.cursor == self.rep(i).offsets()["commit"], (i, st)
        for i in range(len(self.cons)):
            if i not in self.members:
                assert rows[i] == want[:len(rows[i])], f"replica {i}: its rows are not a prefix of the winner's"
        old = [x for x in want if x[2] == (old_lead << 8)]
        assert old and [x for x in rows[self.lead] if x[2] == (old_lead << 8)] == old, \
            "the winner's consumer did not deliver the old term's entries"

    def close(self):
        try:
            for x in self.cons or []:
                if x.rep.h:
                    try:
                        x.rep.consumer_detach()
                    except E.ApusError:
                        pass
        finally:
            super().close()


def _resident_caught_up(x, timeout=60):
    """the resident consumer's cursor, as its status words show it, is its replica's commit offset"""
    t = time.time()
    while True:
        st, o = x.rep.consume_status(), x.rep.offsets()
        if st.cursor == o["commit"] and o["commit"] == o["end"]:
            return st
        assert time.time() - t < timeout, (x.rep.idx, st, o, x.rows_so_far())
        time.sleep(0.002)


def case_takeover(eng, orc, scenario, n, mode, express):
    flags = MODES[mode] | (0 if express else E.F_NO_EXPRESS)
    p = ResidentTakeover(eng, orc, n, 1 << 20, flags, seed=n + 200)
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
    third of a lap, a resident consumer on every replica, attached throughout: follower 2 misses 0.6 to 0.7 of a lap, 1
    takes over with voter 2 (a resend across the ring's wrap and the offset index's), and the new term laps twice.  The consumers
    gate the pruning on both sides; the survivors' rows equal the requests of both terms in order"""
    n, L = 3, 1 << 16
    old, new = lap_stream(20_000, 0, 31), lap_stream(20_000, 1 << 8, 32)
    requests = [(O.CONFIG, 0, 0, b"")]
    rp = AR.Replay(orc, n, L)
    g = E.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES["index_earlyack"] | E.F_AUTOPRUNE | ANY)
    R.lib()
    cons = [R.Resident(r, new_stream(r.device), max_pass=int(m), log_cap=16) for r, m in zip(g.replicas, (7, 64, 256))]
    errs = []
    state = dict(prev=0, k=0, running=[])

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
        for x in cons:
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
        for i in (1, 2):
            eo, oo = g.replicas[i].offsets(), rp.c.offsets(i)
            keys = ("head", "commit", "end") + (("tail",) if i == 1 else ())
            assert {k: eo[k] for k in keys} == {k: oo[k] for k in keys}, (i, eo, oo)
            ei, oi = g.replicas[i].image(), rp.c.image(i)
            d = np.nonzero(ei != oi)[0]
            assert len(d) == 0, f"replica {i}: {len(d)} bytes differ, first at {int(d[0])}"
        # rows: the CSM-like requests of both terms in submission order, on both survivors; the old leader's a prefix
        want = [(t, c_ & 0xFFFF, r_, bytes(p_)) for t, c_, r_, p_ in requests if t not in (O.NOOP, O.CONFIG, O.HEAD)]
        rows = {}
        for i in (1, 2):
            _resident_caught_up(cons[i])
        for i, x in enumerate(cons):
            why, _, _ = x.detach()
            assert why == R.END_STOP, (i, why)
            rows[i] = x.rows()
        for i in (1, 2):
            check_rows(rows[i], want, first_idx=2)
            assert rows[i] == rows[1]
            assert cons[i].rep.consume_status().error == 0
        assert rows[0] == rows[1][:len(rows[0])]
        assert [x for x in rows[1] if x[2] == 0], "the winner delivered no row of the old term"
        print({i: len(r) for i, r in rows.items()}, "rows", flush=True)
    finally:
        try:
            if state["running"]:
                EU.stop_each(eng, state["running"])
        finally:
            g.close()
            rp.close()


def case_replacement(eng, orc):
    """replica 2 of a five-replica group is lost for good; a fresh one is seeded at the position replica 1's resident
    consumer wrote, adjusted in, and runs a resident consumer of its own.  A consumer's state is its rows: the copy
    taken beside the position is replica 1's rows up to it, and the replacement's state is that copy plus its own rows.
    Freeing the lost replica waits for every kernel on the GPU, so the consumers detach for it and attach again."""
    from shadow import sid
    n, L, k = 5, 1 << 22, 2
    lib = eng.lib()
    devs = EU.devices_for(eng, n)
    reps = consumer_group(eng, n, L, leader_flags=ANY, follower_flags=[ANY] * (n - 1))
    R.lib()
    try:
        res = {j: R.Resident(reps[j], new_stream(reps[j].device)) for j in range(n)}
        spare = R.Resident(reps[k], new_stream(reps[k].device))
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)))
        for x in res.values():
            x.start()
        a = S.ragged_stream(400, 500, conns=3, seed=61, close_every=40)
        lead.wait_committed(submit_all(lead, a))
        res[1].wait_rows(len(a) // 2)
        cur, nidx, nrows = res[1].snapshot_position()
        res[1].resume()
        b = [(S.SEND, 7, 1 + q, bytes([q & 0xFF]) * (q % 300)) for q in range(200)]
        lead.wait_committed(submit_all(lead, b))
        for j, x in res.items():
            x.wait_rows(len(a) + len(b))
        EU.stop_each(eng, reps)
        rows = {}
        for j, x in res.items():
            why, _, _ = x.detach()
            assert why == R.END_STOP, (j, why)
            rows[j] = x.rows()
        copy = rows[1][:nrows]
        # the lost follower: every other replica disconnects it, its region goes
        for i in range(n):
            if i != k:
                E._ck(lib.apus_replica_disconnect(reps[i].h, k), "apus_replica_disconnect")
        reps[k].close()
        fresh = E.Replica(devs[k], k, n, 0, 1, L, E.RING_HOST_MAPPED, 0, 0, MODES["index_earlyack"] | ANY, 4)
        for i in range(n):
            if i != k:
                fresh.connect(i, reps[i].export())
                reps[i].connect(k, fresh.export())
        reps[k] = fresh
        fresh.consume_seed(cur, nidx)
        got = E.u64()
        E._ck(lib.apus_ctl_adjust_follower(lead.h, k, sid(1, 1, 0), C.byref(got)), "apus_ctl_adjust_follower")
        E._ck(lib.apus_replica_set_role(fresh.h, 0, 1), "apus_replica_set_role")
        spare.rep = fresh
        res[k] = spare
        rows[k] = []
        for x in res.values():
            x.start()
        EU.launch_each(eng, reps, FOREVER)
        c = [(t, cl + 10, q, p) for t, cl, q, p in S.ragged_stream(300, 500, conns=2, seed=63, close_every=40)]
        lead.wait_committed(submit_all(lead, c))
        total = len(a) + len(b) + len(c)
        for j, x in res.items():
            x.wait_rows(total - len(rows[j]) - (nrows if j == k else 0))
        wait_forwarded_all(reps)
        EU.stop_each(eng, reps)
        for j, x in res.items():
            why, _, _ = x.detach()
            assert why == R.END_STOP, (j, why)
            rows[j] += x.rows()
        check_rows(rows[1], a + b + c, first_idx=2)
        assert copy + rows[k] == rows[1], "the replacement's state differs from the group's"
        for j in range(n):
            if j != k:
                assert rows[j] == rows[1], j
        for r in reps:
            st = r.consume_status()
            assert st.cursor == r.offsets()["commit"] and st.error == 0, (r.idx, st, r.offsets())
    finally:
        close_all(eng, reps)


def case_refusals(eng, orc):
    import torch
    n, L = 3, 1 << 20
    devs = EU.devices_for(eng, n)
    plain = consumer_group(eng, n, L)                              # followers with APUS_F_DEVICE_APPLY only
    other = None
    R.lib()
    try:
        s = new_stream(devs[0])
        with pytest.raises(E.ApusError, match="follower"):
            plain[0].consumer_attach(s)                             # a leader without APUS_F_APPLY_ANY_ROLE
        other = E.Replica(devs[1], 1, n, 0, 1, L, flags=MODES["index_earlyack"])
        with pytest.raises(E.ApusError, match="needs a replica created with APUS_F_DEVICE_APPLY"):
            other.consumer_attach(new_stream(devs[1]))
        with pytest.raises(E.ApusError, match="no resident consumer"):
            other.consumer_detach()
        fol = plain[1]
        with pytest.raises(E.ApusError, match="no resident consumer"):
            fol.consumer_detach()
        fs, fs2, s2 = new_stream(fol.device), new_stream(fol.device), new_stream(plain[2].device)
        x, y = R.Resident(fol, fs), R.Resident(plain[2], s2)
        EU.launch_each(eng, plain, FOREVER)
        lead = plain[0]
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)))
        part = [(S.SEND, 1, 1 + q, b"x" * q) for q in range(30)]
        lead.wait_committed(submit_all(lead, part))
        x.start()
        with pytest.raises(E.ApusError, match="attached already"):
            fol.consumer_attach(fs2)
        for call in (lambda: fol.consume_device(4, 64, stream=fs), lambda: fol.consume_device_packed(4, 64, stream=fs),
                     lambda: fol.consume_wait(1, 1000, stream=fs), lambda: fol.consume_mark(stream=fs)):
            with pytest.raises(E.ApusError, match="resident consumer is attached"):
                call()
        x.wait_rows(len(part))
        t0 = time.perf_counter()
        why, k, _ = x.detach()                                      # returns once the kernel has ended
        assert why == R.END_STOP and k == len(part) and time.perf_counter() - t0 < 5
        assert fs.query(), "detach returned before the consumer's stream was done"
        # accepted again after detach, from the cursor the resident consumer left
        st = fol.consume_status()
        assert st.next_idx == len(part) + 2 and st.cursor == fol.offsets()["commit"], st
        lead.wait_committed(submit_all(lead, [(S.SEND, 1, 100, b"after")]))
        fol.consume_wait(1, 1_000_000, stream=fs)
        out = fol.consume_device(4, 64, stream=fs)
        fol.consume_mark(stream=fs)
        fs.synchronize()
        assert int(out[6].cpu()[0]) == 1 and int(out[3].cpu()[0]) == 100
        # destroy of an attached replica whose consumer kernel runs: the stop word ends it, and destroy returns
        f2 = plain[2]
        y.start()
        y.wait_rows(len(part) + 1)
        EU.stop_each(eng, plain)
        t0 = time.perf_counter()
        f2.close()
        plain.remove(f2)
        assert time.perf_counter() - t0 < 10
        assert s2.query()
        assert int(y.out.cpu()[0]) == R.END_STOP
        torch.cuda.synchronize()
    finally:
        if other is not None:
            other.close()
        close_all(eng, plain)


if __name__ == "__main__":
    EU.worker_main(globals())
