"""Resident submitters through leader take-overs (apus_submitter_attach on every replica, include/apus_submitter.cuh): a
submitter attached to a follower is dormant -- its reserves end NOT_LEADER at once and write nothing, and the host paths
stay open -- until the first launch that runs its replica as leader hands the ring over.  One test kernel per replica
(tests/devicelogic/takeover_submit.cu), launched once, writes through a fail-over beside a resident consumer on every
replica; the rows and the logs are checked against the CPU oracle shadowing the take-over (shadow.Takeover).  Also: the
host's blank CONFIG before the hand-over, a replica that leads twice on the device ring, and the refusals and lifetimes.

Each replica holds a resident launch, a consumer and a submitter, each on a stream of its own: more than the 8 hardware
queues a process gets by default.  So each case runs in a worker process of this file that sets
CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA starts.  Marked gpu."""
import ctypes as C
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":
    os.environ["CUDA_DEVICE_MAX_CONNECTIONS"] = "32"         # before anything starts CUDA
    for p in (HERE, os.path.dirname(HERE)):
        if p not in sys.path:
            sys.path.insert(0, p)

import numpy as np  # noqa: E402
import pytest  # noqa: E402

import engine_util as EU  # noqa: E402
import orc as O  # noqa: E402
import resident as R  # noqa: E402
import streams as S  # noqa: E402
import submitter as SB  # noqa: E402
import takeover_submit as TS  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consumers import ANY, new_stream, oracle_rows  # noqa: E402
from engine_util import MODES, devices_for, eng, run_case, wait_for  # noqa: E402,F401
from takeover_device import DeviceTakeover  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

GATE = b"resident submitter is attached"        # the message of every host call that writes the ring


# ---- the pytest side: one worker process per case ------------------------------------------------------------------
@pytest.mark.parametrize("n", [3, 5])
def test_failover_with_one_kernel_per_replica(eng, n):
    """one submitter kernel and one resident consumer per replica, launched once: the leader writes a mixed stream
    (ragged external images, cmds the descriptor cannot carry, rejected types) and stops mid-stream; the winner's kernel
    waits out NOT_LEADER, then writes its requests in the new term; every surviving consumer's rows are the oracle's
    winner log"""
    run_case(__file__, "failover", n=n)


def test_dormant_writes_nothing(eng):
    """on a follower, reserve ends NOT_LEADER within milliseconds; the doorbell, the submitter's state and the submit
    status are as before"""
    run_case(__file__, "dormant")


def test_host_and_submitter_take_turns(eng):
    """the winner's host submits (its blank CONFIG and more) are accepted while its submitter is dormant and commit
    before the submitter's first ticket; after the hand-over the host is refused"""
    run_case(__file__, "turns")


@pytest.mark.parametrize("resident", [False, True], ids=["host", "resident"])
def test_leading_twice(eng, resident):
    """0 -> 1 -> 0 on the device ring: in its second term replica 0 commits exactly what that term submitted.  host:
    every request through the host, the new term's CONFIG after the winner's launch; resident: replica 0 writes its
    first term from an active submitter, detaches, attaches again dormant and writes its second term from it"""
    run_case(__file__, "twice", resident=resident)


def test_refusals_and_lifetime(eng):
    """a follower on a host-mapped ring, a second attach, set_role on a dormant follower (accepted) and on an active
    leader (refused), and a dormant kernel ended STOPPED by detach and by destroy"""
    run_case(__file__, "lifetime")


# ---- helpers -------------------------------------------------------------------------------------------------------
def _cudart():
    try:
        return C.CDLL("libcudart.so.12")
    except OSError:
        import nvidia.cuda_runtime as ncr
        return C.CDLL(os.path.join(list(ncr.__path__)[0], "lib", "libcudart.so.12"))


def dev_words(device, ptr, n):
    """n 64-bit words of device memory at `ptr`, read with a synchronous copy"""
    rt = _cudart()
    buf = (C.c_uint64 * n)()
    assert rt.cudaSetDevice(device) == 0
    assert rt.cudaMemcpy(buf, C.c_void_p(ptr), C.c_size_t(8 * n), 2) == 0, "cudaMemcpy"   # cudaMemcpyDeviceToHost
    return list(buf)


def view_words(rep, v):
    """(doorbell, the submitter's state words) behind a view"""
    return dev_words(rep.device, v.doorbell, 1)[0], dev_words(rep.device, v.state, 8)


def submit_oracle(c, reqs):
    for typ, clt, rid, payload in reqs:
        assert c.submit(typ, clt, rid, O.cmd_image(payload)) != 0, f"the oracle refused request {rid}"


def as_rows(reqs):
    """the rows a resident consumer writes for requests in log order: the accepted ones"""
    return [(t, c, r, p) for t, c, r, p in reqs if t in SB.ACCEPTED]


def lead_stream(n, seed, first_req_id):
    """the mixed stream of a leader: ragged SENDs, CONNECTs, CLOSEs and CSMs of up to 200 B (external images past 78 B),
    every 23rd of a rejected type, and two SENDs longer than the descriptor carries (both written as NOOPs)"""
    reqs = SB.mixed_requests(n, seed=seed, max_len=200, first_req_id=first_req_id)
    for k, ln in ((n // 5, 65536), (n // 3, 70000)):
        reqs[k] = (S.SEND, 1, reqs[k][2], bytes((5 * i + k) & 0xFF for i in range(ln)))
    return reqs


class SubmitTakeover(DeviceTakeover):
    """Takeover on the device ring with one submitter kernel per replica (all but the leader's dormant from the start)
    and, with `consumers`, a resident consumer per replica; everything is created before the group's first launch"""

    def __init__(self, eng, orc, n, L, flags, seed, reqs, batch=16, modes=None, consumers=True):
        self.cons, self.subs, self.views = None, {}, {}
        launch = EU.launch_each
        if consumers:
            R.lib()
        if reqs:
            TS.lib()

        def first_launch(eng_, reps, *a, **kw):
            if self.cons is None:
                reps_ = sorted(reps, key=lambda r: r.idx)
                self.cons = [R.Resident(r, new_stream(r.device), stride=200, row_cap=1 << 14).start() if consumers
                             else None for r in reps_]
                for r in reps_:
                    if reqs.get(r.idx):
                        mode = (modes or {}).get(r.idx, 0)
                        self.subs[r.idx] = TS.Submitter(new_stream(r.device), reqs[r.idx], batch=batch, mode=mode)
                for r in reps_:                          # the followers' submitters start dormant, launched once
                    if r.idx in self.subs and not r.is_leader:
                        self.attach(r.idx)
            return launch(eng_, reps, *a, **kw)
        EU.launch_each = first_launch
        try:
            super().__init__(eng, orc, n, L, flags, seed)
        finally:
            EU.launch_each = launch

    def attach(self, i):
        """attach replica i's submitter on its kernel's stream and launch its kernel"""
        s = self.subs[i]
        self.views[i] = self.rep(i).submitter_attach(s.stream)
        s.start(self.views[i])

    def detach(self, i):
        self.rep(i).submitter_detach()
        self.views.pop(i)
        return self.subs[i].result()

    def close(self):
        try:
            for i in list(self.views):
                try:
                    self.rep(i).submitter_detach()
                except E.ApusError:
                    pass
            for x in self.cons or []:
                if x is not None:
                    try:
                        x.rep.consumer_detach()
                    except E.ApusError:
                        pass
        finally:
            super().close()

    def wait_commits(self, t, timeout=60):
        wait_for(lambda: self.leader.committed() >= t, f"{t} tickets committed", timeout=timeout)


def _caught_up(x, timeout=60):
    t = time.time()
    while True:
        st, o = x.rep.consume_status(), x.rep.offsets()
        if st.cursor == o["commit"] and o["commit"] == o["end"]:
            return
        assert time.time() - t < timeout, (x.rep.idx, st, o, x.rows_so_far())
        time.sleep(0.002)


# ---- the worker side -----------------------------------------------------------------------------------------------
def case_failover(eng, orc, n):
    L = 1 << 23                                          # the stream stays under a quarter: no HEAD entry is due
    lead = lead_stream(6000, seed=300 + n, first_req_id=10)
    win = lead_stream(1500, seed=400 + n, first_req_id=100_000)
    reqs = {0: lead, 1: win}
    for i in range(2, n):                                # followers that never lead: dormant to the end
        reqs[i] = SB.mixed_requests(8, seed=500 + i, reject_every=0)
    p = SubmitTakeover(eng, orc, n, L, MODES["index_earlyack"] | E.F_AUTOPRUNE | ANY, seed=n + 300, reqs=reqs,
                       batch=1, modes={0: TS.WAIT})
    try:
        base = p.g.tickets                               # the CONFIG and the CONNECT, from the host
        p.attach(0)                                      # a leader: active at once, one request in flight at a time
        p.wait_commits(base + 500)
        fail, pub, tickets = p.detach(0)                 # the old leader's application stops mid-stream
        assert fail in (None, (SB.STEP_RESERVE, SB.STOPPED), (SB.STEP_PUBLISH, SB.STOPPED),
                        (SB.STEP_WAIT, SB.STOPPED)), fail
        P = p.leader.stats()["tickets_submitted"]
        assert 500 <= P - base == pub < len(lead), (P, base, pub)
        assert set(p.subs[0].terms_of_chunks()[:pub]) == {1}
        p.wait_commits(P)
        p.g.tickets = P
        old, _ = SB.ticket_order(lead, tickets, upto=P)
        assert len(old) == P - base
        submit_oracle(p.c, old)
        p.rounds()
        p.settle()
        # the take-over: the winner's blank CONFIG goes through the host before its first launch hands the ring over
        p.take_over(1, list(range(2, n)), before_launch=p.g.prologue)
        p.c.prologue()
        fail, pub, wt = p.subs[1].result()
        assert fail is None and pub == len(win), (fail, pub)
        assert sorted(wt) == list(range(2, 2 + len(win)))
        assert set(p.subs[1].terms_of_chunks()) == {2} and p.subs[1].leading() == 2
        assert p.subs[1].not_leader() > 0, "the winner's kernel never saw NOT_LEADER"
        new, _ = SB.ticket_order(win, wt)
        submit_oracle(p.c, new)
        p.g.tickets = 1 + len(win)
        p.wait_commits(p.g.tickets)
        p.rounds()
        p.settle()
        assert p.leader.device_submit_status()[0] == sum(1 for r in win if not SB.accepted(r))
        p.check_images()
        for i in range(2, n):
            fail, pub, _ = p.detach(i)
            assert fail == (SB.STEP_RESERVE, SB.STOPPED) and pub == 0, (i, fail, pub)
            assert p.subs[i].not_leader() > 0 and p.subs[i].leading() == 0
        # the rows: every surviving consumer's equal the oracle's winner log, which is the old term's committed prefix,
        # the winner's CONFIG (no row), then the winner's tickets in order
        want = oracle_rows(p.c, 1)
        conn0 = [(S.CONNECT, 0, 1, b"")]
        assert [r[1:] for r in want] == as_rows(conn0 + old + new)
        rows = {}
        for i in sorted(p.members | {0}):
            _caught_up(p.cons[i])
        for i, x in enumerate(p.cons):
            why, _, _ = x.detach()
            assert why == R.END_STOP, (i, why)
            rows[i] = x.rows()
        for i in sorted(p.members):
            assert rows[i] == want, f"replica {i}: {len(rows[i])} rows, want {len(want)}"
        assert rows[0] == want[:len(rows[0])] and len(rows[0]) >= len(as_rows(conn0 + old))
        p.cons = None
        print(f"n={n}: old term {P - base} tickets of {len(lead)}, winner {len(win)} tickets after "
              f"{p.subs[1].not_leader()} NOT_LEADER outcomes")
    finally:
        p.close()


def case_dormant(eng, orc):
    n, L = 3, 1 << 22
    SB.lib()
    with EU.device_group(eng, n, L) as g:
        f = g.replicas[1]
        st = new_stream(f.device)
        # the submitter kernel of tests/test_gpu_submit_resident.py, which knows nothing of take-overs
        sub = SB.Submitter(E.SubmitterView(), st, SB.mixed_requests(64, seed=11, max_len=300), batch=8, timeout_s=20)
        g.launch(EU.FOREVER)
        g.leader.wait_committed(g.prologue())
        v = f.submitter_attach(st)
        before = view_words(f, v), f.device_submit_status(), f.stats()["tickets_submitted"]
        assert before[0][0] == 0 and before[0][1][0] == E.SUBMITTER_HOST_HELD and before[0][1][7] == E.SUBMITTER_DORMANT, \
            before
        t0 = time.time()
        sub.view = v
        sub.start()
        fail, pub, tickets = sub.result()
        took = time.time() - t0
        assert fail == (SB.STEP_RESERVE, TS.NOT_LEADER) and pub == 0 and not any(tickets), (fail, pub)
        ns = sub.phase_ns()["reserve"]
        assert ns < 5_000_000 and took < 5, (ns, took)
        after = view_words(f, v), f.device_submit_status(), f.stats()["tickets_submitted"]
        assert after == before, (before, after)
        f.submitter_detach()
        assert (view_words(f, v), f.device_submit_status()) == before[:2]
        g.leader.wait_committed(g.submit(S.SEND, 1, 2, b"the group still runs"))
        print(f"NOT_LEADER after {ns} ns of reserve")


def case_turns(eng, orc):
    n, L = 3, 1 << 22
    win = SB.mixed_requests(600, seed=21, max_len=400, first_req_id=1000)
    host = S.ragged_stream(10, 300, conns=2, seed=22)
    p = SubmitTakeover(eng, orc, n, L, MODES["index_earlyack"], seed=23, reqs={1: win}, batch=8, consumers=False)
    try:
        p.step(20, 2)
        seen = {}

        def before_launch():
            t = p.g.prologue()
            for typ, conn, rid, payload in host:             # accepted: the submitter is dormant
                t = p.g.submit(typ, conn, rid, payload)
            seen["doorbell"] = view_words(p.rep(1), p.views[1])[0]
            seen["tickets"] = t
        p.take_over(1, [2], before_launch=before_launch)
        assert seen == {"doorbell": 1 + len(host), "tickets": 1 + len(host)}, seen
        with pytest.raises(E.ApusError, match="resident submitter is attached"):
            p.g.submit(S.SEND, 1, 99, b"refused")
        lib = eng.lib()
        assert lib.apus_submit_flush(p.leader.h) == E.APUS_ERROR and GATE in lib.apus_last_error()
        fail, pub, wt = p.subs[1].result()
        assert fail is None and pub == len(win), (fail, pub)
        assert sorted(wt) == list(range(2 + len(host), 2 + len(host) + len(win)))
        assert set(p.subs[1].terms_of_chunks()) == {2} and p.subs[1].not_leader() > 0
        p.c.prologue()
        submit_oracle(p.c, host + SB.ticket_order(win, wt)[0])
        p.g.tickets = 1 + len(host) + len(win)
        p.wait_commits(p.g.tickets)
        p.rounds()
        p.settle()
        p.check_offsets()
        p.check_images()
        p.detach(1)
        assert p.leader.stats()["tickets_submitted"] == p.g.tickets
        print(f"{1 + len(host)} host tickets, then {len(win)} from the submitter")
    finally:
        p.close()


def log_entries(img, start, end, L):
    """(idx, term, type, conn, req_id, cmd) of every entry of a log image in [start, end)"""
    out = []
    for off, _ in O.walk_entries(img, start, end, L):
        ln = int(img[off + 48]) | int(img[off + 49]) << 8
        out.append((int(img[off:off + 8].view(np.uint64)[0]), int(img[off + 8:off + 16].view(np.uint64)[0]),
                    int(img[off + 26]), int(img[off + 24]) | int(img[off + 25]) << 8,
                    int(img[off + 16:off + 24].view(np.uint64)[0]), img[off + 50:off + 50 + ln].tobytes()))
    return out


def case_twice(eng, orc, resident):
    n, L = 3, 1 << 22
    first = SB.mixed_requests(300, seed=31, max_len=400, first_req_id=2000, reject_every=0)
    second = SB.mixed_requests(300, seed=32, max_len=400, first_req_id=3000, reject_every=0)
    reqs = {0: first} if resident else {}
    # replica 0's second kernel, made before any replica kernel is resident (its arrays need torch's kernels)
    again = TS.Submitter(new_stream(devices_for(eng, n)[0]), second, batch=8) if resident else None
    p = SubmitTakeover(eng, orc, n, L, MODES["index_earlyack"], seed=33, reqs=reqs, batch=8,
                       modes={0: 0}, consumers=False)
    try:
        # term 1: replica 0 leads (through an active submitter, or the host)
        if resident:
            base = p.g.tickets
            p.attach(0)
            fail, pub, t1 = p.subs[0].result()
            assert fail is None and pub == len(first), (fail, pub)
            p.g.tickets = base + len(first)
            submit_oracle(p.c, SB.ticket_order(first, t1)[0])
            p.check_committed()
            p.detach(0)                                  # before it rejoins as a follower
        else:
            p.step(len(first), 2)
        # term 2: replica 1 leads, replica 0 votes and follows, against the oracle
        if resident:
            p.take_over(1, [0, 2], old_votes=True, before_launch=p.g.prologue)
            p.c.prologue()
        else:
            p.take_over(1, [0, 2], old_votes=True)
            p.new_term()
        p.relaunch(0)
        if resident:                                     # replica 0 attaches again, dormant, and starts a new kernel
            p.subs[0] = again
            p.attach(0)
        p.step(100, 2)
        # term 3: replica 0 leads again on the same device ring.  (The oracle numbers a re-elected leader's entries
        # from where its own first term ended, so this term is checked on the engine's logs alone.)
        start = p.rep(1).offsets()["end"]
        last_idx = p.rep(1).stats()["entries_published"]
        if resident:
            p.take_over(0, [1, 2], old_votes=True, before_launch=p.g.prologue, check_commit=False)
            fail, pub, t3 = p.subs[0].result()
            assert fail is None and pub == len(second), (fail, pub)
            assert set(p.subs[0].terms_of_chunks()) == {3} and p.subs[0].not_leader() > 0
            assert sorted(t3) == list(range(2, 2 + len(second)))
            want = SB.ticket_order(second, t3)[0]
            p.g.tickets = 1 + len(second)
        else:                                            # the CONFIG and the requests after the winner's launch
            p.take_over(0, [1, 2], old_votes=True, check_commit=False)
            p.g.prologue()
            p.g.submit_stream(second)
            want = second
        p.relaunch(1)
        p.wait_commits(p.g.tickets)
        lead = p.leader
        wait_for(lambda: all(p.rep(i).stats()["entries_acked"] >= last_idx + p.g.tickets for i in (1, 2)),
                 "the followers hold the second term", timeout=30)
        assert lead.committed() == p.g.tickets and lead.stats()["tickets_submitted"] == p.g.tickets, \
            (lead.committed(), lead.stats()["tickets_submitted"], p.g.tickets)
        end = lead.offsets()["end"]
        img = lead.image()
        got = log_entries(img, start, end, L)
        assert [e[0] for e in got] == list(range(last_idx + 1, last_idx + 1 + p.g.tickets)), \
            ("idx", last_idx, [e[0] for e in got][:4], len(got), p.g.tickets)
        assert {e[1] for e in got} == {3} and got[0][2] == O.CONFIG, (got[0][:3],)
        assert [e[2:] for e in got[1:]] == [tuple(r) for r in want], "the second term's entries are not its requests"
        ents = O.walk_entries(img, start, end, L)
        for i in (1, 2):
            fi = p.rep(i).image()
            assert np.array_equal(O.mask_replies(fi, ents)[start:end], O.mask_replies(img, ents)[start:end]), i
        print(f"replica 0 led twice: {p.g.tickets} tickets in its second term, idx {last_idx + 1}..")
    finally:
        p.close()


def case_lifetime(eng, orc):
    n, L = 3, 1 << 20
    lib = eng.lib()
    TS.lib()
    with eng.Group(n, devices=devices_for(eng, n), log_size=L) as hm:
        with pytest.raises(E.ApusError, match="follower"):
            hm.replicas[1].submitter_attach()
    g = EU.device_group(eng, n, L)
    try:
        f, lead = g.replicas[1], g.leader
        st = new_stream(f.device)
        reqs = SB.mixed_requests(4, seed=41, reject_every=0)
        subs = [TS.Submitter(st, reqs, batch=1, timeout_s=60) for _ in range(2)]
        v = f.submitter_attach(st)
        with pytest.raises(E.ApusError, match="attached already"):
            f.submitter_attach(st)
        assert lib.apus_replica_set_role(f.h, 0, 1) == E.APUS_OK, lib.apus_last_error()   # dormant: accepted
        ls = new_stream(lead.device)
        lead.submitter_attach(ls)
        assert lib.apus_replica_set_role(lead.h, 0, 2) == E.APUS_ERROR
        assert b"detach first" in lib.apus_last_error()
        lead.submitter_detach()
        # a dormant kernel polls until detach ends it STOPPED; the host ring is untouched
        subs[0].start(v)
        time.sleep(0.2)
        t0 = time.time()
        f.submitter_detach()
        assert time.time() - t0 < 5
        fail, pub, _ = subs[0].result()
        assert fail == (SB.STEP_RESERVE, SB.STOPPED) and pub == 0 and subs[0].not_leader() > 0, fail
        # ... and destroy ends it STOPPED too (the follower's own: freeing another replica's memory would wait for it)
        v = f.submitter_attach(st)
        subs[1].start(v)
        time.sleep(0.2)
        t0 = time.time()
        f.close()
        assert time.time() - t0 < 10
        fail, pub, _ = subs[1].result()
        assert fail == (SB.STEP_RESERVE, SB.STOPPED) and pub == 0, fail
        print("dormant kernels ended STOPPED by detach and by destroy")
    finally:
        g.close()


if __name__ == "__main__":
    EU.worker_main(globals())
