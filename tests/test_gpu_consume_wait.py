"""Stream-ordered consume waits (apus_consume_wait): device consumers that wait for commits on the device, so that an
application enqueues wait -> consume many rounds ahead and synchronises only when it wants to.  Rows are checked against
the request stream and the CPU oracle's log; every wait has a finite timeout, so a defect shows up as an outcome word
or an assertion, not as a stuck device.

As in test_gpu_consume_any_role.py, every replica holds a resident launch plus a copy and a consume stream and the
consumers bring torch streams of their own; a pending wait also holds its consume stream's hardware queue (DESIGN.md
s2).  So each case runs in a worker process of this file that sets CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA starts.
Marked gpu."""
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
import streams as S  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consumers import (ANY, Consumer, catch_up, check_rows, close_all, consumer_group, idx_cap,  # noqa: E402
                       new_stream, oracle_rows, wait_forwarded_all)
from engine_util import MODES, devices_for, eng, run_case, submit_all, tensors  # noqa: E402,F401
from shadow import elect  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

FOREVER = EU.FOREVER
MAX_LEN = 300                  # longest cmd of the streams here: the strided stride, and the packed cap per row
NEVER = 1 << 12                # far more entries than the release cases commit: a wait for them never becomes ready


# N, consumer layout, a small pruning log that laps while waits are pending, consumers on the leader too
AHEAD_CASES = [(3, "strided", False, False), (3, "packed", False, False), (5, "strided", False, False),
               (5, "packed", False, False), (3, "strided", True, False), (5, "packed", True, False)]
LEADER_CASES = [(3, "strided", False, True), (5, "packed", False, True)]


@pytest.mark.parametrize("n,layout,lapping,leader", AHEAD_CASES,
                         ids=[f"n{n}-{lay}-{'lapping' if lap else 'flat'}" for n, lay, lap, _ in AHEAD_CASES])
def test_apply_loop_ahead_of_the_host(eng, n, layout, lapping, leader):
    """every follower enqueues K rounds of wait(B) -> consume(B) before the leader has a request; the requests then
    come in pieces (host submit_uniform and submit_device) with no host synchronise between rounds: every outcome is
    READY, the rows are the request stream and (where the log does not lap) the oracle's rows, and every cursor ends at
    the commit offset.  The lapping case prunes a 256 KiB log behind the consumers several times while waits are
    pending"""
    run_case(__file__, "apply_ahead", n=n, layout=layout, lapping=lapping, leader=leader)


@pytest.mark.parametrize("n,layout,lapping,leader", LEADER_CASES, ids=[f"n{n}-{lay}" for n, lay, _, _ in LEADER_CASES])
def test_apply_loop_ahead_on_the_leader(eng, n, layout, lapping, leader):
    """the same with APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE on every replica: the leader's own waits are READY and
    its rows are the stream's and the oracle's"""
    run_case(__file__, "apply_ahead", n=n, layout=layout, lapping=lapping, leader=leader)


def test_already_ready(eng):
    """a wait for entries that are already committed ends READY at once (host clock far under its timeout), and the
    consume after it delivers them"""
    run_case(__file__, "already_ready")


def test_timeout(eng):
    """wait(1, 200 ms) with nothing submitted ends TIMED_OUT after at least 200 ms on the host clock and within a
    generous bound; the consume after it delivers no row and leaves the cursor where it was"""
    run_case(__file__, "timeout")


def test_release_points(eng):
    """a pending 30 s wait ends RELEASED within 1 s at consume_wait_release (a later wait is not affected), at
    Group.stop() and at close() (destroy)"""
    run_case(__file__, "release")


def test_release_at_takeover(eng):
    """a pending 30 s wait on a follower that takes over ends RELEASED at apus_replica_set_role, which then returns
    within 1 s; a wait enqueued after it sees the old-term entries that commit with the new leader's blank CONFIG, and
    the new leader's rows equal the oracle's"""
    run_case(__file__, "release_takeover")


def test_refusals(eng):
    """min_entries 0 or above idx_cap, timeout_us 0 or above 60 s, a replica without APUS_F_DEVICE_APPLY, a leader
    without APUS_F_APPLY_ANY_ROLE, a misaligned, wrong-device or wrong-dtype outcome: ApusError, nothing enqueued; a
    normal wait and consume work afterwards"""
    run_case(__file__, "refusals")


# ---- the worker side ---------------------------------------------------------------------------------------------
class Ahead:
    """K rounds of consume_wait(B) -> consume(B) on one replica's own stream, each round into its own slice of the
    output and its own outcome word; read back once, at the end"""

    def __init__(self, rep, layout, K, B):
        import torch
        self.rep, self.layout, self.K, self.B = rep, layout, K, B
        self.stream = new_stream(rep.device)
        dev, n = torch.device("cuda", rep.device), K * B
        with torch.cuda.stream(self.stream):
            self.idx = torch.empty(n, dtype=torch.int64, device=dev)
            self.types = torch.empty(n, dtype=torch.uint8, device=dev)
            self.conns = torch.empty(n, dtype=torch.int16, device=dev)
            self.req = torch.empty(n, dtype=torch.int64, device=dev)
            if layout == "strided":
                self.lens = torch.empty(n, dtype=torch.int16, device=dev)
                self.pay = torch.empty((n, MAX_LEN), dtype=torch.uint8, device=dev)
            else:
                self.offs = torch.empty(K * (B + 1), dtype=torch.int64, device=dev)
                self.vals = torch.empty(K * B * MAX_LEN, dtype=torch.uint8, device=dev)
            self.count = torch.full((K,), -1, dtype=torch.int32, device=dev)
            self.outcome = torch.full((K,), -1, dtype=torch.int32, device=dev)

    def enqueue(self, k, timeout_us=10_000_000):
        B, s = self.B, slice(k * self.B, (k + 1) * self.B)
        self.rep.consume_wait(B, timeout_us, outcome=self.outcome[k:k + 1], stream=self.stream)
        head = (self.idx[s], self.types[s], self.conns[s], self.req[s])
        if self.layout == "strided":
            self.rep.consume_device(B, MAX_LEN, out=head + (self.lens[s], self.pay[s], self.count[k:k + 1]),
                                    stream=self.stream)
        else:
            cap = B * MAX_LEN
            self.rep.consume_device_packed(B, cap, out=head + (self.offs[k * (B + 1):(k + 1) * (B + 1)],
                                                               self.vals[k * cap:(k + 1) * cap], self.count[k:k + 1]),
                                           stream=self.stream)

    def finish(self, deadline):
        """wait for the stream without blocking past `deadline` (then release the waits, so that the stream ends);
        returns (outcomes, rows)"""
        import torch
        ev = torch.cuda.Event()
        ev.record(self.stream)
        while not ev.query():
            if time.time() > deadline:
                self.rep.consume_wait_release()
                self.stream.synchronize()
                raise AssertionError(f"replica {self.rep.idx}: its rounds did not end in time; outcomes "
                                     f"{self.outcome.cpu().tolist()}, counts {self.count.cpu().tolist()}")
            time.sleep(0.005)
        out = self.outcome.cpu().numpy()
        cnt = self.count.cpu().numpy()
        idx, ty, co, rq = (t.cpu().numpy() for t in (self.idx, self.types, self.conns, self.req))
        rows = []
        if self.layout == "strided":
            ln, pl = self.lens.cpu().numpy(), self.pay.cpu().numpy()
        else:
            of, va = self.offs.cpu().numpy(), self.vals.cpu().numpy()
        for k in range(self.K):
            for q in range(int(cnt[k])):
                j = k * self.B + q
                if self.layout == "strided":
                    cmd = pl[j, :int(ln[j]) & 0xFFFF].tobytes()
                else:
                    o = of[k * (self.B + 1):(k + 1) * (self.B + 1)]
                    base = k * self.B * MAX_LEN
                    cmd = va[base + int(o[q]):base + int(o[q + 1])].tobytes()
                rows.append((int(idx[j]), int(ty[j]), int(co[j]) & 0xFFFF, int(rq[j]), cmd))
        return out, cnt, rows


def pieces(n_req, seed):
    """n_req SENDs in pieces of 50..400 that alternate between the host (one shape per piece: apus_submit_uniform) and
    device tensors (ragged 0..MAX_LEN B: apus_submit_device)"""
    rng = np.random.default_rng(seed)
    out, rid = [], 1
    while rid <= n_req:
        m = min(int(rng.integers(50, 401)), n_req - rid + 1)
        if len(out) % 2 == 0:
            ln = int(rng.integers(0, MAX_LEN + 1))
            part = [(S.SEND, 3, rid + q, rng.bytes(ln)) for q in range(m)]
        else:
            part = [(S.SEND, 5, rid + q, rng.bytes(int(rng.integers(0, MAX_LEN + 1)))) for q in range(m)]
        out.append(part)
        rid += m
    return out


def submit_piece(lead, k, part):
    if k % 2 == 0:
        ln = len(part[0][3])
        pl = np.frombuffer(b"".join(p for *_, p in part), dtype=np.uint8) if ln else None
        return lead.submit_uniform(len(part), S.SEND, part[0][1], part[0][2], ln, pl) + len(part) - 1
    return lead.submit_device(*tensors(part, lead.device, MAX_LEN)) + len(part) - 1


def case_apply_ahead(eng, orc, n, layout, lapping, leader):
    B = 128
    if lapping:
        L, n_req, B = 1 << 18, 5200, 256  # about 4.3 laps of the log; the HEAD entries the leader adds are not counted
        K = (n_req + 1) // B              # ... so K * B <= the entries there will be: every round becomes ready
    else:
        L, K = 1 << 22, 24
        n_req = K * B - 1                 # the CONFIG and the requests fill the K rounds exactly
    parts = pieces(n_req, seed=300 + n + (7 if lapping else 0) + (11 if leader else 0))
    allreq = [x for p in parts for x in p]
    ff = [ANY if leader else E.F_DEVICE_APPLY] * (n - 1)
    reps = consumer_group(eng, n, L, leader_flags=(ANY if leader else 0) | (E.F_AUTOPRUNE if lapping else 0),
                          follower_flags=ff, ring_mode=E.RING_DEVICE)
    who = list(range(n)) if leader else list(range(1, n))
    try:
        got = {}
        ahead = {i: Ahead(reps[i], layout, K, B) for i in who}
        cons = {i: Consumer(reps[i], MAX_LEN, 512, new_stream(reps[i].device)) for i in who}  # the catch-up after the rounds
        # (the launch first: a launch copies its arguments on a stream that may share a queue with a pending wait)
        EU.launch_each(eng, reps, FOREVER)
        for i in who:                                                    # before the leader has any request
            for k in range(K):
                ahead[i].enqueue(k)
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = 0
        for k, part in enumerate(parts):
            t = submit_piece(lead, k, part)
        lead.wait_committed(t, 120_000_000)
        deadline = time.time() + 120
        for i in who:
            out, cnt, rows = ahead[i].finish(deadline)
            assert np.all(out == E.WAIT_READY), f"replica {i}: outcomes {out.tolist()}"
            assert reps[i].consume_wait_status().outcome == E.WAIT_READY
            # a READY wait for B entries and a consume of B entries: each round examined exactly B entries
            st = catch_up(cons[i])
            rows += cons[i].rows
            check_rows(rows, allreq, first_idx=2)
            assert st.error == 0
            if not lapping:
                assert st.next_idx == K * B + 1, st
            got[i] = rows
        heads = lead.stats()["auto_heads"]
        if lapping:
            assert heads >= 4, f"the log was pruned {heads} times: it did not lap while the waits were pending"
        wait_forwarded_all(reps)
        EU.stop_each(eng, reps)
        commit = lead.offsets()["commit"]
        for i in who:
            assert reps[i].consume_status().cursor == reps[i].offsets()["commit"] == commit
        if not lapping:
            c = EU.oracle_cluster(orc, n, L, allreq)
            import types as T
            EU.compare_group_to_oracle(T.SimpleNamespace(n=n, replicas=reps, leader_idx=0), c, exact=True)
            for i in who:
                assert got[i] == oracle_rows(c, i), f"replica {i}: rows differ from the oracle's log"
            c.close()
        print(f"{len(who)} consumers, {K} rounds of {B} each enqueued ahead, {heads} HEAD entries")
    finally:
        close_all(eng, reps)


def _group(eng, n, L):
    return E.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES["index_earlyack"] | ANY)


def _word(t):
    return int(t.cpu()[0])


def case_already_ready(eng, orc):
    import torch
    n, L = 3, 1 << 20
    reps = consumer_group(eng, n, L)
    try:
        cn = Consumer(reps[1], MAX_LEN, 512, new_stream(reps[1].device))
        oc = torch.full((1,), -1, dtype=torch.int32, device=torch.device("cuda", reps[1].device))
        EU.launch_each(eng, reps, FOREVER)
        stream = [(S.SEND, 2, 1 + k, bytes([k & 0xFF]) * (k % 90)) for k in range(100)]
        reps[0].submit(O.CONFIG, 0, 0, O.cid_image(n))
        reps[0].wait_committed(submit_all(reps[0], stream))
        commit = reps[0].offsets()["commit"]
        t_end = time.time() + 30
        while reps[1].offsets()["commit"] != commit:
            assert time.time() < t_end
            time.sleep(0.002)
        time.sleep(0.05)
        t0 = time.perf_counter()
        reps[1].consume_wait(101, 10_000_000, outcome=oc, stream=cn.stream)
        cn.stream.synchronize()
        dt = time.perf_counter() - t0
        assert _word(oc) == E.WAIT_READY and dt < 0.5, (_word(oc), dt)
        ws = reps[1].consume_wait_status()
        assert ws.outcome == E.WAIT_READY and ws.available == 101, ws
        k, st = cn.step(101)
        assert k == 100 and st.next_idx == 102 and st.cursor == commit, (k, st)
        check_rows(cn.rows, stream, first_idx=2)
        print(f"a ready wait took {dt * 1e3:.3f} ms on the host clock")
    finally:
        close_all(eng, reps)


def case_timeout(eng, orc):
    import torch
    n, L = 3, 1 << 20
    reps = consumer_group(eng, n, L)
    try:
        cn = Consumer(reps[1], MAX_LEN, 512, new_stream(reps[1].device))
        oc = torch.full((1,), -1, dtype=torch.int32, device=torch.device("cuda", reps[1].device))
        EU.launch_each(eng, reps, FOREVER)
        before = reps[1].consume_status()
        t0 = time.perf_counter()
        reps[1].consume_wait(1, 200_000, outcome=oc, stream=cn.stream)
        cn.stream.synchronize()
        dt = time.perf_counter() - t0
        assert _word(oc) == E.WAIT_TIMED_OUT, _word(oc)
        assert 0.2 <= dt < 2.0, dt
        assert reps[1].consume_wait_status() == (E.WAIT_TIMED_OUT, 0)
        k, st = cn.step(64)
        assert k == 0 and (st.cursor, st.next_idx) == (before.cursor, before.next_idx) == (0, 1), (k, st, before)
        print(f"a 200 ms wait took {dt * 1e3:.1f} ms on the host clock")
    finally:
        close_all(eng, reps)


def _pending(rep, oc, stream):
    """a wait that cannot become ready, 30 s long, left to run for a moment"""
    rep.consume_wait(NEVER, 30_000_000, outcome=oc, stream=stream)
    time.sleep(0.2)
    assert not stream.query(), "a wait that cannot become ready has ended"


def case_release(eng, orc):
    import torch
    n, L = 3, 1 << 20
    g = _group(eng, n, L)
    try:
        r = g.replicas[1]
        st = new_stream(r.device)
        oc = torch.full((4,), -1, dtype=torch.int32, device=torch.device("cuda", r.device))
        EU.launch_each(eng, g.replicas, FOREVER)
        g.leader.wait_committed(g.prologue())
        # apus_consume_wait_release; a wait enqueued after it is not affected
        _pending(r, oc[0:1], st)
        t0 = time.perf_counter()
        r.consume_wait_release()
        st.synchronize()
        dt = time.perf_counter() - t0
        assert _word(oc[0:1]) == E.WAIT_RELEASED and dt < 1.0, (_word(oc[0:1]), dt)
        assert r.consume_wait_status().outcome == E.WAIT_RELEASED
        r.consume_wait(2, 10_000_000, outcome=oc[1:2], stream=st)
        g.leader.wait_committed(g.submit(S.SEND, 1, 1, b"after the release"))
        st.synchronize()
        assert _word(oc[1:2]) == E.WAIT_READY and r.consume_wait_status() == (E.WAIT_READY, 2)
        # Group.stop()
        _pending(r, oc[2:3], st)
        t0 = time.perf_counter()
        g.stop()
        st.synchronize()
        dt = time.perf_counter() - t0
        assert _word(oc[2:3]) == E.WAIT_RELEASED and dt < 1.0, (_word(oc[2:3]), dt)
        # close(): destroy ends the wait before it frees the words the wait polls
        _pending(r, oc[3:4], st)
        t0 = time.perf_counter()
        r.close()
        dt = time.perf_counter() - t0
        st.synchronize()
        assert _word(oc[3:4]) == E.WAIT_RELEASED and dt < 1.0, (_word(oc[3:4]), dt)
        print("released at apus_consume_wait_release, apus_replicas_stop and apus_replica_destroy")
    finally:
        try:
            EU.stop_each(eng, [x for x in g.replicas if x.h])
        finally:
            g.close()


def case_release_takeover(eng, orc):
    import torch
    n, L = 3, 1 << 20
    g = _group(eng, n, L)
    cons = [Consumer(r, MAX_LEN, 512, new_stream(r.device)) for r in g.replicas]
    c = None
    try:
        oc = torch.full((2,), -1, dtype=torch.int32, device=torch.device("cuda", g.replicas[1].device))
        EU.launch_each(eng, g.replicas, FOREVER)
        g.prologue()
        stream = S.ragged_stream(300, MAX_LEN, conns=3, seed=77, close_every=40)
        g.leader.wait_committed(submit_all(g.leader, stream))
        _, st = cons[1].step(50)                          # the winner's consumer has read only part of the old term
        assert st.next_idx == 51, st
        t_end = time.time() + 30
        while any(g.replicas[i].stats()["entries_acked"] < len(stream) + 1 for i in (1, 2)):
            assert time.time() < t_end
            time.sleep(0.002)
        EU.stop_each(eng, g.replicas)
        c = EU.oracle_cluster(orc, n, L, stream)
        _pending(g.replicas[1], oc[0:1], cons[1].stream)
        t0 = time.perf_counter()
        elect(eng, g, c, [1, 2], 1, [2], 2)                # apus_replica_set_role drains the winner's consume stream
        dt = time.perf_counter() - t0
        cons[1].stream.synchronize()
        assert _word(oc[0:1]) == E.WAIT_RELEASED and dt < 1.0, (_word(oc[0:1]), dt)
        # the new term: its blank CONFIG commits the old-term entries the winner had not seen committed
        g.prologue()
        c.prologue()
        for _ in range(2):
            c.round()
        rest = len(stream) + 2 - 50                       # the old CONFIG and stream, the new CONFIG, minus what was read
        r = g.replicas[1]
        EU.launch_each(eng, [g.replicas[1], g.replicas[2]], FOREVER)
        r.consume_wait(rest, 20_000_000, outcome=oc[1:2], stream=cons[1].stream)
        k, st = cons[1].step(rest)
        assert _word(oc[1:2]) == E.WAIT_READY, _word(oc[1:2])
        assert r.consume_wait_status() == (E.WAIT_READY, rest)
        assert st.error == 0 and st.next_idx == len(stream) + 3, st
        assert cons[1].rows == oracle_rows(c, 1), "the new leader's rows differ from the oracle's"
        EU.stop_each(eng, [g.replicas[1], g.replicas[2]])
        assert st.cursor == r.offsets()["commit"] == c.offsets(1)["commit"]
        print(f"set_role returned in {dt * 1e3:.1f} ms; {len(cons[1].rows)} rows on the new leader")
    finally:
        for r in g.replicas:
            try:
                EU.stop_each(eng, [r])
            except Exception:      # noqa: BLE001 - not running
                pass
        g.close()
        if c is not None:
            c.close()


def case_refusals(eng, orc):
    import torch
    n, L = 3, 1 << 20
    reps = consumer_group(eng, n, L, follower_flags=[E.F_DEVICE_APPLY, 0])
    try:
        r = reps[1]
        dev = torch.device("cuda", r.device)
        cn = Consumer(r, MAX_LEN, 512, new_stream(r.device))
        buf = torch.zeros(8, dtype=torch.uint8, device=dev)
        cap = idx_cap(L)
        for args, msg in (((0, 1000), "min_entries"), ((cap + 1, 1000), "min_entries"), ((1, 0), "timeout_us"),
                          ((1, 60_000_001), "timeout_us")):
            with pytest.raises(E.ApusError, match=msg):
                r.consume_wait(*args, stream=cn.stream)
        r.consume_wait(cap, 1, stream=cn.stream)          # the bounds themselves are accepted: idx_cap, 1 us
        with pytest.raises(E.ApusError, match="needs a replica created with APUS_F_DEVICE_APPLY"):
            reps[2].consume_wait(1, 1000)
        with pytest.raises(E.ApusError, match="APUS_F_DEVICE_APPLY"):
            reps[2].consume_wait_release()
        with pytest.raises(E.ApusError, match="consumption is a follower's"):
            reps[0].consume_wait(1, 1000)
        with pytest.raises(E.ApusError, match="misaligned outcome"):
            E._ck(E.lib().apus_consume_wait(r.h, 1, 1000, buf.data_ptr() + 1, cn.stream.cuda_stream), "apus_consume_wait")
        with pytest.raises(E.ApusError, match="is on cpu"):
            r.consume_wait(1, 1000, outcome=torch.zeros(1, dtype=torch.int32))
        with pytest.raises(E.ApusError, match="dtype"):
            r.consume_wait(1, 1000, outcome=torch.zeros(1, dtype=torch.int64, device=dev), stream=cn.stream)
        with pytest.raises(E.ApusError, match="shape"):
            r.consume_wait(1, 1000, outcome=torch.zeros(2, dtype=torch.int32, device=dev), stream=cn.stream)
        cn.stream.synchronize()
        assert r.consume_wait_status().outcome == E.WAIT_TIMED_OUT    # the 1 us wait above, and no other
        # a normal wait and consume still work
        oc = torch.full((1,), -1, dtype=torch.uint32, device=dev)
        EU.launch_each(eng, reps, FOREVER)
        r.consume_wait(11, 10_000_000, outcome=oc, stream=cn.stream)
        reps[0].submit(O.CONFIG, 0, 0, O.cid_image(n))
        stream = [(S.SEND, 4, 1 + k, b"x" * k) for k in range(10)]
        reps[0].wait_committed(submit_all(reps[0], stream))
        k, st = cn.step(64)
        assert int(oc.cpu()[0]) == E.WAIT_READY and k == 10 and st.error == 0, (int(oc.cpu()[0]), k, st)
        check_rows(cn.rows, stream, first_idx=2)
    finally:
        close_all(eng, reps)


if __name__ == "__main__":
    EU.worker_main(globals())
