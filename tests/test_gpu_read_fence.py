"""Read fences (apus_read_fence): linearizable reads from any replica's device state.  A fence confirms the leader this
replica knew against a majority of SIDs, takes its commit, and waits in stream order until this replica holds the
committed entries through it and the last of them is of the leader's term; the application then answers a read from a
state that has applied through the fence's read index F.  Every fence has a finite timeout, so a defect shows up as an
outcome word or an assertion, not as a stuck device.

As in test_gpu_consume_wait.py, every replica holds a resident launch plus a copy and a consume stream, and a pending
fence holds its consume stream's hardware queue (DESIGN.md s2).  So each case runs in a worker process of this file that
sets CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA starts.  Marked gpu."""
import os
import subprocess
import sys
import threading
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
from consumers import ANY, Consumer, catch_up, check_rows, close_all, consumer_group, new_stream, oracle_rows  # noqa: E402
from engine_util import MODES, devices_for, eng, run_case, tensors  # noqa: E402,F401
from shadow import elect, sid  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

FOREVER = EU.FOREVER
MAX_LEN = 64                   # longest cmd of the streams here: the strided stride, and the packed cap per row
SENTINEL = 0x5EED              # an index word no fence of these cases writes
UINT64_MAX = E.UINT64_MAX

LOAD_CASES = [(3, "strided"), (3, "packed"), (5, "strided"), (5, "packed")]


@pytest.mark.parametrize("n,layout", LOAD_CASES, ids=[f"n{n}-{lay}" for n, lay in LOAD_CASES])
def test_linearizable_under_load(eng, n, layout):
    """a writer thread submits a seeded stream through host and device batches without pause; every replica, the
    leader included, runs rounds of fence -> consume -> fold enqueued ahead of the host, reading the leader's committed
    tickets T0 before each fence.  Every fence is READY and the fold had applied through its F; a fence whose F is short
    of T0 (the tickets word runs a few stores ahead of the consumer record F covers) is followed by one more, which
    covers T0, and otherwise the fold had applied T0 and everything before it; at the end every replica's rows are the
    stream's and the oracle's"""
    run_case(__file__, "under_load", n=n, layout=layout)


def test_own_term_entry_after_a_takeover(eng):
    """a take-over whose voter and winner move their SIDs as dare_entry.c does: before the winner runs, a fence on the
    voter and one on the winner time out (their last committed entry is of the old term); a fence enqueued with a long
    timeout ends READY once the winner's blank CONFIG commits, with F at or past its idx.  A fence pending on the winner
    when apus_replica_set_role takes over ends RELEASED"""
    run_case(__file__, "own_term")


def test_deposed_leader(eng):
    """fences are READY on the leader and a follower; with a minority of SIDs moved to t+1 still READY; with a majority
    moved, NOT_LEADER on the leader (its SID still at t) and on a follower while the leader's kernel keeps committing,
    and a NOT_LEADER fence leaves its index word untouched"""
    run_case(__file__, "deposed")


def test_release_and_timeout(eng):
    """a pending 30 s fence ends RELEASED within 1 s at consume_wait_release (a later fence is not affected), at stop
    and at destroy, and at the destroy of a peer it maps; a fence after that peer's destroy counts it as not connected;
    a follower whose kernel is stopped times out; fences run in call order with consume waits and consume calls"""
    run_case(__file__, "release_timeout")


def test_refusals(eng):
    """a replica without F_DEVICE_APPLY | F_APPLY_ANY_ROLE, timeout_us 0 or above 60 s, a null or misaligned index, a
    misaligned outcome, and a replica that maps a peer through CUDA IPC: ApusError, with nothing enqueued and nothing
    written; a fence afterwards works"""
    run_case(__file__, "refusals")


# ---- the worker side ---------------------------------------------------------------------------------------------
def _word(t):
    return int(t.cpu()[0])


def _group(eng, n, L):
    return E.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES["index_earlyack"] | ANY)


class Rounds:
    """K rounds of read_fence -> consume -> fold on one replica's own stream, each round into its own slice of the
    output, index and outcome words.  The fold is the application's apply: `state` = the largest idx applied so far,
    `applied[k]` its value after round k."""

    def __init__(self, rep, layout, K, B):
        import torch
        self.rep, self.layout, self.K, self.B = rep, layout, K, B
        self.stream = new_stream(rep.device)
        dev, n = torch.device("cuda", rep.device), K * B
        with torch.cuda.stream(self.stream):
            self.idx = torch.zeros(n, dtype=torch.int64, device=dev)
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
            self.index = torch.zeros(K, dtype=torch.int64, device=dev)
            self.outcome = torch.full((K,), -1, dtype=torch.int32, device=dev)
            self.state = torch.zeros(1, dtype=torch.int64, device=dev)
            self.applied = torch.zeros(K, dtype=torch.int64, device=dev)
            self.fold(slice(0, 1), 0)                  # loads the fold's kernels before any replica kernel is resident
            self.state.zero_()
        self.stream.synchronize()
        self.t0 = [0] * K

    def fold(self, s, k):
        """on the stream: state = max(state, idx of the rows in s), applied[k] = state (rows past count are 0)"""
        import torch
        torch.maximum(self.state, self.idx[s].amax(0, keepdim=True), out=self.state)
        self.applied[k:k + 1].copy_(self.state)

    def enqueue(self, k, t0, timeout_us=20_000_000):
        import torch
        B, s = self.B, slice(k * self.B, (k + 1) * self.B)
        self.t0[k] = t0
        self.rep.read_fence(timeout_us, index=self.index[k:k + 1], outcome=self.outcome[k:k + 1], stream=self.stream)
        head = (self.idx[s], self.types[s], self.conns[s], self.req[s])
        if self.layout == "strided":
            self.rep.consume_device(B, MAX_LEN, out=head + (self.lens[s], self.pay[s], self.count[k:k + 1]),
                                    stream=self.stream)
        else:
            cap = B * MAX_LEN
            self.rep.consume_device_packed(B, cap, out=head + (self.offs[k * (B + 1):(k + 1) * (B + 1)],
                                                               self.vals[k * cap:(k + 1) * cap], self.count[k:k + 1]),
                                           stream=self.stream)
        with torch.cuda.stream(self.stream):          # (the row indices are zeroed after each read-back)
            self.fold(s, k)

    def finish(self, deadline):
        """wait for the stream without blocking past `deadline`; returns (outcomes, F, applied, rows) and clears the
        row indices for the next batch of rounds"""
        import torch
        ev = torch.cuda.Event()
        ev.record(self.stream)
        while not ev.query():
            if time.time() > deadline:
                self.rep.consume_wait_release()
                self.stream.synchronize()
                raise AssertionError(f"replica {self.rep.idx}: its rounds did not end in time; outcomes "
                                     f"{self.outcome.cpu().tolist()}")
            time.sleep(0.002)
        out, F, app, cnt = (t.cpu().numpy() for t in (self.outcome, self.index, self.applied, self.count))
        idx, ty, co, rq = (t.cpu().numpy() for t in (self.idx, self.types, self.conns, self.req))
        if self.layout == "strided":
            ln, pl = self.lens.cpu().numpy(), self.pay.cpu().numpy()
        else:
            of, va = self.offs.cpu().numpy(), self.vals.cpu().numpy()
        rows = []
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
        with torch.cuda.stream(self.stream):
            self.idx.zero_()
            self.outcome.fill_(-1)
        return out, F, app, rows


def pieces(n_req, seed):
    """n_req SENDs in pieces of 20..200 that alternate between the host (one length per piece: apus_submit_uniform)
    and device tensors (ragged 0..MAX_LEN B: apus_submit_device)"""
    rng = np.random.default_rng(seed)
    out, rid = [], 1
    while rid <= n_req:
        m = min(int(rng.integers(20, 201)), n_req - rid + 1)
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


def case_under_load(eng, orc, n, layout):
    L, K, B, batches = 1 << 23, 8, 16384, 6
    parts = pieces(40_000, seed=500 + n + (3 if layout == "packed" else 0))
    allreq = [x for p in parts for x in p]
    reps = consumer_group(eng, n, L, leader_flags=ANY, follower_flags=[ANY] * (n - 1), ring_mode=E.RING_DEVICE)
    lead = reps[0]
    failure = []
    stop_writer = threading.Event()

    def writer():
        try:
            for k, part in enumerate(parts):
                if stop_writer.is_set():
                    break
                while True:
                    try:
                        submit_piece(lead, k, part)
                        break
                    except BlockingIOError:             # ring full: the consumers hold the pruning back
                        time.sleep(0.001)
                time.sleep(0.002)
        except BaseException as e:                      # noqa: BLE001 - reported by the main thread
            failure.append(e)

    try:
        rounds = {i: Rounds(reps[i], layout, K, B) for i in range(n)}
        cons = {i: Consumer(reps[i], MAX_LEN, 512, new_stream(reps[i].device)) for i in range(n)}
        EU.launch_each(eng, reps, FOREVER)
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)), 10_000_000)
        th = threading.Thread(target=writer)
        th.start()
        rows = {i: [] for i in range(n)}
        fences = short = 0
        for b in range(batches):
            for k in range(K):
                for i in range(n):
                    rounds[i].enqueue(k, lead.committed())      # T0 read before this fence is enqueued
            deadline = time.time() + 60
            for i in range(n):
                out, F, app, got = rounds[i].finish(deadline)
                assert np.all(out == E.WAIT_READY), f"replica {i}, batch {b}: outcomes {out.tolist()}"
                behind = 0
                for k in range(K):
                    t0 = rounds[i].t0[k]
                    # no HEAD entries (no pruning rule) and one CONFIG at idx 1: entry idx == ticket.  T0 comes from
                    # the tickets word, which the leader's commit warp stores a few stores before its consumer record,
                    # the word F is guaranteed to cover (apus_gpu.h): a fence that began in between may end short of
                    # T0, and the application then fences again
                    if F[k] < t0:
                        behind = max(behind, t0)
                        short += 1
                    elif t0 >= 2:
                        assert app[k] >= t0, f"replica {i}, batch {b}, round {k}: applied {app[k]} < T0 {t0}"
                    if F[k] >= 2:
                        assert app[k] >= F[k], f"replica {i}, batch {b}, round {k}: applied {app[k]} < F {F[k]}"
                if behind:
                    ix, oc = reps[i].read_fence(20_000_000, stream=rounds[i].stream)
                    rounds[i].stream.synchronize()
                    assert _word(oc) == E.WAIT_READY and _word(ix) >= behind, (i, b, _word(oc), _word(ix), behind)
                fences += K
                rows[i] += got
            assert not failure, failure
        stop_writer.set()
        th.join()
        assert not failure, failure
        t_last = lead.submit(S.SEND, 9, 10**6, b"last")
        lead.wait_committed(t_last, 10_000_000)
        stream = allreq[:t_last - 2] + [(S.SEND, 9, 10**6, b"last")]     # ticket 1 is the CONFIG
        for i in range(n):
            catch_up(cons[i])
            check_rows(rows[i] + cons[i].rows, stream, first_idx=2)
        EU.stop_each(eng, reps)
        c = EU.oracle_cluster(orc, n, L, stream)
        for i in range(n):
            assert rows[i] + cons[i].rows == oracle_rows(c, i), f"replica {i}: rows differ from the oracle's log"
        c.close()
        print(f"{fences} fences READY over {len(stream)} requests; {short} ended short of T0 and were followed by one more")
    finally:
        stop_writer.set()
        close_all(eng, reps)


def _set_sid(lib, rep, s):
    E._ck(lib.apus_ctl_set_sid(rep.h, s), "apus_ctl_set_sid")


def case_own_term(eng, orc):
    import torch
    n, L = 3, 1 << 20
    g = _group(eng, n, L)
    lib = eng.lib()
    c = None
    try:
        st = {i: new_stream(g.replicas[i].device) for i in (1, 2)}
        EU.launch_each(eng, g.replicas, FOREVER)
        g.prologue()
        stream = S.ragged_stream(300, MAX_LEN, conns=3, seed=91, close_every=40)
        g.leader.wait_committed(EU.submit_all(g.leader, stream))
        t_end = time.time() + 30
        while any(g.replicas[i].stats()["entries_acked"] < len(stream) + 1 for i in (1, 2)):
            assert time.time() < t_end
            time.sleep(0.002)
        EU.stop_each(eng, g.replicas)
        c = EU.oracle_cluster(orc, n, L, stream)
        # the winner-to-be learns of term 2 first (its candidacy), so a fence on it waits for an entry of term 2; the
        # take-over's set_role releases that fence
        E._ck(lib.apus_replica_set_role(g.replicas[1].h, 0, 2), "apus_replica_set_role")
        pend = g.replicas[1].read_fence(30_000_000, stream=st[1])
        time.sleep(0.2)
        assert not st[1].query(), "a fence that cannot become ready has ended"
        # the voter and the winner move their SIDs to the new term before the votes, as dare_entry.c's elect does
        for i in (1, 2):
            _set_sid(lib, g.replicas[i], sid(2, 0, 1))
        t0 = time.perf_counter()
        elect(eng, g, c, [1, 2], 1, [2], 2)
        st[1].synchronize()
        assert _word(pend[1]) == E.WAIT_RELEASED and time.perf_counter() - t0 < 5.0, _word(pend[1])
        # before the winner runs: its commit covers only old-term entries, so no fence can be READY
        for i in (1, 2):
            ix, oc = g.replicas[i].read_fence(300_000, stream=st[i])
            st[i].synchronize()
            assert _word(oc) == E.WAIT_TIMED_OUT, (i, _word(oc))
            assert g.replicas[i].read_fence_status() == (E.WAIT_TIMED_OUT, 0)
        # a long fence on the voter, then the new term runs: READY once the blank CONFIG commits
        ix, oc = g.replicas[2].read_fence(20_000_000, stream=st[2])
        g.prologue()
        c.prologue()
        for _ in range(2):
            c.round()
        cfg_idx = len(stream) + 2                         # the old CONFIG and stream, then the new CONFIG
        EU.launch_each(eng, [g.replicas[1], g.replicas[2]], FOREVER)
        st[2].synchronize()
        assert _word(oc) == E.WAIT_READY, _word(oc)
        assert _word(ix) >= cfg_idx, (_word(ix), cfg_idx)
        assert g.replicas[2].read_fence_status() == (E.WAIT_READY, _word(ix))
        ix1, oc1 = g.replicas[1].read_fence(20_000_000, stream=st[1])
        st[1].synchronize()
        assert _word(oc1) == E.WAIT_READY and _word(ix1) >= cfg_idx, (_word(oc1), _word(ix1))
        EU.stop_each(eng, [g.replicas[1], g.replicas[2]])
        print(f"F {_word(ix)} on the voter, {_word(ix1)} on the winner; blank CONFIG at idx {cfg_idx}")
    finally:
        for r in g.replicas:
            try:
                EU.stop_each(eng, [r])
            except Exception:      # noqa: BLE001 - not running
                pass
        g.close()
        if c is not None:
            c.close()


def _fence(rep, stream, timeout_us=5_000_000):
    """one fence with its index word pre-set to SENTINEL; returns (outcome, index word)"""
    import torch
    with torch.cuda.stream(stream):
        ix = torch.full((1,), SENTINEL, dtype=torch.int64, device=torch.device("cuda", rep.device))
    _, oc = rep.read_fence(timeout_us, index=ix, stream=stream)
    stream.synchronize()
    return _word(oc), _word(ix)


def case_deposed(eng, orc):
    n, L = 5, 1 << 20
    g = _group(eng, n, L)
    lib = eng.lib()
    try:
        st = {i: new_stream(g.replicas[i].device) for i in range(n)}
        EU.launch_each(eng, g.replicas, FOREVER)
        g.leader.wait_committed(g.prologue())
        t = g.submit(S.SEND, 1, 1, b"one")
        g.leader.wait_committed(t)
        for i in (0, 3):
            o, f = _fence(g.replicas[i], st[i])
            assert o == E.WAIT_READY and f >= t, (i, o, f)
        # a minority at t+1 (a candidate and one voter of a newer term that has not won): still READY
        for i in (3, 4):
            _set_sid(lib, g.replicas[i], sid(2, 0, 3))
        for i in (0, 1, 3):
            o, f = _fence(g.replicas[i], st[i])
            assert o == E.WAIT_READY and f >= t, ("minority", i, o, f)
        # a majority at t+1: a newer leader may exist.  The old leader's kernel runs on and still commits
        _set_sid(lib, g.replicas[2], sid(2, 0, 3))
        t = g.submit(S.SEND, 1, 2, b"two")
        g.leader.wait_committed(t)
        for i in (0, 1, 3):
            o, f = _fence(g.replicas[i], st[i])
            assert o == E.WAIT_NOT_LEADER and f == SENTINEL, ("majority", i, o, f)
            assert g.replicas[i].read_fence_status() == (E.WAIT_NOT_LEADER, 0)
        t = g.submit(S.SEND, 1, 3, b"three")
        g.leader.wait_committed(t)                        # the leader's kernel keeps running
        print("READY with a minority at t+1, NOT_LEADER with a majority on the leader and on followers")
    finally:
        try:
            EU.stop_each(eng, g.replicas)
        finally:
            g.close()


def _pending(rep, stream, oc):
    """a fence that cannot become READY (nothing committed yet, or this replica's kernel is stopped behind the leader's
    commit), 30 s long, left to run for a moment"""
    rep.read_fence(30_000_000, outcome=oc, stream=stream)
    time.sleep(0.2)
    assert not stream.query(), "a fence that cannot become ready has ended"


def case_release_timeout(eng, orc):
    import torch
    n, L = 5, 1 << 20
    g = _group(eng, n, L)
    try:
        reps, r = g.replicas, g.replicas[1]
        dev = torch.device("cuda", r.device)
        st = {i: new_stream(reps[i].device) for i in range(n)}
        oc = torch.full((8,), -1, dtype=torch.int32, device=dev)
        EU.launch_each(eng, reps, FOREVER)
        # consume_wait_release, then stop: nothing is committed yet, so these fences could only end by a release
        for q, release in ((0, r.consume_wait_release), (1, lambda: EU.stop_each(eng, reps))):
            _pending(r, st[1], oc[q:q + 1])
            t0 = time.perf_counter()
            release()
            st[1].synchronize()
            assert _word(oc[q:q + 1]) == E.WAIT_RELEASED and time.perf_counter() - t0 < 1.0, (q, _word(oc[q:q + 1]))
            assert r.read_fence_status() == (E.WAIT_RELEASED, 0)
        EU.launch_each(eng, reps, FOREVER)
        # call order with consume waits and consume calls: wait(2) -> fence -> consume -> fence, the later fence not
        # affected by the releases before it
        cn = Consumer(r, MAX_LEN, 512, st[1])
        r.consume_wait(2, 10_000_000, outcome=oc[2:3], stream=st[1])
        ix, _ = r.read_fence(10_000_000, outcome=oc[3:4], stream=st[1])
        g.leader.wait_committed(g.prologue())
        t = g.submit(S.SEND, 1, 1, b"after the release")
        g.leader.wait_committed(t)
        k, cst = cn.step(64)
        ix2, _ = r.read_fence(10_000_000, outcome=oc[4:5], stream=st[1])
        st[1].synchronize()
        assert [_word(oc[q:q + 1]) for q in (2, 3, 4)] == [E.WAIT_READY] * 3, oc.cpu().tolist()
        assert _word(ix) == 2 and k == 1 and cst.next_idx == 3 and _word(ix2) == 2, (_word(ix), k, cst, _word(ix2))
        # followers 3 and 4 stopped; the leader commits on with 1 and 2; a fence on 3 times out
        EU.stop_each(eng, [reps[3], reps[4]])
        g.leader.wait_committed(g.submit(S.SEND, 1, 2, b"without 3 and 4"))
        t0 = time.perf_counter()
        _, o3 = reps[3].read_fence(300_000, stream=st[3])
        st[3].synchronize()
        dt = time.perf_counter() - t0
        assert _word(o3) == E.WAIT_TIMED_OUT and 0.3 <= dt < 3.0, (_word(o3), dt)
        # the destroy of 4 ends its own pending fence and the one pending on 3, which maps it.  (Freeing a region
        # waits for the kernels resident on its GPU, so the running replicas stop first; stopping them releases only
        # their own fences.)
        EU.stop_each(eng, reps[:3])
        o = {i: torch.full((1,), -1, dtype=torch.int32, device=torch.device("cuda", reps[i].device)) for i in (3, 4)}
        for i in (3, 4):
            _pending(reps[i], st[i], o[i])
        t0 = time.perf_counter()
        reps[4].close()
        dt = time.perf_counter() - t0
        for i in (3, 4):
            st[i].synchronize()
        assert (_word(o[3]), _word(o[4])) == (E.WAIT_RELEASED, E.WAIT_RELEASED) and dt < 2.0, (_word(o[3]), _word(o[4]), dt)
        # a fence after it counts 4 as not connected: four of five members left at term t, READY
        EU.launch_each(eng, reps[:3], FOREVER)
        ix3, o1 = r.read_fence(10_000_000, stream=st[1])
        st[1].synchronize()
        assert _word(o1) == E.WAIT_READY and _word(ix3) == 3, (_word(o1), _word(ix3))
        # destroy of the replica itself
        EU.stop_each(eng, reps[:3])
        _pending(reps[3], st[3], o[3])
        t0 = time.perf_counter()
        reps[3].close()
        st[3].synchronize()
        assert _word(o[3]) == E.WAIT_RELEASED and time.perf_counter() - t0 < 2.0, _word(o[3])
        print("released at consume_wait_release, stop, a peer's destroy and destroy; timed out on a stopped follower")
    finally:
        for x in g.replicas:
            if x.h:
                try:
                    EU.stop_each(eng, [x])
                except Exception:      # noqa: BLE001 - not running
                    pass
        g.close()


IPC_PEER = r"""
import sys
sys.path.insert(0, sys.argv[1])
from apus_b200 import engine as E
r = E.Replica(0, 1, 2, 0, 1, 1 << 20, flags=E.F_DEVICE_STATS | E.F_DEVICE_APPLY | E.F_APPLY_ANY_ROLE)
print(r.export().hex(), flush=True)
sys.stdin.readline()
r.close()
"""


def case_refusals(eng, orc):
    import torch
    n, L = 3, 1 << 20
    reps = consumer_group(eng, n, L, leader_flags=ANY, follower_flags=[E.F_DEVICE_APPLY, 0])
    try:
        r0 = reps[0]
        dev = torch.device("cuda", r0.device)
        s = new_stream(r0.device)
        buf = torch.zeros(4, dtype=torch.int64, device=dev)
        ob = torch.zeros(4, dtype=torch.int32, device=dev)
        lib = E.lib()
        for args, msg in (((0,), "timeout_us"), ((60_000_001,), "timeout_us")):
            with pytest.raises(E.ApusError, match=msg):
                r0.read_fence(*args, stream=s)
        for rep in (reps[1], reps[2]):
            with pytest.raises(E.ApusError, match="APUS_F_DEVICE_APPLY \\| APUS_F_APPLY_ANY_ROLE"):
                rep.read_fence(1000)
        with pytest.raises(E.ApusError, match="null argument"):
            E._ck(lib.apus_read_fence(r0.h, 1000, None, None, s.cuda_stream), "apus_read_fence")
        with pytest.raises(E.ApusError, match="misaligned"):
            E._ck(lib.apus_read_fence(r0.h, 1000, buf.data_ptr() + 4, None, s.cuda_stream), "apus_read_fence")
        with pytest.raises(E.ApusError, match="misaligned"):
            E._ck(lib.apus_read_fence(r0.h, 1000, buf.data_ptr(), ob.data_ptr() + 1, s.cuda_stream), "apus_read_fence")
        with pytest.raises(E.ApusError, match="dtype"):
            r0.read_fence(1000, index=torch.zeros(1, dtype=torch.int32, device=dev), stream=s)
        # a replica of another process, mapped through CUDA IPC
        p = subprocess.Popen([sys.executable, "-c", IPC_PEER, os.path.dirname(HERE)], stdin=subprocess.PIPE,
                             stdout=subprocess.PIPE, text=True)
        try:
            blob = bytes.fromhex(p.stdout.readline().strip())
            solo = E.Replica(r0.device, 0, 2, 0, 1, 1 << 20, flags=MODES["index_earlyack"] | ANY)
            try:
                solo.connect(1, blob)
                with pytest.raises(E.ApusError, match="CUDA IPC"):
                    solo.read_fence(1000, stream=s)
                assert solo.read_fence_status().outcome == UINT64_MAX
            finally:
                solo.close()
        finally:
            p.stdin.write("\n")
            p.stdin.flush()
            p.wait(60)
        s.synchronize()
        # nothing was enqueued or written
        assert r0.read_fence_status() == (UINT64_MAX, 0)
        assert buf.cpu().tolist() == [0] * 4 and ob.cpu().tolist() == [0] * 4
        # the bounds themselves are accepted, and a normal fence works
        EU.launch_each(eng, reps, FOREVER)
        r0.wait_committed(r0.submit(O.CONFIG, 0, 0, O.cid_image(n)))
        r0.read_fence(1, stream=s)
        ix, oc = r0.read_fence(60_000_000, stream=s)
        s.synchronize()
        assert _word(oc) == E.WAIT_READY and _word(ix) == 1, (_word(oc), _word(ix))
    finally:
        close_all(eng, reps)


if __name__ == "__main__":
    EU.worker_main(globals())
