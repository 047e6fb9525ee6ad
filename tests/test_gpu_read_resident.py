"""Resident readers (apus_reader_attach, include/apus_reader.cuh): read fences run by the application's own persistent
kernel, with no host call per fence.  The test reader (tests/devicelogic/resident_reads.cu, tests/reader.py) fences on
several slots at once and logs, for every fence, the term and leader it took from the role word, K, the members its
confirmation counted, its outcome and F, and, beside a resident consumer, the idx that consumer had applied when the
read was served.  Every fence and every launch has a finite timeout, so a defect shows up as an outcome or an
assertion, not as a stuck device.

As in the other resident modules, each case runs in a worker process of this file that sets
CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA starts.  Marked gpu."""
import ctypes as C
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
import reader as RD  # noqa: E402
import resident as RS  # noqa: E402
import streams as S  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consumers import ANY, check_rows, close_all, consumer_group, new_stream  # noqa: E402
from engine_util import MODES, devices_for, eng, run_case, tensors  # noqa: E402,F401
from shadow import elect, sid  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

FOREVER = EU.FOREVER
MAX_LEN = 64
READY, TIMED_OUT, RELEASED, NOT_LEADER = E.WAIT_READY, E.WAIT_TIMED_OUT, E.WAIT_RELEASED, E.WAIT_NOT_LEADER

LOAD_CASES = [(3, "strided"), (3, "packed"), (5, "strided"), (5, "packed")]


@pytest.mark.parametrize("n,layout", LOAD_CASES, ids=[f"n{n}-{lay}" for n, lay in LOAD_CASES])
def test_linearizable_under_load(eng, n, layout):
    """a writer thread submits a seeded stream through host batches and strided or packed device batches; every
    replica, the leader included, runs a resident consumer and a resident reader with four slots fencing at once.  Every
    fence is READY with the role the group started with and every member counted, and the read is served at applied >=
    F; a fence whose F is short of T0 (the committed tickets read before it began) is followed in its slot by one that
    covers T0.  The consumers' rows are the stream's"""
    run_case(__file__, "under_load", n=n, layout=layout)


def test_takeover(eng):
    """with readers attached throughout: a fence pending on the winner-to-be when the take-over's set_role runs ends
    RELEASED; fences after set_role carry the new term and leader, time out on the voter and the winner until the
    winner's blank CONFIG commits, then end READY with F at or past its idx"""
    run_case(__file__, "takeover")


def test_deposed_leader(eng):
    """READY on the leader and a follower; with a minority of SIDs moved to t+1 still READY; with a majority moved,
    NOT_LEADER on the leader and on a follower while the leader's kernel keeps committing"""
    run_case(__file__, "deposed")


def test_disconnects_against_running_fences(eng):
    """four slots fence without pause while peers are disconnected one by one: once a disconnect has returned, no
    fence that began later counts that member; READY while a majority is mapped, NOT_LEADER below N/2 + 1 and without
    the leader, READY again after reconnecting"""
    run_case(__file__, "disconnects")


def test_release_points_and_lifetime(eng):
    """a 30 s fence ends RELEASED within 1 s at consume_wait_release, at stop, at detach and at a take-over's
    set_role; a follower whose kernel is stopped times out; destroy of the reader's own replica ends its fence; the
    destroy of a peer (resident kernels detached first) leaves that peer out of the table after reattach"""
    run_case(__file__, "release_lifetime")


def test_peer_destroy_on_another_gpu(eng):
    """the destroy of a peer on a second GPU while a reader on the first fences without pause: no fence that began
    after the destroy returned counts it"""
    if E.lib().apus_device_count() < 2:
        pytest.skip("needs a second GPU")
    run_case(__file__, "peer_other_gpu")


def test_refusals(eng):
    """no flags, a replica that maps a peer through CUDA IPC, a second attach, a null view, detach without attach and
    an IPC connect while attached: ApusError with nothing written.  Stream fences beside an attached reader are READY
    and agree with its F"""
    run_case(__file__, "refusals")


# ---- the worker side ---------------------------------------------------------------------------------------------
def _load():
    RS.lib()
    RD.lib()


def _group(eng, n, L, devices=None):
    return E.Group(n, devices=devices or devices_for(eng, n), log_size=L, flags=MODES["index_earlyack"] | ANY)


def _set_sid(lib, rep, s):
    E._ck(lib.apus_ctl_set_sid(rep.h, s), "apus_ctl_set_sid")


def _members(view):
    """the member words of an attached reader's block (pinned: the device address is the host address)"""
    return list(C.cast(view.member, C.POINTER(C.c_uint64 * E.MAX_SERVERS)).contents)


def _packed(part, device):
    import torch
    dev = torch.device("cuda", device)
    offs = np.zeros(len(part) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(p) for *_, p in part])
    vals = np.frombuffer(b"".join(p for *_, p in part) or b"\0", dtype=np.uint8)
    return (torch.from_numpy(np.array([t for t, *_ in part], dtype=np.uint8)).to(dev),
            torch.from_numpy(np.array([c for _, c, _, _ in part], dtype=np.uint16).view(np.int16)).to(dev),
            torch.from_numpy(np.array([r for _, _, r, _ in part], dtype=np.uint64).view(np.int64)).to(dev),
            torch.from_numpy(offs).to(dev), torch.from_numpy(vals.copy()).to(dev))


def pieces(n_req, seed):
    """n_req SENDs in pieces of 20..200 that alternate between the host (one length per piece) and device tensors
    (ragged, 0..MAX_LEN B)"""
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


def submit_piece(lead, k, part, layout):
    if k % 2 == 0:
        ln = len(part[0][3])
        pl = np.frombuffer(b"".join(p for *_, p in part), dtype=np.uint8) if ln else None
        return lead.submit_uniform(len(part), S.SEND, part[0][1], part[0][2], ln, pl)
    if layout == "strided":
        return lead.submit_device(*tensors(part, lead.device, MAX_LEN))
    return lead.submit_device_packed(*_packed(part, lead.device))


def check_covering(fences, what):
    """the linearizability checks of every READY fence, slot by slot: served at applied >= F, and a fence whose F is
    short of T0 is followed by one that covers it.  Returns how many were short"""
    short = 0
    by_slot = {}
    for f in fences:
        by_slot.setdefault(f.slot, []).append(f)
    for s, fs in by_slot.items():
        for q, f in enumerate(fs):
            assert f.outcome == READY, (what, f)
            assert f.applied >= f.F, (what, "applied < F", f)
            if f.F < f.T0:
                short += 1
                if q + 1 < len(fs):
                    assert fs[q + 1].F >= f.T0, (what, "the next fence does not cover T0", f, fs[q + 1])
    return short


def case_under_load(eng, orc, n, layout):
    L = 1 << 23
    _load()
    parts = pieces(30_000, seed=700 + n + (3 if layout == "packed" else 0))
    allreq = [x for p in parts for x in p]
    reps = consumer_group(eng, n, L, leader_flags=ANY, follower_flags=[ANY] * (n - 1), ring_mode=E.RING_DEVICE)
    lead = reps[0]
    failure, cons, rds = [], {}, {}
    stop_writer = threading.Event()

    def writer():
        try:
            for k, part in enumerate(parts):
                if stop_writer.is_set():
                    break
                while True:
                    try:
                        submit_piece(lead, k, part, layout)
                        break
                    except BlockingIOError:             # ring full: the consumers hold the pruning back
                        time.sleep(0.001)
                time.sleep(0.002)
        except BaseException as e:                      # noqa: BLE001 - reported by the main thread
            failure.append(e)

    try:
        for i in range(n):
            cons[i] = RS.Resident(reps[i], new_stream(reps[i].device), stride=MAX_LEN, row_cap=1 << 16)
        EU.launch_each(eng, reps, FOREVER)
        for i in range(n):
            cons[i].start()
            rds[i] = RD.Reader(reps[i], new_stream(reps[i].device), slots=4, target=400, timeout_us=20_000_000,
                               gap_us=2000, deadline_s=120, log_cap=400, t0_word=lead.committed_word(),
                               consumer=cons[i]).start()
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)), 10_000_000)
        th = threading.Thread(target=writer)
        th.start()
        for i in range(n):
            rds[i].wait(150)
        stop_writer.set()
        th.join()
        assert not failure, failure
        t_last = lead.submit(S.SEND, 9, 10**6, b"last")
        lead.wait_committed(t_last, 10_000_000)
        fences = short = 0
        for i in range(n):
            why, fs = rds[i].detach()
            assert set(why.values()) == {RD.END_TARGET}, (i, why)
            assert len(fs) == 4 * 400, (i, len(fs))
            assert {(f.t, f.L, f.mask) for f in fs} == {(1, 0, (1 << n) - 1)}, (i, {(f.t, f.L, f.mask) for f in fs})
            short += check_covering(fs, f"replica {i}")
            fences += len(fs)
        stream = allreq[:t_last - 2] + [(S.SEND, 9, 10**6, b"last")]     # ticket 1 is the CONFIG
        for i in range(n):
            cons[i].wait_rows(len(stream))
            _, nrows, _ = cons[i].detach()
            check_rows(cons[i].rows(), stream, first_idx=2)
        print(f"{fences} resident fences READY over {len(stream)} requests; {short} ended short of T0 and were followed "
              f"by one that covers it")
    finally:
        stop_writer.set()
        for i, r in rds.items():
            try:
                reps[i].reader_detach()
            except E.ApusError:
                pass
        for i, c in cons.items():
            try:
                reps[i].consumer_detach()
            except E.ApusError:
                pass
        close_all(eng, reps)


def case_takeover(eng, orc):
    n, L = 3, 1 << 20
    _load()
    g = _group(eng, n, L)
    lib = eng.lib()
    c = None
    try:
        st = {i: new_stream(g.replicas[i].device) for i in (1, 2)}
        EU.launch_each(eng, g.replicas, FOREVER)
        g.prologue()
        stream = S.ragged_stream(300, MAX_LEN, conns=3, seed=93, close_every=40)
        g.leader.wait_committed(EU.submit_all(g.leader, stream))
        EU.wait_for(lambda: all(g.replicas[i].stats()["entries_acked"] >= len(stream) + 1 for i in (1, 2)), "acks")
        EU.stop_each(eng, g.replicas)
        c = EU.oracle_cluster(orc, n, L, stream)
        # the winner-to-be learns of term 2 first: a fence on it waits for an entry of term 2
        E._ck(lib.apus_replica_set_role(g.replicas[1].h, 0, 2), "apus_replica_set_role")
        pend = RD.Reader(g.replicas[1], st[1], slots=1, target=1, timeout_us=30_000_000).start()
        time.sleep(0.2)
        assert not pend.done(), "a fence that cannot become ready has ended"
        for i in (1, 2):
            _set_sid(lib, g.replicas[i], sid(2, 0, 1))
        t0 = time.perf_counter()
        elect(eng, g, c, [1, 2], 1, [2], 2)
        pend.wait(5)
        _, fs = pend.result()
        assert [(f.outcome, f.t, f.L) for f in fs] == [(RELEASED, 2, 0)], fs
        assert time.perf_counter() - t0 < 5.0
        # the same attachment on 1, a new one on 2: fences carry (2, 1) and time out until the blank CONFIG commits
        r1 = RD.Reader(g.replicas[1], st[1], slots=2, timeout_us=300_000, gap_us=1000, deadline_s=60).start(pend.view)
        r2 = RD.Reader(g.replicas[2], st[2], slots=2, timeout_us=300_000, gap_us=1000, deadline_s=60).start()
        time.sleep(1.0)
        g.prologue()
        c.prologue()
        for _ in range(2):
            c.round()
        cfg_idx = len(stream) + 2
        EU.launch_each(eng, [g.replicas[1], g.replicas[2]], FOREVER)
        g.leader.wait_committed(g.tickets)
        time.sleep(0.5)
        for i, r in ((1, r1), (2, r2)):
            _, fs = r.detach()
            assert fs and {(f.t, f.L) for f in fs} == {(2, 1)}, (i, {(f.t, f.L) for f in fs})
            outs = [f.outcome for f in fs]
            assert TIMED_OUT in outs and READY in outs, (i, outs)
            assert all(o in (READY, TIMED_OUT, RELEASED) for o in outs), (i, outs)
            for f in fs:
                if f.outcome == READY:
                    assert f.F >= cfg_idx, (i, f, cfg_idx)
            # per slot: timeouts, then READY from the blank CONFIG's commit on (the last fence may end at detach)
            for s in {f.slot for f in fs}:
                o = [f.outcome for f in fs if f.slot == s]
                first = o.index(READY)
                assert all(x == TIMED_OUT for x in o[:first]), (i, s, o)
                assert all(x == READY for x in o[first:-1]), (i, s, o)
        EU.stop_each(eng, [g.replicas[1], g.replicas[2]])
        print(f"RELEASED at set_role; TIMED_OUT then READY with F >= {cfg_idx} on the voter and the winner")
    finally:
        for r in g.replicas:
            try:
                EU.stop_each(eng, [r])
            except Exception:      # noqa: BLE001 - not running
                pass
        g.close()
        if c is not None:
            c.close()


def _burst(rep, stream, view, k=16, timeout_us=5_000_000):
    r = RD.Reader(rep, stream, slots=2, target=k, timeout_us=timeout_us).start(view)
    r.wait(30)
    return r.result()[1]


def case_deposed(eng, orc):
    n, L = 5, 1 << 20
    _load()
    g = _group(eng, n, L)
    lib = eng.lib()
    views = {}
    try:
        st = {i: new_stream(g.replicas[i].device) for i in range(n)}
        EU.launch_each(eng, g.replicas, FOREVER)
        g.leader.wait_committed(g.prologue())
        t = g.submit(S.SEND, 1, 1, b"one")
        g.leader.wait_committed(t)
        for i in (0, 1, 3):
            views[i] = g.replicas[i].reader_attach(st[i])
        for i in (0, 3):
            fs = _burst(g.replicas[i], st[i], views[i])
            assert all(f.outcome == READY and f.F >= t and f.mask == 0b11111 for f in fs), (i, fs[:2])
        for i in (3, 4):
            _set_sid(lib, g.replicas[i], sid(2, 0, 3))
        for i in (0, 1, 3):
            fs = _burst(g.replicas[i], st[i], views[i])
            assert all(f.outcome == READY and f.F >= t and f.mask == 0b00111 for f in fs), ("minority", i, fs[:2])
        _set_sid(lib, g.replicas[2], sid(2, 0, 3))
        t = g.submit(S.SEND, 1, 2, b"two")
        g.leader.wait_committed(t)
        for i in (0, 1, 3):
            fs = _burst(g.replicas[i], st[i], views[i])
            assert all(f.outcome == NOT_LEADER and f.mask == 0b00011 for f in fs), ("majority", i, fs[:2])
        g.leader.wait_committed(g.submit(S.SEND, 1, 3, b"three"))       # the leader's kernel keeps running
        print("READY with a minority at t+1, NOT_LEADER with a majority on the leader and on followers")
    finally:
        for i in views:
            g.replicas[i].reader_detach()
        try:
            EU.stop_each(eng, g.replicas)
        finally:
            g.close()


def case_disconnects(eng, orc):
    n, L = 5, 1 << 20
    _load()
    g = _group(eng, n, L)
    lib = eng.lib()
    r = None
    try:
        reps, me = g.replicas, g.replicas[1]
        s1 = new_stream(me.device)
        EU.launch_each(eng, reps, FOREVER)
        g.leader.wait_committed(g.prologue())
        t = g.submit(S.SEND, 1, 1, b"held everywhere")
        g.leader.wait_committed(t)
        ix, oc = me.read_fence(5_000_000, stream=s1)          # replica 1 holds everything the leader has committed
        s1.synchronize()
        assert (int(oc.cpu()[0]), int(ix.cpu()[0])) == (READY, t)
        EU.stop_each(eng, reps)
        blobs = {j: reps[j].export() for j in range(n)}
        r = RD.Reader(me, s1, slots=4, timeout_us=1_000_000, gap_us=20, deadline_s=60, log_cap=1 << 16).start()
        time.sleep(0.05)
        # (member disconnected, the members still counted, the outcome of a fence that begins after it)
        steps = [(4, 0b01111, READY), (3, 0b00111, READY), (2, 0b00011, NOT_LEADER), (0, 0, NOT_LEADER)]
        marks = []
        for m, _, _ in steps:
            before = r.begun()
            E._ck(lib.apus_replica_disconnect(me.h, m), "apus_replica_disconnect")
            marks.append((before, r.begun()))
            time.sleep(0.05)
        before = r.begun()
        for m in (0, 2, 3, 4):
            me.connect(m, blobs[m])
        after = r.begun()
        time.sleep(0.05)
        why, fs = r.detach()
        r = None
        assert set(why.values()) == {RD.END_STOP}, why
        by_slot = {}
        for f in fs:
            by_slot.setdefault(f.slot, []).append(f)
        for w, sf in by_slot.items():
            assert all(f.seq == q for q, f in enumerate(sf)), "log ordered by seq"
            for k, (m, mask, out) in enumerate(steps):
                # fences seq >= after_k began after call k returned; fence nxt - 1 may still have been reading the
                # member words when call k + 1 began
                after_k = marks[k][1][w]
                nxt = marks[k + 1][0][w] if k + 1 < len(steps) else before[w]
                assert nxt - after_k >= 3, (w, k, after_k, nxt)     # fences ran between the calls
                for f in sf[after_k:before[w] - 1]:                  # (before the reconnects)
                    assert not f.mask & (1 << m), (w, k, f)
                for f in sf[after_k:nxt - 1]:
                    assert (f.outcome, f.mask) == (out, mask), (w, k, f)
            tail = sf[after[w]:-1]
            assert tail and all((f.outcome, f.mask) == (READY, 0b11111) for f in tail), (w, tail[:2])
        print(f"{len(fs)} fences beside four disconnects and a reconnect; none counted a member after its disconnect")
    finally:
        if r is not None:
            me.reader_detach()
        try:
            EU.stop_each(eng, g.replicas)
        finally:
            g.close()


def _pending_reader(rep, stream, view=None, timeout_us=30_000_000):
    r = RD.Reader(rep, stream, slots=1, target=1, timeout_us=timeout_us).start(view)
    time.sleep(0.2)
    assert not r.done(), "a fence that cannot become ready has ended"
    return r


def _ends(r, outcome, within):
    t0 = time.perf_counter()
    r.wait(10)
    dt = time.perf_counter() - t0
    _, fs = r.result()
    assert len(fs) == 1 and fs[0].outcome == outcome and dt < within, (fs, dt)
    return fs[0]


def case_release_lifetime(eng, orc):
    n, L = 5, 1 << 20
    _load()
    g = _group(eng, n, L)
    lib = eng.lib()
    attached = set()
    try:
        reps, me = g.replicas, g.replicas[1]
        st = {i: new_stream(reps[i].device) for i in range(n)}
        EU.launch_each(eng, reps, FOREVER)
        # nothing committed yet: these fences can only end by a release
        r = _pending_reader(me, st[1])
        attached.add(1)
        me.consume_wait_release()
        _ends(r, RELEASED, 1.0)
        r = _pending_reader(me, st[1], r.view)
        EU.stop_each(eng, reps)
        _ends(r, RELEASED, 1.0)
        r = _pending_reader(me, st[1], r.view)
        me.reader_detach()
        attached.discard(1)
        _ends(r, RELEASED, 1.0)
        # a follower whose kernel is stopped behind the leader's commit times out
        EU.launch_each(eng, reps, FOREVER)
        g.leader.wait_committed(g.prologue())
        EU.stop_each(eng, [reps[3], reps[4]])
        g.leader.wait_committed(g.submit(S.SEND, 1, 1, b"without 3 and 4"))
        r3 = RD.Reader(reps[3], st[3], slots=1, target=1, timeout_us=300_000).start()
        attached.add(3)
        f = _ends(r3, TIMED_OUT, 3.0)
        assert 300e6 <= f.t_end - f.t_begin < 3e9, f
        # a take-over's set_role: the fence of a replica that has learnt of term 2 waits for an entry of term 2
        EU.stop_each(eng, reps[:3])
        E._ck(lib.apus_replica_set_role(me.h, 0, 2), "apus_replica_set_role")
        r = _pending_reader(me, st[1])
        attached.add(1)
        E._ck(lib.apus_replica_set_role(me.h, 1, 2), "apus_replica_set_role")
        f = _ends(r, RELEASED, 1.0)
        assert (f.t, f.L) == (2, 0), f
        # the destroy of the reader's own replica (3 is stopped behind the commit)
        r3 = _pending_reader(reps[3], st[3], r3.view)
        t0 = time.perf_counter()
        reps[3].close()
        attached.discard(3)
        assert time.perf_counter() - t0 < 2.0
        _ends(r3, RELEASED, 1.0)
        # the destroy of a peer, with every resident kernel of the GPU detached first: after reattach the peer is out of
        # the table, and a fence counts what is left
        me.reader_detach()
        attached.discard(1)
        reps[4].close()
        v = me.reader_attach(st[1])
        attached.add(1)
        mem = _members(v)
        assert [bool(x) for x in mem[:n]] == [True, True, True, False, False], mem
        assert mem[1] and all(x == 0 for x in mem[n:]), mem
        fs = _burst(me, st[1], v, k=4, timeout_us=300_000)
        assert all(f.mask == 0b00111 and (f.t, f.L) == (2, 1) for f in fs), fs
        print("RELEASED at consume_wait_release, stop, detach, set_role and destroy; TIMED_OUT on a stopped follower")
    finally:
        for i in attached:
            if g.replicas[i].h:
                g.replicas[i].reader_detach()
        for x in g.replicas:
            if x.h:
                try:
                    EU.stop_each(eng, [x])
                except Exception:      # noqa: BLE001 - not running
                    pass
        g.close()


def case_peer_other_gpu(eng, orc):
    n, L = 3, 1 << 20
    _load()
    g = _group(eng, n, L, devices=[0, 0, 1])
    r = None
    try:
        reps, me = g.replicas, g.replicas[1]
        s1 = new_stream(me.device)
        EU.launch_each(eng, reps, FOREVER)
        g.leader.wait_committed(g.prologue())
        EU.stop_each(eng, reps)
        r = RD.Reader(me, s1, slots=4, timeout_us=1_000_000, gap_us=20, deadline_s=60, log_cap=1 << 16).start()
        time.sleep(0.05)
        reps[2].close()
        b = r.begun()
        time.sleep(0.05)
        _, fs = r.detach()
        r = None
        for f in fs:
            assert f.outcome in (READY, RELEASED), f
            if f.seq >= b[f.slot]:
                assert not f.mask & 0b100, f
        print(f"{len(fs)} fences beside the destroy of a peer on another GPU")
    finally:
        if r is not None:
            me.reader_detach()
        try:
            EU.stop_each(eng, [x for x in g.replicas if x.h])
        finally:
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
    n, L = 3, 1 << 20
    _load()
    reps = consumer_group(eng, n, L, leader_flags=ANY, follower_flags=[E.F_DEVICE_APPLY, 0])
    lib = E.lib()
    attached = False
    try:
        r0 = reps[0]
        s = new_stream(r0.device)
        for rep in (reps[1], reps[2]):
            v = E.ReaderView()
            assert lib.apus_reader_attach(rep.h, s.cuda_stream, C.byref(v)) == E.APUS_ERROR
            assert b"APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE" in lib.apus_last_error()
            assert bytes(v) == bytes(C.sizeof(v))
        with pytest.raises(E.ApusError, match="no resident reader is attached"):
            r0.reader_detach()
        assert lib.apus_reader_attach(r0.h, s.cuda_stream, None) == E.APUS_ERROR
        assert lib.apus_last_error() == b"null argument"
        # a replica of another process, mapped through CUDA IPC
        p = subprocess.Popen([sys.executable, "-c", IPC_PEER, os.path.dirname(HERE)], stdin=subprocess.PIPE,
                             stdout=subprocess.PIPE, text=True)
        try:
            blob = bytes.fromhex(p.stdout.readline().strip())
            solo = E.Replica(r0.device, 0, 2, 0, 1, 1 << 20, flags=MODES["index_earlyack"] | ANY)
            try:
                solo.connect(1, blob)
                v = E.ReaderView()
                assert lib.apus_reader_attach(solo.h, s.cuda_stream, C.byref(v)) == E.APUS_ERROR
                assert b"CUDA IPC" in lib.apus_last_error() and bytes(v) == bytes(C.sizeof(v))
            finally:
                solo.close()
            # an IPC connect while a reader is attached
            solo = E.Replica(r0.device, 0, 2, 0, 1, 1 << 20, flags=MODES["index_earlyack"] | ANY)
            try:
                v = solo.reader_attach(s)
                before = _members(v)
                with pytest.raises(E.ApusError, match="resident reader is attached"):
                    solo.connect(1, blob)
                assert _members(v) == before
                with pytest.raises(E.ApusError, match="attached already"):
                    solo.reader_attach(s)
                solo.reader_detach()
            finally:
                solo.close()
        finally:
            p.stdin.write("\n")
            p.stdin.flush()
            p.wait(60)
        # beside an attached reader, stream fences are READY and agree with its F
        v = r0.reader_attach(s)
        attached = True
        with pytest.raises(E.ApusError, match="attached already"):
            r0.reader_attach(s)
        EU.launch_each(eng, reps, FOREVER)
        t = r0.submit(O.CONFIG, 0, 0, O.cid_image(n))
        r0.wait_committed(t)
        fs = _burst(r0, s, v, k=8, timeout_us=5_000_000)
        ix, oc = r0.read_fence(5_000_000, stream=s)
        s.synchronize()
        assert int(oc.cpu()[0]) == READY and all(f.outcome == READY and f.F == int(ix.cpu()[0]) == t for f in fs), fs
        assert r0.read_fence_status() == (READY, t)
        print("refusals with nothing written; stream and resident fences agree")
    finally:
        if attached:
            reps[0].reader_detach()
        close_all(eng, reps)


if __name__ == "__main__":
    EU.worker_main(globals())
