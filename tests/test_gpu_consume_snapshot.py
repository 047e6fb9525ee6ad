"""Replacing a lost replica of a group that applies in GPU memory (APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE): a
consumer's position is marked in stream order (apus_consume_mark) and the application's state copied right behind it
while the group runs; a fresh replica's consumers are seeded there (apus_consume_seed), and the leader's adjustment
accepts it from there and resends the live log.  Every replica folds its rows into a device state with an
order-sensitive fold, so a missed, repeated or reordered row shows as a different state.

Each case runs in a worker process of this file that sets CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA starts (as
test_gpu_consume_any_role does: the replicas' launches and side streams and the consumers' streams need more than the
default 8 hardware queues).  Marked gpu."""
import os
import sys
import threading
import time

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":
    os.environ["CUDA_DEVICE_MAX_CONNECTIONS"] = "32"         # before anything starts CUDA
    for p in (HERE, os.path.dirname(HERE)):
        if p not in sys.path:
            sys.path.insert(0, p)

import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402
import pytest  # noqa: E402

import engine_util as EU  # noqa: E402
import orc as O  # noqa: E402
import ring_edges as RE  # noqa: E402
import streams as S  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consumers import ANY, Consumer, PackedConsumer, check_rows, idx_cap, new_stream  # noqa: E402
from engine_util import MODES, devices_for, eng, run_case, wait_for  # noqa: E402,F401
from shadow import sid  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

FOREVER = EU.FOREVER
M64 = (1 << 64) - 1
INDEX_OFF = 65536 + 320 * 1024          # apus_layout.h APUS_INDEX_OFF: the offset index follows the log header


# ---- the pytest side: one worker process per case ------------------------------------------------------------------
# N, consumer layout, whose consumer is marked, whether the replacement's consumer is held back after the join
REPLACE_CASES = [(3, "strided", 0, True), (3, "packed", 1, False), (5, "packed", 0, False), (5, "strided", 2, False)]


@pytest.mark.parametrize("n,layout,source,hold", REPLACE_CASES,
                         ids=[f"n{n}-{lay}-from{s}" + ("-held" if h else "") for n, lay, s, h in REPLACE_CASES])
def test_replace_a_follower(eng, n, layout, source, hold):
    """a follower is lost for good and the rest prune past everything it held; a fresh replica is refused without a seed,
    then seeded at a mark of replica `source`'s consumer taken while the group runs, adjusted and relaunched: its state
    equals every other replica's after more traffic, its rows start at the mark and equal the source's from there, and
    its live log equals the leader's.  N = 3: leader and replacement alone then commit; `hold`: with the replacement's
    consumer held back the leader's head never passes its seed"""
    run_case(__file__, "replace", n=n, layout=layout, source=source, hold=hold)


def test_marks_at_the_ring_end(eng):
    """a mark whose cursor stands at a wrap gap (behind the last entry before the ring's end, the next entry wrapped to
    0) and one just after the wrap are both accepted, and the replacement then applies what every replica applies"""
    run_case(__file__, "ring_end")


def test_refusals_write_nothing(eng):
    """seed on a replica with entries, after a consume call, with its kernel in flight, or without
    APUS_F_APPLY_ANY_ROLE; adjustment with a seed behind the head (APUS_RETRY), past the commit, at a non-boundary or
    with the wrong idx; a misaligned mark: each refused, each writing nothing to the peer"""
    run_case(__file__, "refusals")


# ---- the device state: an order-sensitive fold of the rows -----------------------------------------------------------
P = 0x100000001B3                        # odd: invertible modulo 2**64
Q = pow(P, -1, 1 << 64)
HA, HB, HC, HD = 0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x27D4EB2F165667C5
MAXN = 4096


def s64(x):
    x &= M64
    return x - (1 << 64) if x >> 63 else x


def row_hash(idx, ty, conn, rq, ln):
    return (idx * HA + rq * HB + ((ty << 16) | conn) * HC + ln * HD) & M64


def fold_host(s, rows):
    """the fold of `rows` onto state word s, on the host: s := s * P + h(row), row by row"""
    for i, ty, co, rq, pl in rows:
        s = (s * P + row_hash(i, ty, co, rq, len(pl))) & M64
    return s


class Fold:
    """per device: Q**(i + 1) as an int64 table, so that k rows fold in one pass of device ops:
    s := P**k * (s + sum_i h_i * Q**(i + 1)) == s * P**k + sum_i h_i * P**(k - 1 - i) (all modulo 2**64).  Every view
    it takes starts where its tensor does, and P**k is a host scalar: the same kernels run whatever k is, so that
    warm_fold loads them all before the replica kernels are resident"""

    def __init__(self, device):
        import torch
        dev = torch.device("cuda", device)
        self.dev = dev
        self.qpow = torch.tensor([s64(pow(Q, i + 1, 1 << 64)) for i in range(MAXN)], dtype=torch.int64, device=dev)
        self.k = [s64(x) for x in (HA, HB, HC, HD)]

    def apply(self, state, k, idx, ty, conn, rq, ln):
        """fold rows 0 .. k-1 of the consume outputs into state[0], on the current stream"""
        import torch
        if k == 0:
            return
        h = (idx[:k] * self.k[0] + rq[:k] * self.k[1] +
             ((ty[:k].to(torch.int64) << 16) | (conn[:k].to(torch.int64) & 0xFFFF)) * self.k[2] +
             (ln[:k].to(torch.int64) & 0xFFFF) * self.k[3])
        state[:1].add_((h * self.qpow[:k]).sum())
        state[:1].mul_(s64(pow(P, k, 1 << 64)))


class Applier:
    """one replica's device consumer (strided or packed) on a stream of its own, applying every call's rows to its
    device state in stream order; from its own thread it also marks its position and copies the state right behind the
    mark when asked"""

    def __init__(self, rep, layout, fold, state=None, lens=()):
        import torch
        self.rep, self.layout, self.fold = rep, layout, fold
        stream = new_stream(rep.device)
        if layout == "strided":
            self.cn = Consumer(rep, 1500, MAXN, stream=stream)
        else:
            self.cn = PackedConsumer(rep, list(lens), max_n_cap=MAXN, cap_max=1 << 21, seed=rep.idx + 7)
            self.cn.stream = stream
        dev = torch.device("cuda", rep.device)
        with torch.cuda.stream(stream):
            self.state = torch.zeros(1, dtype=torch.int64, device=dev) if state is None else state.to(dev).clone()
            self.mark_buf = torch.zeros(2, dtype=torch.int64, device=dev)
        stream.synchronize()
        self.s0 = int(self.state.cpu()[0]) & M64
        self.want, self.snaps = threading.Event(), []
        self.halt, self.errs, self.th = threading.Event(), [], None

    def step(self, max_n):
        import torch
        k, st = self.cn.step(max_n)
        with torch.cuda.stream(self.cn.stream):
            if self.layout == "strided":
                idx, ty, co, rq, ln = self.cn.out[:5]
            else:
                idx, ty, co, rq, of = self.cn.buf[:5]
                ln = of[1:k + 1] - of[:k] if k else of[:0]
            self.fold.apply(self.state, k, idx, ty, co, rq, ln)
        if self.want.is_set():
            self.snapshot()
        return k, st

    def snapshot(self):
        """the mark and the state behind it, in this consumer's stream order; the rows received before the mark"""
        import torch
        self.want.clear()
        self.rep.consume_mark(out=self.mark_buf, stream=self.cn.stream)
        with torch.cuda.stream(self.cn.stream):
            copy = self.state.clone()
        self.cn.stream.synchronize()
        m = self.mark_buf.cpu().numpy().astype(np.uint64)
        self.snaps.append((int(m[0]), int(m[1]), copy, len(self.cn.rows)))
        return self.snaps[-1]

    def start(self, seed, sizes=(1, 7, 64, 512, 4096)):
        def run():
            rng = np.random.default_rng(seed)
            try:
                while not self.halt.is_set():
                    self.step(int(rng.choice(sizes)))
                    time.sleep(0.0005)
            except Exception as e:        # noqa: BLE001 - reported by stop()
                self.errs.append(e)
        self.halt.clear()
        self.th = threading.Thread(target=run)
        self.th.start()

    def stop(self):
        self.halt.set()
        if self.th:
            self.th.join(120)
            assert not self.th.is_alive()
        self.th = None
        assert not self.errs, self.errs

    def take(self, timeout=60):
        """a snapshot taken by the running thread"""
        n0 = len(self.snaps)
        self.want.set()
        wait_for(lambda: len(self.snaps) > n0 or self.errs, "a snapshot", timeout)
        assert not self.errs, self.errs
        return self.snaps[-1]

    def catch_up(self, timeout=120):
        """(thread stopped) consume until nothing is left and the cursor is the replica's commit offset"""
        t_end = time.time() + timeout
        while True:
            k, st = self.step(MAXN)
            if k == 0 and st.cursor == self.rep.offsets()["commit"]:
                return st
            assert time.time() < t_end, (st, self.rep.offsets())

    def value(self):
        # (the stream only: a device-wide synchronise would wait for the resident replica kernels)
        self.cn.stream.synchronize()
        v = int(self.state.cpu()[0]) & M64
        assert v == fold_host(self.s0, self.cn.rows), "the device fold differs from the host fold of the same rows"
        return v


def warm_fold(fold):
    """load the fold's kernels before replica kernels are resident (a kernel loaded lazily waits for them), with the
    packed layout's lengths (offsets[1:] - offsets[:-1]) as well"""
    import torch
    st = torch.zeros(1, dtype=torch.int64, device=fold.dev)
    z = torch.zeros(MAXN + 1, dtype=torch.int64, device=fold.dev)
    for k in (1, 2, 3, 4, 5, 64, MAXN):
        fold.apply(st, k, z, z.to(torch.uint8), z.to(torch.int16), z, z.to(torch.int16))
        fold.apply(st, k, z, z.to(torch.uint8), z.to(torch.int16), z, z[1:k + 1] - z[:k])
    torch.cuda.synchronize(fold.dev)


# ---- a group that loses a follower -------------------------------------------------------------------------------------
def region_bytes(rep, off, n):
    """bytes [off, off + n) of a replica's HBM region, read through the region pointer its peer handle carries here"""
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


def peer_state(rep, L):
    """everything an adjustment could write on a peer: control block, log header, offset index, entries, offsets and
    consume status"""
    raw = [region_bytes(rep, o, k) for o, k in ((0, 4096), (65536, 64), (INDEX_OFF, 4 * idx_cap(L)))]
    return raw, rep.image(), rep.offsets(), tuple(rep.consume_status())


def same_state(a, b):
    for x, y in zip(a[0], b[0]):
        d = np.nonzero(x != y)[0]
        assert len(d) == 0, f"region bytes differ from +{int(d[0])}"
    assert np.array_equal(a[1], b[1]) and a[2:] == b[2:], "the peer's log, offsets or consume status changed"


class Group:
    """n replicas (0 the leader) that prune on the device, each applying in GPU memory from its own thread"""

    def __init__(self, eng, n, L, layout, lens):
        self.eng, self.n, self.L, self.layout, self.lens = eng, n, L, layout, lens
        self.lib = eng.lib()
        self.devs = devices_for(eng, n)
        self.reps = EU.connected([E.Replica(self.devs[i], i, n, 0, 1, L, E.RING_HOST_MAPPED, 1 << 14, 1 << 22,
                                            MODES["index_earlyack"] | ANY | (E.F_AUTOPRUNE if i == 0 else 0), 4)
                                  for i in range(n)])
        self.folds = {d: Fold(d) for d in set(self.devs)}
        for f in self.folds.values():
            warm_fold(f)
        self.app = {i: Applier(r, layout, self.folds[r.device], lens=lens) for i, r in enumerate(self.reps)}
        self.live = set(range(n))
        self.running = set()
        self.requests = []
        self.rid = 1

    @property
    def lead(self):
        return self.reps[0]

    def launch(self, idxs=None):
        idxs = sorted(self.live if idxs is None else idxs)
        EU.launch_each(self.eng, [self.reps[i] for i in idxs])
        self.running |= set(idxs)

    def stop(self):
        if self.running:
            EU.stop_each(self.eng, [self.reps[i] for i in sorted(self.running)])
        self.running = set()

    def prologue(self):
        """the CONFIG entry a leader starts its term with (idx 1)"""
        self.lead.wait_committed(self.lead.submit(O.CONFIG, 0, 0, O.cid_image(self.n)), 60_000_000)

    def drop(self, k, r):
        """(every replica stopped) replica r in slot k goes away: disconnected on every live replica, then freed"""
        for i in self.live - {k}:
            E._ck(self.lib.apus_replica_disconnect(self.reps[i].h, k), "apus_replica_disconnect")
        r.close()

    def traffic(self, nbytes, seed, max_len=1500):
        """ragged SENDs of nbytes log bytes or more, committed"""
        part = []
        for typ, clt, _, pl in S.ragged_stream(max(8, int(nbytes / (64 + max_len / 2))), max_len, conns=1, seed=seed):
            if typ == S.SEND:
                part.append((S.SEND, 1, self.rid, pl))
                self.rid += 1
        if not self.requests:
            part = [(S.CONNECT, 1, 0, b"")] + part
        assert len(part) <= 1 << 14, "one part must fit the submission ring"
        self.requests += part
        t = EU.submit_all(self.lead, part)
        self.lead.wait_committed(t, 120_000_000)
        return t

    def lose(self, k):
        """follower k is gone for good: every replica stops, every other disconnects it, its region is freed"""
        self.stop()
        self.app[k].stop()
        self.live.discard(k)
        self.drop(k, self.reps[k])
        del self.app[k]

    def fresh(self, k, flags=ANY):
        """a new replica in slot k, connected both ways to every live replica (every replica stopped)"""
        r = E.Replica(self.devs[k], k, self.n, 0, 1, self.L, E.RING_HOST_MAPPED, 1 << 14, 1 << 22,
                      MODES["index_earlyack"] | flags, 4)
        for i in self.live:
            r.connect(i, self.reps[i].export())
            self.reps[i].connect(k, r.export())
        return r

    def adjust(self, k):
        got = C.c_uint64()
        E._ck(self.lib.apus_ctl_adjust_follower(self.lead.h, k, sid(1, 1, 0), C.byref(got)), "apus_ctl_adjust_follower")
        return int(got.value)

    def join(self, k, r, mark):
        """seed r at mark = (cursor, next idx), adjust it and make it follow; checks the resend and the record"""
        r.consume_seed(mark[0], mark[1])
        assert tuple(r.consume_status())[:2] == mark
        lo = self.lead.offsets()
        resent = self.adjust(k)
        assert resent == (lo["end"] - lo["head"]) % self.L, (resent, lo)
        E._ck(self.lib.apus_replica_set_role(r.h, 0, 1), "apus_replica_set_role")
        assert self.lead.remote_apply_offsets()[k] == mark[0], "the leader does not count the seed as the apply offset"
        ro = r.offsets()
        assert (ro["head"], ro["commit"], ro["end"]) == (lo["head"], lo["commit"], lo["end"]), (ro, lo)
        a, b = lo["head"], lo["end"]
        if a != b:
            live = [(a, b)] if a < b else [(a, self.L), (0, b)]
            for x, y in live:
                assert np.array_equal(r.image(x, y), self.lead.image(x, y)), f"live log [{x}, {y}) differs"
        self.reps[k] = r
        self.live.add(k)

    def head_idx(self):
        o = self.lead.offsets()
        return RE.u64(self.lead.image(o["head"], o["head"] + 8), 0)

    def settle_all(self):
        """(traffic over, replicas running) every applier catches up to its commit, every state is the same"""
        for a in self.app.values():
            a.stop()
        wait_for(lambda: all(self.reps[i].offsets()["commit"] == self.lead.offsets()["commit"] for i in self.running),
                 "followers to follow the commit", 30)
        vals = {}
        for i, a in self.app.items():
            a.catch_up()
            vals[i] = a.value()
        return vals

    def close(self):
        for a in self.app.values():
            a.halt.set()
        for a in self.app.values():
            if a.th:
                a.th.join(60)
        try:
            self.stop()
        finally:
            for i in self.live:
                self.reps[i].close()


# ---- the worker side ---------------------------------------------------------------------------------------------
def case_replace(eng, orc, n, layout, source, hold):
    L = 1 << 20
    lost = n - 1
    g = Group(eng, n, L, layout, lens=())
    try:
        g.launch()
        g.prologue()
        for i, a in g.app.items():
            a.start(10 + i)
        g.traffic(0.6 * L, 1)
        lost_held = g.reps[lost].stats()["entries_acked"]
        assert lost_held > 0
        g.lose(lost)
        g.launch()
        for lap in range(8):
            g.traffic(0.5 * L, 100 + lap)
            if g.head_idx() > lost_held + 1:
                break
        hidx = g.head_idx()
        assert hidx > lost_held + 1, (hidx, lost_held)
        print(f"lost {lost} (held {lost_held}); head idx now {hidx}", flush=True)
        # mark and copy while the group runs.  With requests in flight the head may pass the mark before the leader
        # stops (the adjustment says APUS_RETRY, and the replacement goes); a mark taken once they are committed holds
        for attempt in range(2):
            th = threading.Thread(target=g.traffic, args=(0.1 * L, 900)) if attempt == 0 else None
            if th:
                th.start()
            cur, nidx, snap, nrows = g.app[source].take()
            if th:
                th.join(120)
            assert nidx >= hidx, (nidx, hidx)
            g.stop()
            r = g.fresh(lost)
            if attempt == 0:
                with pytest.raises(E.ApusError, match="shares no entry"):      # a fresh replica without a seed
                    g.adjust(lost)
            try:
                g.join(lost, r, (cur, nidx))
                break
            except BlockingIOError as e:
                assert attempt == 0 and "behind my head" in str(e), e
                print(f"mark {cur}/{nidx} taken with requests in flight: {e}", flush=True)
                g.drop(lost, r)
                g.launch()
        print(f"joined at {cur}/{nidx}", flush=True)
        src_rows = g.app[source].cn.rows
        a = Applier(r, layout, g.folds[r.device], state=snap)
        g.app[lost] = a
        g.launch()
        if hold:
            # the replacement's consumer held back at the seed: more than a lap of requests cannot all commit, and the
            # leader's head never passes the seed
            h0 = g.lead.offsets()["head"]
            moved, last = 0, h0
            t0 = g.lead.committed()
            th = threading.Thread(target=g.traffic, args=(1.3 * L, 950))
            th.start()
            still = time.time()
            prev = g.lead.committed()
            while time.time() - still < 1.0:
                h = g.lead.offsets()["head"]
                moved += (h - last) % L
                last = h
                c_ = g.lead.committed()
                if c_ != prev:
                    prev, still = c_, time.time()
                time.sleep(0.002)
            assert moved <= (cur - h0) % L, f"the head moved {moved} B past {h0}, the seed is {(cur - h0) % L} B ahead"
            assert prev > t0 and th.is_alive(), "the held consumer did not hold the leader back"
            print(f"held: head moved {moved} B, commits {t0} -> {prev}", flush=True)
            a.start(77)
            th.join(300)
            assert not th.is_alive()
        else:
            a.start(77)
        for i in g.app:
            if i != lost and not g.app[i].th:
                g.app[i].start(40 + i)
        g.traffic(0.8 * L, 2)
        vals = g.settle_all()
        assert len(set(vals.values())) == 1, vals
        check_rows(g.app[0].cn.rows, [(t, c_ & 0xFFFF, r_, bytes(p)) for t, c_, r_, p in g.requests], first_idx=2)
        rows = a.cn.rows
        assert rows and rows[0][0] >= nidx and (nrows == 0 or src_rows[nrows - 1][0] < nidx)
        assert rows == g.app[source].cn.rows[nrows:], "the replacement's rows are not the source's from the mark on"
        st = r.consume_status()
        assert st.error == 0 and st.cursor == r.offsets()["commit"] == g.lead.offsets()["commit"]
        if n == 3:
            # a real member: with the other follower stopped and disconnected, leader and replacement alone commit
            other = 1
            g.stop()
            for i in (0, lost):
                E._ck(g.lib.apus_replica_disconnect(g.reps[i].h, other), "apus_replica_disconnect")
            g.app[other].stop()
            g.launch([0, lost])
            for i in (0, lost):
                g.app[i].start(60 + i)
            g.traffic(0.3 * L, 3)
            del g.app[other]
            vals = g.settle_all()
            assert vals[0] == vals[lost], vals
        print(f"n={n} {layout} from {source}: seed {cur}/{nidx}, head idx {hidx}, lost held {lost_held}, "
              f"{len(rows)} rows on the replacement")
    finally:
        g.close()


class Driver:
    """ring_edges.fill_to's driver on the running group: one committed SEND per call, the appliers caught up after it"""

    def __init__(self, g):
        self.g, self.L, self.ends_at_len = g, g.L, False

    def end(self):
        return self.g.lead.offsets()["end"]

    def last_ended_at_len(self):
        return self.ends_at_len

    def send(self, stride):
        e = self.end()
        self.g.requests.append((S.SEND, 1, self.g.rid, b"x" * (stride - RE.HDR)))
        t = self.g.lead.submit(S.SEND, 1, self.g.rid, b"x" * (stride - RE.HDR))
        self.g.rid += 1
        self.g.lead.wait_committed(t, 60_000_000)
        self.ends_at_len = RE.landing(self.L, e, stride, True)[0] + stride == self.L
        for a in self.g.app.values():
            a.catch_up()


def case_ring_end(eng, orc):
    n, L = 5, 1 << 18
    g = Group(eng, n, L, "strided", lens=())
    try:
        g.lose(3)
        g.lose(4)
        g.launch()
        g.prologue()
        d = Driver(g)
        for a in g.app.values():
            a.catch_up()
        while (L - 300 - d.end()) % L > 32 << 10:
            d.send(RE.HDR + 1500)
        RE.fill_to(d, L - 300, RE.HDR + 1500)          # every filler fits a row
        print("end at", d.end(), flush=True)
        # the next entry (a HEAD of the pruning rule may come first) wraps to 0 and leaves a gap behind the last entry
        stride = RE.edge_stride("send")
        g.requests.append((S.SEND, 1, g.rid, b"y" * RE.SEND_LEN))
        g.lead.wait_committed(g.lead.submit(S.SEND, 1, g.rid, b"y" * RE.SEND_LEN), 60_000_000)
        g.rid += 1
        o = g.lead.offsets()
        ents = O.walk_entries(g.lead.image(), o["head"], o["end"], L)
        k0 = [q for q, (off, _) in enumerate(ents) if off == 0]
        assert k0 and k0[0] > 0, (o, ents[-4:])
        gap = ents[k0[0] - 1][0] + ents[k0[0] - 1][1]
        img = g.lead.image()
        w = RE.u64(img, 0)
        assert gap < L and ents[k0[0]][1] == stride, (gap, ents[k0[0]])
        # mark A: the leader's consumer stops right behind the last entry before the gap
        a0 = g.app[0]
        nx = a0.rep.consume_status().next_idx
        if w > nx:
            a0.step(w - nx)
        st = a0.rep.consume_status()
        assert (st.cursor, st.next_idx) == (gap, w), (st, gap, w)
        mark_a = a0.snapshot()
        # mark B: follower 1's consumer just after the wrap, behind the entry at 0; one more entry follows it
        g.app[1].catch_up()
        mark_b = g.app[1].snapshot()
        assert mark_b[:2] == (stride, w + 1), (mark_b[:2], stride, w)
        d.send(RE.HDR + 10)
        g.stop()
        # both replacements at once, into the two free slots
        for slot, (cur, nidx, snap, _) in ((3, mark_a), (4, mark_b)):
            r = g.fresh(slot)
            g.join(slot, r, (cur, nidx))
            g.app[slot] = Applier(r, "strided", g.folds[r.device], state=snap)
        g.launch()
        for i, a in g.app.items():
            a.start(20 + i)
        for q in range(3):
            g.traffic(0.3 * L, 500 + q, max_len=600)
        vals = g.settle_all()
        assert len(set(vals.values())) == 1, vals
        for slot, src, mark in ((3, 0, mark_a), (4, 1, mark_b)):
            assert g.app[slot].cn.rows == g.app[src].cn.rows[mark[3]:], f"replacement {slot}: its rows differ"
        check_rows(g.app[0].cn.rows, [(t, c_ & 0xFFFF, r_, bytes(p)) for t, c_, r_, p in g.requests], first_idx=2)
        print(f"marks at the ring's end accepted: A {mark_a[:2]} (gap), B {mark_b[:2]}")
    finally:
        g.close()


def refused(fn, match, rc=E.ApusError):
    with pytest.raises(rc, match=match):
        fn()


def case_refusals(eng, orc):
    import torch
    n, L = 3, 1 << 20
    g = Group(eng, n, L, "strided", lens=())
    extra = []
    try:
        lib = g.lib
        # seed refusals, each leaving the replica as it was
        plain = E.Replica(g.devs[1], 1, n, 0, 1, L, flags=MODES["index_earlyack"] | E.F_DEVICE_APPLY)
        extra.append(plain)
        for r, match in ((plain, "APUS_F_APPLY_ANY_ROLE"), (g.lead, "a leader")):
            before = peer_state(r, L)
            refused(lambda: r.consume_seed(0, 1), match)
            same_state(before, peer_state(r, L))
        g.launch()
        g.prologue()
        for i, a in g.app.items():
            a.start(10 + i)
        g.traffic(0.3 * L, 1)
        old = g.app[0].take()                           # a mark the head will pass
        g.traffic(0.2 * L, 2)
        refused(lambda: g.reps[1].consume_seed(0, 1), "stop the kernel first")
        g.lose(2)
        # replica 1 quiet (kernel stopped, its consumer's thread ended), so that only the refused seed could write
        g.app[1].stop()
        before = peer_state(g.reps[1], L)
        refused(lambda: g.reps[1].consume_seed(0, 1), "holds entries")
        same_state(before, peer_state(g.reps[1], L))
        g.app[1].start(21)
        g.launch()
        for lap in range(8):
            g.traffic(0.5 * L, 100 + lap)
            if g.head_idx() > old[1]:
                break
        assert g.head_idx() > old[1]
        for a in g.app.values():
            a.stop()
        g.stop()
        # a fresh replica after a consume call (nothing delivered), and one in flight
        r = g.fresh(2)
        extra.append(r)
        r.consume_device(4, 16)
        torch.cuda.synchronize(r.device)
        before = peer_state(r, L)
        refused(lambda: r.consume_seed(0, 1), "consume work has been enqueued")
        same_state(before, peer_state(r, L))
        extra.remove(r)
        g.drop(2, r)
        r = g.fresh(2)
        EU.launch_each(eng, [r])
        try:
            refused(lambda: r.consume_seed(0, 1), "stop the kernel first")
        finally:
            EU.stop_each(eng, [r])
            g.drop(2, r)
        # adjustments: the leader's log as it stands, a seed per attempt on a fresh replica
        lo, lc = g.lead.offsets(), g.lead.stats()
        img = g.lead.image()
        ents = O.walk_entries(img, lo["head"], lo["end"], L)
        committed = lc["entries_published"]
        mid_off, _ = ents[len(ents) // 2]
        mid_idx = RE.u64(img, mid_off)
        cases = [((old[0], old[1]), E.APUS_RETRY, "behind my head"),
                 ((lo["commit"], committed + 2), E.APUS_ERROR, "past my commit"),
                 (((mid_off + 8) % L, mid_idx), E.APUS_ERROR, "no consumer of my log stands there"),
                 ((mid_off, mid_idx + 1), E.APUS_ERROR, "no consumer of my log stands there")]
        lead_ctl = region_bytes(g.lead, 0, 4096)
        for mark, rc, match in cases:
            r = g.fresh(2)
            try:
                r.consume_seed(*mark)
                before = peer_state(r, L)
                got = C.c_uint64()
                assert lib.apus_ctl_adjust_follower(g.lead.h, 2, sid(1, 1, 0), C.byref(got)) == rc, mark
                assert match in lib.apus_last_error().decode(), (mark, lib.apus_last_error())
                same_state(before, peer_state(r, L))
                assert np.array_equal(lead_ctl, region_bytes(g.lead, 0, 4096)), "the leader's control block changed"
            finally:
                g.drop(2, r)
        # a misaligned mark: refused with nothing enqueued
        buf = torch.zeros(4, dtype=torch.int64, device=torch.device("cuda", g.lead.device))
        assert lib.apus_consume_mark(g.lead.h, buf.data_ptr() + 8, None) == E.APUS_ERROR
        assert "misaligned" in lib.apus_last_error().decode()
        refused(lambda: g.lead.consume_mark(out=buf[1:3]), "misaligned")
        torch.cuda.synchronize(g.lead.device)
        assert int(buf.abs().sum().cpu()) == 0
        # and the accepted one, at the mark the leader's consumer stands at now
        a0 = g.app[0]
        a0.catch_up()
        cur, nidx, _, _ = a0.snapshot()
        r = g.fresh(2)
        g.join(2, r, (cur, nidx))
        print("refusals ok; accepted", (cur, nidx))
    finally:
        for r in extra:
            r.close()
        g.close()


if __name__ == "__main__":
    EU.worker_main(globals())
