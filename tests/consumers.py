"""Device consumers for the GPU tests (APUS_F_DEVICE_APPLY, apus_consume_device / apus_consume_device_packed): groups
whose replicas consume on the device, consumers that keep every row they received and every cursor they reported, and
the checks of those rows against the request stream and the CPU oracle's log.  Importing this module starts no CUDA
context: torch is loaded where it is used."""
import ctypes as C
import os
import time

import numpy as np

import autoprune_replay as AR
import engine_util as EU
import orc as O
from apus_b200 import engine as E

ANY = E.F_DEVICE_APPLY | E.F_APPLY_ANY_ROLE
SENTINEL = 0xA5


def new_stream(device):
    """A CUDA stream of its own, created with the runtime rather than taken from torch's pool.  The pool creates dozens
    of streams at once, and those wrap around the 32 hardware queues onto the replicas' own streams.  A consumer stream
    that shares a queue with the leader's streams makes them wait behind its pending consume waits (DESIGN.md s2)."""
    import torch
    try:
        rt = C.CDLL("libcudart.so.12")
    except OSError:
        import nvidia.cuda_runtime as ncr
        rt = C.CDLL(os.path.join(list(ncr.__path__)[0], "lib", "libcudart.so.12"))
    s = C.c_void_p()
    assert rt.cudaSetDevice(device) == 0, f"cudaSetDevice({device})"
    assert rt.cudaStreamCreateWithFlags(C.byref(s), 1) == 0, "cudaStreamCreateWithFlags"   # cudaStreamNonBlocking
    return torch.cuda.ExternalStream(s.value, device=torch.device("cuda", device))


def consumer_group(eng, n, L, mode=EU.MODES["index_earlyack"], leader_flags=0, ring_mode=None, ring_slots=0,
                   ring_bytes=0, ctas=4, follower_flags=None):
    """n connected replicas, replica 0 the leader; every follower consumes on the device (APUS_F_DEVICE_APPLY) unless
    `follower_flags` (one entry per follower) says otherwise"""
    devs = EU.devices_for(eng, n)
    ring_mode = E.RING_HOST_MAPPED if ring_mode is None else ring_mode
    ff = [E.F_DEVICE_APPLY] * (n - 1) if follower_flags is None else follower_flags
    return EU.connected([E.Replica(devs[i], i, n, 0, 1, L, ring_mode, ring_slots, ring_bytes,
                                   (mode | leader_flags) if i == 0 else (mode | ff[i - 1]), ctas) for i in range(n)])


def close_all(eng, reps):
    try:
        EU.stop_each(eng, reps)
    finally:
        for r in reps:
            r.close()


class _ConsumerBase:
    """What a replica's device consumer keeps in either layout: its own stream, the rows received, the calls made and
    the cursors reported"""

    def __init__(self, rep, stream=None):
        import torch
        self.rep = rep
        self.stream = torch.cuda.Stream(device=rep.device) if stream is None else stream
        self.rows = []            # (idx, type, conn, req_id, cmd bytes)
        self.calls = 0
        # cursors as absolute positions (ring bytes consumed), each with the time its call was made: the cursor did
        # not exist before that, so a HEAD read earlier cannot legitimately carry it
        self.cur, self.at, self.reports = 0, 0, []

    def _status(self, t_call):
        """after a call made at t_call: its status, which must carry no error, and the cursor it reported"""
        self.calls += 1
        st = self.rep.consume_status()
        assert st.error == 0, st
        adv = (st.cursor - self.cur) % self.rep.log_len
        if adv:
            self.cur, self.at = st.cursor, self.at + adv
            self.reports.append((self.at, t_call))
        return st


class Consumer(_ConsumerBase):
    """One replica's device consumer: consume_device into reused tensors on its own stream (one of torch's, or
    `stream`), rows copied to the host only to be checked"""

    def __init__(self, rep, stride, cap, stream=None):
        super().__init__(rep, stream)
        self.stride, self.cap = stride, cap
        self.out = None

    def step(self, max_n, stride=None):
        stride = self.stride if stride is None else stride
        if self.out is None or self.out[5].shape[1] != stride or self.out[0].shape[0] != max_n:
            self.out = None
        t_call = time.perf_counter()
        self.out = self.rep.consume_device(max_n, stride, out=self.out, stream=self.stream)
        self.stream.synchronize()
        k = int(self.out[6].cpu()[0])
        idx, ty, co, rq, ln, pl = (t[:k].cpu().numpy() for t in self.out[:6])
        for q in range(k):
            self.rows.append((int(idx[q]), int(ty[q]), int(co[q]) & 0xFFFF, int(rq[q]), pl[q, :int(ln[q]) & 0xFFFF].tobytes()))
        return k, self._status(t_call)


class PackedConsumer(_ConsumerBase):
    """One replica's packed device consumer: consume_device_packed into slices of reused buffers on its own stream,
    with a sentinel in the output before every call.  values_cap is chosen from the lengths of the rows still to come
    (`lens`): on a cumulative boundary, one byte short of it or one byte past it; after a stop on the first row, the
    capacity need_stride asks for.  Rows are copied to the host only to be checked."""

    def __init__(self, rep, lens, max_n_cap=4096, cap_max=1 << 22, seed=0):
        import torch
        super().__init__(rep)
        self.lens = np.asarray(lens, dtype=np.int64)
        dev = torch.device("cuda", rep.device)
        with torch.cuda.stream(self.stream):
            self.buf = (torch.empty(max_n_cap, dtype=torch.int64, device=dev),
                        torch.empty(max_n_cap, dtype=torch.uint8, device=dev),
                        torch.empty(max_n_cap, dtype=torch.int16, device=dev),
                        torch.empty(max_n_cap, dtype=torch.int64, device=dev),
                        torch.empty(max_n_cap + 1, dtype=torch.int64, device=dev),
                        torch.empty(cap_max, dtype=torch.uint8, device=dev),
                        torch.empty(1, dtype=torch.int32, device=dev))
        self.cap_max = cap_max
        self.rng = np.random.default_rng(seed)
        self.need = 0
        self.exact = None            # set: every row still to come is committed, and no NOOP / CONFIG / HEAD is ahead

    def pick_cap(self, max_n):
        nxt = self.lens[len(self.rows):len(self.rows) + max_n]
        if self.need:
            return self.need
        if len(nxt) == 0:
            return int(self.rng.integers(0, 70000))
        cum = np.cumsum(nxt)
        r = int(self.rng.integers(0, len(cum)))
        return int(min(self.cap_max, max(0, cum[r] + int(self.rng.integers(-1, 2)))))

    def step(self, max_n, cap=None):
        import torch
        cap = self.pick_cap(max_n) if cap is None else cap
        idx, ty, co, rq, of, va, cn = self.buf
        out = (idx[:max_n], ty[:max_n], co[:max_n], rq[:max_n], of[:max_n + 1], va[:cap], cn)
        with_exact = self.exact is not None and self.exact()
        with torch.cuda.stream(self.stream):
            of.fill_(-7)
            va[:min(cap + 1, self.cap_max)].fill_(SENTINEL)
        t_call = time.perf_counter()
        self.rep.consume_device_packed(max_n, cap, out=out, stream=self.stream)
        self.stream.synchronize()
        k = int(cn.cpu()[0])
        offs = of[:max_n + 1].cpu().numpy()
        vals = va[:min(cap + 1, self.cap_max)].cpu().numpy()
        assert offs[0] == 0 and np.all(np.diff(offs[:k + 1]) >= 0), offs[:k + 1]
        assert np.all(offs[k + 1:] == -7), "offsets past count were written"
        assert offs[k] <= cap, (k, offs[k], cap)
        assert np.all(vals[offs[k]:] == SENTINEL), "bytes past offsets[count] were written"
        ii, tt, cc, rr = (x[:k].cpu().numpy() for x in (idx, ty, co, rq))
        for q in range(k):
            self.rows.append((int(ii[q]), int(tt[q]), int(cc[q]) & 0xFFFF, int(rr[q]), vals[offs[q]:offs[q + 1]].tobytes()))
        st = self._status(t_call)
        nxt = self.lens[len(self.rows) - k:len(self.rows) - k + max_n]
        if with_exact and len(nxt):
            cum = np.cumsum(nxt)
            want = int(np.searchsorted(cum, cap, side="right"))
            assert k == min(max_n, len(nxt), want), (k, max_n, len(nxt), want, cap)
            if want == 0:
                assert st.need_stride == nxt[0], (st.need_stride, nxt[0])
        if k:
            assert st.need_stride == 0, st
        self.need = st.need_stride
        return k, st


def check_rows(rows, stream, first_idx=None):
    """rows are the stream's requests, in order, with strictly increasing idx; none missing, none duplicated"""
    assert len(rows) == len(stream), (len(rows), len(stream))
    for q, ((i, ty, co, rq, pl), (sty, sco, srq, spl)) in enumerate(zip(rows, stream)):
        assert (ty, co, rq, pl) == (sty, sco, srq, bytes(spl)), (q, rows[q][:4], (sty, sco, srq, len(spl)))
        if q:
            assert i > rows[q - 1][0], (q, i, rows[q - 1][0])
    if first_idx is not None and rows:
        assert rows[0][0] == first_idx, (rows[0][0], first_idx)


def oracle_rows(c, i):
    """the CSM-like entries of replica i of the oracle cluster, as rows (the log must not have lapped)"""
    img, end, L = c.image(i), c.offsets(i)["end"], c.len
    out = []
    for off, _ in O.walk_entries(img, 0, end, L):
        ty = int(img[off + 26])
        if ty in (O.NOOP, O.CONFIG, O.HEAD):
            continue
        ln = int(img[off + 48]) | int(img[off + 49]) << 8
        out.append((int(img[off:off + 8].view(np.uint64)[0]), ty, int(img[off + 24]) | int(img[off + 25]) << 8,
                    int(img[off + 16:off + 24].view(np.uint64)[0]), img[off + 50:off + 50 + ln].tobytes()))
    return out


def drain(cons, done, maxns, rng, pause=0.0):
    """consume until done() says everything is committed and the consumer has caught up"""
    while True:
        k, st = cons.step(int(rng.choice(maxns)))
        if k == 0 and done(st):
            return
        if pause:
            time.sleep(pause)


def catch_up(cn, timeout=60):
    """consume until nothing is left and the cursor is the replica's commit offset"""
    t_end = time.time() + timeout
    while True:
        k, st = cn.step(512)
        if k == 0 and st.cursor == cn.rep.offsets()["commit"]:
            return st
        assert time.time() < t_end, (st, cn.rep.offsets())


def wait_forwarded_all(reps, timeout=30):
    """every replica of `reps` has forwarded its consumers' cursor: its apply offset is its commit offset"""
    t = time.time()
    while True:
        offs = [r.offsets() for r in reps]
        if all(o["apply"] == o["commit"] for o in offs):
            return
        assert time.time() - t < timeout, offs
        time.sleep(0.002)


def wait_forwarded(reps, timeout=30):
    """every follower's kernel (reps[1:]) has forwarded its consumers' cursor"""
    wait_forwarded_all(reps[1:], timeout)


def idx_cap(L):
    """the offset index's size in words for an L-byte log"""
    cap = 1024
    while cap * 64 < L:
        cap <<= 1
    return cap


def heads_against_reports(L, segs, reports, lagging, hits):
    """on_head for Replay.launch (the rule of autoprune_replay.replay_recordings, with the device consumers' cursors among
    the reports): a HEAD may carry no head past any follower's last report made before the HEAD was first read, and the
    head it carries is one of those reports, or the tail once every follower had reported the HEAD's own position.
    `segs`: the host recorder's reads; `reports`: {follower: [(absolute offset, time)]}; `hits` counts the HEADs that
    carry a cursor of the `lagging` consumer."""
    starts = np.array([s for s, _, _ in segs], dtype=np.int64)
    stops = np.array([s + len(b) for s, b, _ in segs], dtype=np.int64)
    times = np.array([t for _, _, t in segs], dtype=np.float64)
    reps = {j: [(0, float("-inf"))] + sorted(rs, key=lambda x: x[1]) for j, rs in reports.items()}

    def on_head(e, at, prev_at):
        seen = (starts <= at) & (stops >= at + e.stride)
        if not seen.any():
            return "the host recorder never read it"
        t = times[seen].min()
        v = at - AR.dist(e.value, e.off, L)                      # the head it carries, as an absolute position
        legal, last = set(), {}
        for j, rs in reps.items():
            before = [a for a, tr in rs if tr < t]
            last[j] = max(before)
            legal.update(before)
            if v > last[j]:
                return (f"head {e.value} (absolute {v}) is past follower {j}'s last report {last[j]} before the HEAD "
                        f"was first read")
        if v in {a for a, _ in reps[lagging]}:
            hits.append(v)
        if v in legal or (v == prev_at and all(x == at for x in last.values())):
            return None
        return f"head {e.value} (absolute {v}) is no report made before the HEAD was first read (last reports {last})"
    return on_head
