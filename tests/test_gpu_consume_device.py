"""Committed entries consumed straight into GPU memory on followers (APUS_F_DEVICE_APPLY, apus_consume_device): every
row a consumer receives is checked against the request stream and, where the log does not lap, against the CPU
oracle's log; the consumers' cursor is what the leader's pruning rule reads, so a multi-lap launch fails here if the
leader overwrites entries a consumer has not read.  Marked gpu."""
import threading
import time
import types as T

import numpy as np
import pytest

import autoprune_replay as AR
import engine_util as EU
import orc as O
import streams as S
from test_gpu_device_submit import tensors
from test_gpu_parity import MODES, devices_for
from test_gpu_prune_in_launch import _submit_all

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

FOREVER = EU.FOREVER
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    import apus_b200
    if apus_b200.lib().apus_device_count() < 1:
        pytest.fail("no CUDA device visible on a gpu-marked test")
    import torch
    for d in range(torch.cuda.device_count()):
        # load torch's kernels before the replica kernels are resident (a lazy load may wait for running kernels)
        x = torch.zeros(16, dtype=torch.uint8, device=torch.device("cuda", d))
        x.fill_(1)
        x.clone()
        torch.cuda.synchronize(d)
    return apus_b200


@pytest.fixture(scope="module", autouse=True)
def release_torch_memory():
    yield
    import gc
    import torch
    gc.collect()
    if torch.cuda.is_initialized():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def consumer_group(eng, n, L, mode=MODES["index_earlyack"], leader_flags=0, ring_mode=None, ring_slots=0, ring_bytes=0,
                   ctas=4, follower_flags=None):
    """n connected replicas, replica 0 the leader; every follower consumes on the device (APUS_F_DEVICE_APPLY) unless
    `follower_flags` (one entry per follower) says otherwise"""
    from apus_b200 import engine as E
    devs = devices_for(eng, n)
    ring_mode = E.RING_HOST_MAPPED if ring_mode is None else ring_mode
    ff = [E.F_DEVICE_APPLY] * (n - 1) if follower_flags is None else follower_flags
    reps = [E.Replica(devs[i], i, n, 0, 1, L, ring_mode, ring_slots, ring_bytes,
                      (mode | leader_flags) if i == 0 else (mode | ff[i - 1]), ctas) for i in range(n)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    return reps


def close_all(eng, reps):
    try:
        EU.stop_each(eng, reps)
    finally:
        for r in reps:
            r.close()


class _ConsumerBase:
    """What a follower's device consumer keeps in either layout: its own stream, the rows received, the calls made and
    the cursors reported"""

    def __init__(self, rep):
        import torch
        self.rep = rep
        self.stream = torch.cuda.Stream(device=rep.device)
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
    """One follower's device consumer: consume_device into reused tensors on its own stream, rows copied to the host
    only to be checked"""

    def __init__(self, rep, stride, cap):
        super().__init__(rep)
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
    """One follower's packed device consumer: consume_device_packed into slices of reused buffers on its own stream,
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
        assert offs[k] <= cap
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
        assert rows[0][0] == first_idx


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


def wait_forwarded(reps, timeout=30):
    """every follower's kernel has forwarded its consumers' cursor: its apply offset is its commit offset"""
    t = time.time()
    while True:
        offs = [r.offsets() for r in reps[1:]]
        if all(o["apply"] == o["commit"] for o in offs):
            return
        assert time.time() - t < timeout, offs
        time.sleep(0.002)


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("n", [3, 5])
def test_ragged_stream_rows_match_oracle(eng, orc, n, mode):
    """ragged_stream (0..1500 B, CONNECT / CLOSE churn), consumed with max_n from 1 up while the kernels run: every row
    equals the stream and the oracle's log; the logs stay byte-equal to the oracle's; the final cursor is every
    follower's commit offset, and the follower kernels forward it as their apply offset"""
    L = 1 << 22
    stream = S.ragged_stream(2500, 1500, conns=4, seed=500 + n, close_every=40)
    reps = consumer_group(eng, n, L, MODES[mode])
    rng = np.random.default_rng(n * 31 + len(mode))
    try:
        cons = [Consumer(r, 1500, 4096) for r in reps[1:]]
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = _submit_all(lead, stream)
        last_idx = len(stream) + 1
        for c in cons:
            drain(c, lambda st: st.next_idx == last_idx + 1, [1, 2, 7, 64, 333, 4096], rng)
        lead.wait_committed(t)
        wait_forwarded(reps)
        EU.stop_each(eng, reps)
        c = EU.oracle_cluster(orc, n, L, stream)
        EU.compare_group_to_oracle(T.SimpleNamespace(n=n, replicas=reps, leader_idx=0), c, exact=True)
        for j, cn in enumerate(cons, 1):
            check_rows(cn.rows, stream, first_idx=2)
            assert cn.rows == oracle_rows(c, j)
            st = reps[j].consume_status()
            assert st.cursor == reps[j].offsets()["commit"] == c.offsets(j)["commit"]
            assert st.next_idx == last_idx + 1 and st.error == 0
        c.close()
    finally:
        close_all(eng, reps)


@pytest.mark.parametrize("express", [True, False])
def test_express_traffic(eng, express):
    """Closed-loop requests, one in flight, on a 64 KiB ring with pruning: the log laps about five times and the
    offset index (1024 words) about three, so the index word of a self-certified entry, until the leader's own store
    lands, is one an earlier lap wrote.  The consumers run while the followers verify certificates (express on: counted
    with APUS_F_PROFILE) and find those entries through the index words the followers store themselves."""
    from apus_b200 import engine as E
    n, L, nreq, ln = 3, 1 << 16, 3000, 40
    reps = consumer_group(eng, n, L, leader_flags=E.F_AUTOPRUNE | (0 if express else E.F_NO_EXPRESS),
                          follower_flags=[E.F_DEVICE_APPLY | E.F_PROFILE] * (n - 1))
    try:
        cons = [Consumer(r, 64, 512) for r in reps[1:]]
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        lead.wait_committed(lead.submit(O.CONFIG, 0, 0, O.cid_image(n)))
        stop = threading.Event()
        errs = []

        def run(cn, seed):
            try:
                drain(cn, lambda st: stop.is_set() and st.next_idx == nreq + 2 + lead.stats()["auto_heads"],
                      [1, 3, 16, 512], np.random.default_rng(seed))
            except Exception as e:        # noqa: BLE001 - reported below
                errs.append(e)
        th = [threading.Thread(target=run, args=(cn, 70 + k)) for k, cn in enumerate(cons)]
        for x in th:
            x.start()
        lat = lead.closed_loop(nreq, ln, 9, 1)
        stop.set()
        for x in th:
            x.join(120)
            assert not x.is_alive()
        assert not errs, errs
        assert len(lat) == nreq
        heads = lead.stats()["auto_heads"]
        assert nreq * (64 + ln) >= 4 * L and heads >= 3, heads
        pl = bytes((k * 131 + 7) & 0xFF for k in range(ln))
        want = [(S.SEND, 9, 1 + i, pl) for i in range(nreq)]
        for cn in cons:
            check_rows(cn.rows, want, first_idx=2)
            certs = cn.rep.stats()["phase_ns"][0]             # certificates this follower verified
            assert (certs > 0) if express else (certs == 0), certs
    finally:
        close_all(eng, reps)


def _lap_case(kind, L):
    if kind == "ragged1500":
        return S.ragged_stream(int(6.5 * 1.15 * L / 814) + 1, 1500, conns=3, seed=97, close_every=20), 1500
    return S.sized_stream(int(6.5 * L / 6200) + 1, 3072, 9216, seed=98), 9216


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


@pytest.mark.parametrize("layout", ["strided", "packed"])
@pytest.mark.parametrize("kind,L,ctas", [("ragged1500", 1 << 18, 2), ("sized3k9k", 1 << 15, 4)])
def test_pruning_in_one_launch_replayed(eng, orc, kind, L, ctas, layout):
    """One launch laps a small ring more than six times with APUS_F_AUTOPRUNE.  Followers 2 and 3 consume on the
    device, strided or packed, from host threads, 3 lagging with small max_n and pauses; follower 1's host applies
    through a recorder (APUS_F_HOST_APPLY), which gives the replay the leader's append sequence byte for byte.  Every
    HEAD entry must carry a head no further than any follower's report made before the HEAD was first read -- the
    lagging consumer's cursor among them -- and be one of those reports; the HEADs are replayed into the oracle, every
    recorded read is compared with it, and at the end every byte and offset of every replica.  Every row of every
    consumer equals the stream."""
    from apus_b200 import engine as E
    n = 4
    stream, stride = _lap_case(kind, L)
    requests = [(O.CONFIG, 0, 0, b"")] + stream
    reps = consumer_group(eng, n, L, leader_flags=E.F_AUTOPRUNE, ring_slots=1 << 14, ring_bytes=1 << 17, ctas=ctas,
                          follower_flags=[E.F_HOST_APPLY, E.F_DEVICE_APPLY, E.F_DEVICE_APPLY])
    rec = AR.Recorder(reps[1], 1, L)
    rp = AR.Replay(orc, n, L)
    try:
        if layout == "strided":
            cons = [Consumer(r, stride, 256) for r in reps[2:]]
        else:
            cons = [PackedConsumer(r, [len(p) for *_, p in stream], max_n_cap=256, cap_max=1 << 20, seed=90 + k)
                    for k, r in enumerate(reps[2:])]
        errs, total = [], {}

        def run(cn, lag, seed):
            rng = np.random.default_rng(seed)
            try:
                drain(cn, lambda st: "t" in total and st.next_idx > total["t"] + total["heads"](),
                      [1, 2, 3] if lag else [16, 256], rng, pause=0.002 if lag else 0.0)
            except Exception as e:        # noqa: BLE001 - reported below
                errs.append(e)
        total["heads"] = lambda: reps[0].stats()["auto_heads"]
        th = [threading.Thread(target=run, args=(cn, k == len(cons) - 1, 90 + k)) for k, cn in enumerate(cons)]
        rec.start()
        for x in th:
            x.start()
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = _submit_all(lead, stream)
        deadline = time.time() + 300
        while lead.committed() < t:
            rec.check()
            assert not errs, errs
            assert time.time() < deadline, f"committed {lead.committed()} of {t}; leader {lead.offsets()}"
            time.sleep(0.005)
        total["t"] = t
        final = lead.offsets()["end"]
        rec.finish(final)
        for x in th:
            x.join(300)
            assert not x.is_alive()
        assert not errs, errs
        wait_forwarded(reps)
        EU.stop_each(eng, reps)

        # replay the leader's append sequence, HEAD entries included, cut at every read of the recorder
        pieces, flat, src, gaps = AR.recording_pieces([rec.rec], L)
        assert gaps[1] is None, gaps
        hits = []
        on_head = heads_against_reports(L, rec.rec.segs, {1: rec.rec.reports, 2: cons[0].reports, 3: cons[1].reports},
                                        3, hits)
        for c0, lc in pieces:
            rp.launch(lc, requests, replica=src, on_head=on_head)
            for s, b, _ in rec.rec.segs:
                if s + len(b) == c0 + len(lc.buf):
                    AR.compare_read(rp, 1, s, b, flat)
        assert rp.pos == len(requests)
        assert rp.written >= 6 * L, rp.written / L
        assert hits, "no HEAD carried the lagging consumer's cursor: the test never gated the pruning rule"
        for cn in cons:
            assert cn.at == rp.written                          # the cursors reached the final end, in absolute terms
        # every byte and offset of every replica, reply bytes included; a follower's apply is its consumer's cursor
        for i, r in enumerate(reps):
            eo, oo = r.offsets(), rp.c.offsets(i)
            for key in ("end", "commit", "head"):
                assert eo[key] == oo[key], (i, key, eo, oo)
            assert eo["apply"] == (oo["apply"] if i == 0 else final), (i, eo)
            ei, oi = r.image(), rp.c.image(i)
            d = np.nonzero(ei != oi)[0]
            assert len(d) == 0, f"replica {i}: {len(d)} bytes differ, first at {int(d[0])}"
        st = lead.stats()
        assert st["bytes_replicated"] == rp.c.bytes_replicated()
        assert st["auto_heads"] == len(rp.heads) >= int(rp.written / L), (st["auto_heads"], len(rp.heads))
        AR.assert_heads_have_teeth(rp, rp.c.image(0))
        for cn in cons:
            check_rows(cn.rows, stream, first_idx=2)
            assert cn.rep.consume_status().next_idx == t + st["auto_heads"] + 1
        print(f"{rp.written / L:.2f} laps, {len(rp.heads)} HEAD entries replayed, {len(hits)} carried the lagging "
              f"consumer's cursor, {cons[1].calls} calls of the lagging consumer")
    finally:
        rec.stop.set()
        close_all(eng, reps)
        rp.close()


def synth_rows(seed, req_ids, length):
    """payload bytes of the device-generated requests req_ids (apus_submit_synth), one row each, vectorised"""
    r = np.asarray(req_ids, dtype=np.uint64)[:, None]
    w = np.arange((length + 3) // 4, dtype=np.uint64)[None, :]
    M = np.uint64(0xFFFFFFFF)
    x = (np.uint64(seed) ^ ((r * np.uint64(0x9E3779B1)) & M) ^ (((r >> np.uint64(32)) * np.uint64(0x7F4A7C15)) & M)
         ^ ((w * np.uint64(0x85EBCA77)) & M))
    x ^= x >> np.uint64(16); x = (x * np.uint64(0x7FEB352D)) & M
    x ^= x >> np.uint64(15); x = (x * np.uint64(0x846CA68B)) & M
    x ^= x >> np.uint64(16)
    return np.ascontiguousarray(x.astype(np.uint32)).view(np.uint8)[:, :length]


def test_benchmark_shape(eng):
    """bench.py's placement: 5 replicas, 64 B requests from apus_submit_synth, 16 leader CTAs, a 4 MiB ring lapped 8
    times with device-side pruning; every follower consumes every row"""
    import torch
    from apus_b200 import engine as E
    n, L, seed = 5, 4 << 20, 0xC0DE
    nreq = int(8.5 * L / 128)
    reps = consumer_group(eng, n, L, leader_flags=E.F_AUTOPRUNE, ring_mode=E.RING_DEVICE, ring_slots=1 << 19,
                          ring_bytes=8 << 20, ctas=16)
    try:
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        lead.submit(S.CONNECT, 0, 1, b"")
        t = lead.submit_synth(nreq, S.SEND, 0, 2, 64, seed) + nreq - 1
        EU.launch_each(eng, reps, FOREVER)
        got = []
        for r in reps[1:]:
            got.append({"rows": 0, "out": None, "stream": torch.cuda.Stream(device=r.device)})
        errs = []

        def run(r, g):
            try:
                while True:
                    g["out"] = r.consume_device(1 << 16, 64, out=g["out"], stream=g["stream"])
                    g["stream"].synchronize()
                    k = int(g["out"][6].cpu()[0])
                    if k:
                        idx, ty, co, rq, ln, pl = (x[:k].cpu().numpy() for x in g["out"][:6])
                        base = g["rows"]
                        if base == 0:
                            assert (int(ty[0]), int(rq[0])) == (S.CONNECT, 1)
                            idx, ty, co, rq, ln, pl = idx[1:], ty[1:], co[1:], rq[1:], ln[1:], pl[1:]
                            base = 1
                        want_rq = np.arange(base + 1, base + 1 + len(rq), dtype=np.uint64)
                        assert np.array_equal(rq.view(np.uint64), want_rq)
                        assert np.all(ty == S.SEND) and np.all(co == 0) and np.all(ln == 64)
                        assert np.array_equal(pl, synth_rows(seed, want_rq, 64))
                        g["rows"] += k
                    st = r.consume_status()
                    assert st.error == 0
                    if g["rows"] == nreq + 1:
                        return
            except Exception as e:        # noqa: BLE001 - reported below
                errs.append(e)
        th = [threading.Thread(target=run, args=(r, g)) for r, g in zip(reps[1:], got)]
        for x in th:
            x.start()
        lead.wait_committed(t, 300_000_000)
        for x in th:
            x.join(300)
            assert not x.is_alive()
        assert not errs, errs
        assert lead.stats()["auto_heads"] >= 8
    finally:
        close_all(eng, reps)


def test_device_round_trip(eng):
    """requests from tensors on the leader (submit_device), rows into tensors on every follower (consume_device): the
    rows are torch.equal to the inputs; invalid device requests become NOOP entries, skipped, whose idx shows the gap"""
    import torch
    from apus_b200 import engine as E
    n, L, stride = 3, 1 << 22, 200
    part = [(S.SEND, 5, 2 + k, bytes([(k * 7 + i) & 0xFF for i in range(k % 190)])) for k in range(1500)]
    bad = {17: 0, 400: 9}
    reps = consumer_group(eng, n, L, ring_mode=E.RING_DEVICE)
    try:
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        lead.submit(S.CONNECT, 5, 1, b"")
        ty, co, ri, le, pl = tensors(part, lead.device, stride)
        for k, v in bad.items():
            ty[k] = v
        t0 = lead.submit_device(ty, co, ri, le, pl)
        EU.launch_each(eng, reps, t0 + len(part) - 1)
        for r in reps:
            r.wait(60_000)
        keep = torch.tensor([k not in bad for k in range(len(part))], device=torch.device("cuda", lead.device))
        for r in reps[1:]:
            dev = torch.device("cuda", r.device)
            out = r.consume_device(4096, stride)
            torch.cuda.synchronize(r.device)
            k = int(out[6].cpu()[0])
            assert k == 1 + len(part) - len(bad)
            idx, oty, oco, ori, ole, opl = out[:6]
            assert (int(oty[0]), int(ori[0])) == (S.CONNECT, 1) and int(idx[0]) == 2
            kd = keep.to(dev)
            assert torch.equal(oty[1:k], ty.to(dev)[kd]) and torch.equal(oco[1:k], co.to(dev)[kd])
            assert torch.equal(ori[1:k], ri.to(dev)[kd]) and torch.equal(ole[1:k], le.to(dev)[kd])
            lens = le.to(dev)[kd].long()
            mask = torch.arange(stride, device=dev)[None, :] < lens[:, None]
            assert torch.equal(opl[1:k][mask], pl.to(dev)[kd][mask])
            want_idx = torch.arange(3, 3 + len(part), device=dev)[kd]
            assert torch.equal(idx[1:k], want_idx)
            st = r.consume_status()
            assert st.error == 0 and st.next_idx == 3 + len(part) and st.cursor == r.offsets()["commit"]
    finally:
        close_all(eng, reps)


def test_stride_too_small(eng):
    """examination stops exactly before the first entry whose cmd exceeds the stride; need_stride tells the stride it
    needs, and a retry with it continues with no gap"""
    n, L = 3, 1 << 22
    stream = [(S.CONNECT, 1, 1, b"")] + [(S.SEND, 1, 2 + k, bytes([k & 0xFF]) * (900 if k == 30 else 20 + k % 50))
                                         for k in range(80)]
    reps = consumer_group(eng, n, L)
    try:
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = _submit_all(lead, stream)
        EU.launch_each(eng, reps, t)
        for r in reps:
            r.wait(60_000)
        for r in reps[1:]:
            cn = Consumer(r, 100, 1000)
            k, st = cn.step(1000)
            assert k == 31 and st.need_stride == 900 and st.next_idx == 2 + 31
            k2, st2 = cn.step(1000)
            assert k2 == 0 and st2.need_stride == 900 and st2.cursor == st.cursor
            k3, st3 = cn.step(1000, stride=900)
            assert k3 == len(stream) - 31 and st3.need_stride == 0
            check_rows(cn.rows, stream, first_idx=2)
            assert [x[0] for x in cn.rows] == list(range(2, 2 + len(stream)))
            assert st3.cursor == r.offsets()["commit"]
    finally:
        close_all(eng, reps)


def test_stream_order(eng):
    """a consume queued behind a long op on the caller's stream runs after it (its outputs are overwritten only in
    stream order), work queued behind the consume sees its rows, and calls alternating between two streams deliver rows
    in call order"""
    import torch
    n, L = 3, 1 << 22
    stream = [(S.CONNECT, 2, 1, b"")] + [(S.SEND, 2, 2 + k, b"row %d" % k) for k in range(200)]
    reps = consumer_group(eng, n, L)
    try:
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = _submit_all(lead, stream)
        EU.launch_each(eng, reps, t)
        for r in reps:
            r.wait(60_000)
        r = reps[1]
        dev = torch.device("cuda", r.device)
        sa, sb = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        out = r.consume_device(8, 16, stream=sa)                 # examine idx 1..8: the CONFIG, then rows idx 2..8
        sa.synchronize()
        first = out[0][:int(out[6].cpu()[0])].clone()
        with torch.cuda.stream(sa):
            torch.cuda._sleep(50_000_000)
            for x in out:
                x.fill_(0x5A) if x.dtype == torch.uint8 else x.fill_(-3)
            r.consume_device(8, 16, out=out, stream=sa)
            seen = out[0].clone()
            done = torch.cuda.Event()
            done.record(sa)
        assert not done.query(), "the consume did not queue behind the long op"
        sa.synchronize()
        assert torch.equal(seen, torch.arange(9, 17, device=dev)), seen
        assert torch.equal(first, torch.arange(2, 9, device=dev)), first
        rows = []
        for q in range(20):
            s = sa if q % 2 == 0 else sb
            o = r.consume_device(5, 16, stream=s)
            rows.append((s, o))
        idx = []
        for s, o in rows:
            s.synchronize()
            idx += o[0][:int(o[6].cpu()[0])].cpu().tolist()
        assert idx == list(range(17, 17 + 100)), idx
        assert r.consume_status().error == 0
    finally:
        close_all(eng, reps)


def test_argument_checks(eng):
    import ctypes as C
    import torch
    from apus_b200 import engine as E
    n, L = 3, 1 << 20
    devs = devices_for(eng, n)
    with pytest.raises(E.ApusError, match="exclude each other"):
        E.Replica(devs[1], 1, n, 0, 1, L, flags=E.F_DEVICE_APPLY | E.F_HOST_APPLY)
    with pytest.raises(E.ApusError, match="followers"):
        E.Replica(devs[0], 0, n, 0, 1, L, flags=E.F_DEVICE_APPLY)
    reps = consumer_group(eng, n, L)
    plain = E.Replica(devs[2], 2, n, 0, 1, L, flags=MODES["index_earlyack"])
    try:
        with pytest.raises(E.ApusError, match="follower"):
            reps[0].consume_device(4, 16)                         # the leader
        with pytest.raises(E.ApusError, match="DEVICE_APPLY"):
            plain.consume_device(4, 16)                           # no flag
        with pytest.raises(E.ApusError, match="DEVICE_APPLY"):
            plain.consume_status()
        with pytest.raises(E.ApusError, match="max_n"):
            reps[1].consume_device(0, 16)
        out = reps[1].consume_device(4, 16)
        ptrs = [x.data_ptr() for x in out]
        s = torch.cuda.current_stream(reps[1].device).cuda_stream
        for k in range(7):                                        # each array null in turn
            p = list(ptrs)
            p[k] = None
            rc = E.lib().apus_consume_device(reps[1].h, 4, p[0], p[1], p[2], p[3], p[4], p[5], 16, p[6], s)
            assert rc == E.APUS_ERROR, k
        for k, sh in ((0, 4), (2, 1), (3, 4), (4, 1), (6, 2)):      # each 2/4/8 B array misaligned in turn
            p = list(ptrs)
            p[k] += sh
            rc = E.lib().apus_consume_device(reps[1].h, 4, p[0], p[1], p[2], p[3], p[4], p[5], 16, p[6], s)
            assert rc == E.APUS_ERROR and b"misaligned" in E.lib().apus_last_error(), k
        # payloads may be null when the stride is 0
        assert E.lib().apus_consume_device(reps[1].h, 4, ptrs[0], ptrs[1], ptrs[2], ptrs[3], ptrs[4], None, 0, ptrs[6],
                                           s) == E.APUS_OK
        torch.cuda.synchronize(reps[1].device)
        E.lib().apus_replica_set_role.argtypes = [C.c_void_p, C.c_uint8, C.c_uint64]
        with pytest.raises(E.ApusError, match="keeps its role"):
            E._ck(E.lib().apus_replica_set_role(reps[1].h, 1, 2), "apus_replica_set_role")
        E.lib().apus_ctl_adjust_follower.argtypes = [C.c_void_p, C.c_uint8, C.c_uint64, C.POINTER(C.c_uint64)]
        got = C.c_uint64()
        with pytest.raises(E.ApusError, match="consumes on the device"):
            E._ck(E.lib().apus_ctl_adjust_follower(reps[0].h, 1, 5, C.byref(got)), "apus_ctl_adjust_follower")
        assert reps[1].consume_status().error == 0
    finally:
        plain.close()
        close_all(eng, reps)


def test_destroy_right_after_enqueue(eng):
    """destroying a replica right after a consume was enqueued (behind a long op) completes, and nothing stays pending"""
    import torch
    n, L = 3, 1 << 20
    reps = consumer_group(eng, n, L)
    try:
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = _submit_all(lead, [(S.CONNECT, 1, 1, b"")] + [(S.SEND, 1, 2 + k, b"x" * k) for k in range(50)])
        EU.launch_each(eng, reps, t)
        for r in reps:
            r.wait(60_000)
        r = reps[2]
        st = torch.cuda.Stream(device=r.device)
        out = r.consume_device(64, 64, stream=st)
        st.synchronize()
        with torch.cuda.stream(st):
            torch.cuda._sleep(20_000_000)
            r.consume_device(64, 64, out=out, stream=st)
            ev = torch.cuda.Event()
            ev.record(st)
        t0 = time.monotonic()
        r.close()
        assert time.monotonic() - t0 < 10
        st.synchronize()                                          # nothing the stream waits for is left pending
        assert ev.query()
        assert int(out[6].cpu()[0]) == 0                          # everything was delivered by the first call
    finally:
        close_all(eng, [x for x in reps if x.h])
