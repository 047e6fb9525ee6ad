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
from consumers import (Consumer, PackedConsumer, check_rows, close_all, consumer_group, drain, heads_against_reports,
                       oracle_rows, wait_forwarded)
from engine_util import MODES, devices_for, eng, submit_all, tensors, torch_module  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

FOREVER = EU.FOREVER


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
        t = submit_all(lead, stream)
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
        t = submit_all(lead, stream)
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
        t = submit_all(lead, stream)
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
        t = submit_all(lead, stream)
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
        with pytest.raises(E.ApusError, match="keeps its role"):
            E._ck(E.lib().apus_replica_set_role(reps[1].h, 1, 2), "apus_replica_set_role")
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
        t = submit_all(lead, [(S.CONNECT, 1, 1, b"")] + [(S.SEND, 1, 2 + k, b"x" * k) for k in range(50)])
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
