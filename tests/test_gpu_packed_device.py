"""Ragged requests straight between GPU buffers in the packed (jagged) layout: values + offsets[n+1], as torch keeps
ragged byte data.  apus_submit_device_packed batches are checked byte for byte against the CPU oracle, interleaved with
strided device batches and host batches; apus_consume_device_packed rows are checked against the request stream and,
where the log does not lap, the oracle's log, with the capacity stop exercised on, one byte short of and one byte past
the cumulative boundaries of the rows.  Marked gpu."""
import time
import types as T

import numpy as np
import pytest

import engine_util as EU
import orc as O
import streams as S
from consumers import PackedConsumer, check_rows, close_all, consumer_group, drain, oracle_rows, wait_forwarded
from engine_util import (MODES, device_group, devices_for, eng, prune_both, submit_all, submit_host,  # noqa: F401
                         tensors, torch_module, wrap_stream)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

FOREVER = EU.FOREVER


def heavy_stream(n_req, seed, conns=3, tail_every=40):
    """SENDs of 0..256 B with a heavy tail: about one in `tail_every` is 1 KiB..64 KiB, 65535 B included"""
    rng = np.random.default_rng(seed)
    out = [(S.CONNECT, c, 1, b"") for c in range(conns)]
    rid = [1] * conns
    for i in range(n_req):
        c = int(rng.integers(0, conns))
        rid[c] += 1
        if rng.integers(0, tail_every) == 0:
            ln = 65535 if rng.integers(0, 4) == 0 else int(rng.integers(1024, 65536))
        else:
            ln = int(rng.integers(0, 257))
        out.append((S.SEND, c, rid[c], rng.integers(0, 256, size=ln, dtype=np.uint8).tobytes()))
    return out


def packed(part, device, lead=0, slack=0, lens=None):
    """the tailq_entry_t fields of `part` in the packed layout: (types, conns, req_ids, offsets, values), with the cmds
    starting `lead` bytes into values and `slack` bytes after the last; `lens` overrides a request's length (its bytes
    then come from the buffer around it)"""
    import torch
    ls = [len(p) for *_, p in part]
    if lens:
        for k, v in lens.items():
            ls[k] = v
    offs = lead + np.concatenate([[0], np.cumsum(ls)]).astype(np.int64)
    vals = np.full(int(offs[-1]) + slack, 0x3C, dtype=np.uint8)
    for k, (*_, p) in enumerate(part):
        if p:
            vals[offs[k]:offs[k] + len(p)] = np.frombuffer(p, dtype=np.uint8)
    dev = torch.device("cuda", device)
    return (torch.from_numpy(np.array([t for t, *_ in part], dtype=np.uint8)).to(dev),
            torch.from_numpy(np.array([c for _, c, _, _ in part], dtype=np.uint16).view(np.int16)).to(dev),
            torch.from_numpy(np.array([r for _, _, r, _ in part], dtype=np.uint64).view(np.int64)).to(dev),
            torch.from_numpy(offs).to(dev), torch.from_numpy(vals).to(dev))


def submit_retry(g, fn):
    """fn() until the rings have room: a full payload ring drains when the kernels consume it"""
    while True:
        try:
            return fn()
        except BlockingIOError:
            g.run()


def submit_mixed_packed(g, part, rng, max_cut=300):
    """`part` cut into packed device batches of varied sizes (some with offsets[0] > 0 into a larger values buffer),
    strided device batches and host batches; the tickets must follow one another"""
    k = 0
    dev = g.leader.device
    while k < len(part):
        way = int(rng.integers(0, 4))
        cut = part[k:k + int(rng.integers(1, max_cut if way < 2 else 60))]
        want = g.tickets + 1
        if way == 0:
            args = packed(cut, dev, lead=int(rng.integers(1, 5000)), slack=int(rng.integers(0, 3000)))
            t0 = submit_retry(g, lambda: g.submit_device_packed(*args))
        elif way == 1:
            t0 = submit_retry(g, lambda: g.submit_device_packed(*packed(cut, dev)))
        elif way == 2:
            t0 = submit_retry(g, lambda: g.submit_device(*tensors(cut, dev)))
        else:
            t0 = submit_retry(g, lambda: submit_host(g, cut))
        assert t0 == want and g.tickets == want + len(cut) - 1, (t0, want, g.tickets)
        k += len(cut)


def _stream(kind, n):
    if kind == "ragged":
        return S.ragged_stream(3000, 1500, conns=4, seed=600 + n, close_every=50)
    return heavy_stream(2000, 610 + n)


@pytest.mark.parametrize("kind", ["ragged", "heavy"])
@pytest.mark.parametrize("n", [3, 5])
def test_packed_batches_match_oracle(eng, orc, n, kind):
    """packed batches of varied sizes, some with offsets[0] > 0 into a larger values buffer, interleaved with strided
    device batches and host batches: the same logs as the oracle's for the same stream, no request rejected"""
    L = 1 << 22
    stream = _stream(kind, n)
    rng = np.random.default_rng(n * 7 + len(kind))
    with device_group(eng, n, L) as g:
        g.prologue()
        submit_mixed_packed(g, stream, rng)
        g.run()
        c = EU.oracle_cluster(orc, n, L, stream)
        EU.compare_group_to_oracle(g, c, exact=True)
        assert g.leader.committed() == len(stream) + 1
        assert g.leader.device_submit_status() == (0, 0)
        c.close()


def test_batch_refused_strided_is_accepted_packed(eng, orc):
    """1024 heavy-tailed requests with one 65535 B cmd: strided, stride 65535 reserves 1024 x 65552 B, more than the
    default 16 MiB payload ring; packed, the reservation is bounded by the values bytes and the batch goes through"""
    n, L = 3, 1 << 23
    part = heavy_stream(1021, 620, tail_every=10 ** 9)
    part[500] = (part[500][0], part[500][1], part[500][2], bytes(range(256)) * 255 + bytes(255))
    assert len(part) == 1024 and max(len(p) for *_, p in part) == 65535
    with device_group(eng, n, L) as g:
        g.prologue()
        with pytest.raises(eng.ApusError, match="can never fit"):
            g.submit_device(*tensors(part, g.leader.device, 65535))
        g.submit_device_packed(*packed(part, g.leader.device))
        g.run()
        c = EU.oracle_cluster(orc, n, L, part)
        EU.compare_group_to_oracle(g, c, exact=True)
        assert g.leader.device_submit_status() == (0, 0)
        c.close()


@pytest.mark.parametrize("kind,seed,ctas", [("ragged1500", 631, 2), ("u960", 632, 4), ("heavy", 633, 16)])
def test_packed_batches_lap_payload_ring_and_log(eng, orc, kind, seed, ctas):
    """The smallest payload ring (128 KiB) and a 256 KiB log: packed batches wrap the payload ring many times and the
    log more than four times, with HEAD entries at quiescent points"""
    n, L, R = 3, 1 << 18, 1 << 17
    if kind == "heavy":
        stream = heavy_stream(int(4.5 * L / 300), seed, tail_every=60)
        stream = [(t, c, r, p[:12000]) for t, c, r, p in stream]          # a 60-request cut stays below R
    else:
        stream = wrap_stream(kind, seed, L)
    assert S.stream_bytes(stream) >= 4 * L
    step = max(1, int(0.3 * L * len(stream) / S.stream_bytes(stream)))
    rng = np.random.default_rng(seed)
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, n, leader=0, term=1, length=L)
    c.prologue()
    reserved = 0
    with device_group(eng, n, L, ring_slots=1 << 12, ring_bytes=R, flags=MODES["index_earlyack"], leader_ctas=ctas) as g:
        g.prologue()
        total = 1
        for k in range(0, len(stream), step):
            part = stream[k:k + step]
            for typ, clt, rid, payload in part:
                assert c.submit(typ, clt, rid, O.cmd_image(payload)) != 0
            c.round(); c.round()
            j = 0
            while j < len(part):
                cut = part[j:j + int(rng.integers(1, 60))]
                args = packed(cut, g.leader.device, lead=int(rng.integers(0, 64)))
                try:
                    g.submit_device_packed(*args)
                except BlockingIOError:
                    g.run()
                    continue
                reserved += min(len(cut) * 65552, (args[4].numel() + 17 * len(cut) + 15) & ~15)
                j += len(cut)
            total += len(part)
            g.run()
            if prune_both(g, c):
                total += 1
                c.round(); c.round()
                g.run()
        EU.compare_group_to_oracle(g, c, exact=True)
        assert reserved >= 5 * R
        assert g.leader.committed() == total
        assert g.leader.offsets()["head"] == c.offsets(0)["head"] != 0
        assert g.leader.device_submit_status() == (0, 0)
    c.close()


def test_packed_rejections(eng, orc):
    """invalid types and cmds above 65535 B become NOOPs at their own tickets; a batch with one decreasing offset, and
    a batch whose offsets end past values, become NOOPs entirely; every batch after them still matches the oracle"""
    import torch
    n, L = 3, 1 << 22
    rng = np.random.default_rng(640)
    base = S.ragged_stream(400, 1500, conns=2, seed=641)
    a, b, cc, d = base[:100], base[100:200], base[200:300], base[300:]
    with device_group(eng, n, L) as g:
        g.prologue()
        expect = []
        # per request: types 0, 2, 3, 9 and a 70000 B cmd
        bad = {7: 0, 13: 2, 21: 3, 30: 9}
        too_long = 44
        ty, co, ri, of, va = packed(a, g.leader.device, lens={too_long: 70000})
        for k, t in bad.items():
            ty[k] = t
        t_a = g.submit_device_packed(ty, co, ri, of, va)
        expect += [(O.NOOP, c_, r_, b"") if (k in bad or k == too_long) else (t_, c_, r_, p_)
                   for k, (t_, c_, r_, p_) in enumerate(a)]
        torch.cuda.synchronize(g.leader.device)
        assert g.leader.device_submit_status() == (5, t_a + 7)
        g.submit_device_packed(*packed(b, g.leader.device))          # a good batch after it
        expect += b
        # one decreasing offset: the whole batch
        ty, co, ri, of, va = packed(cc, g.leader.device, lead=100)
        of[37] = of[36] - 1
        t_c = g.submit_device_packed(ty, co, ri, of, va)
        expect += [(O.NOOP, c_, r_, b"") for _, c_, r_, _ in cc]
        # offsets[n] past values: the whole batch
        ty, co, ri, of, va = packed(d, g.leader.device)
        t_d = g.submit_device_packed(ty, co, ri, of, va[:-1])
        expect += [(O.NOOP, c_, r_, b"") for _, c_, r_, _ in d]
        torch.cuda.synchronize(g.leader.device)
        assert g.leader.device_submit_status() == (5 + len(cc) + len(d), t_a + 7)
        assert t_d == t_c + len(cc)
        # later batches, every layout
        more = S.ragged_stream(600, 1500, conns=2, seed=642)
        more = [(t_, c_ + 10, r_, p_) for t_, c_, r_, p_ in more]
        submit_mixed_packed(g, more, rng, max_cut=100)
        expect += more
        g.run()
        c = EU.oracle_cluster(orc, n, L, expect)
        EU.compare_group_to_oracle(g, c, exact=True)
        assert g.leader.device_submit_status() == (5 + len(cc) + len(d), t_a + 7)
        c.close()


@pytest.mark.parametrize("bad", ["decrease", "overrun"])
def test_batch_verdict_reaches_every_block(eng, orc, bad):
    """a batch of 700 requests spans three packing blocks (256 requests each); the one bad offset lies in a single block
    -- a decrease inside the third, or offsets[n] past values, which only the last request's block sees -- and every
    request of every block becomes a NOOP, so the blocks without a bad offset pack nothing into the reservation the
    scan computed as empty; the batches after it match the oracle"""
    import torch
    n, L = 3, 1 << 22
    rng = np.random.default_rng(660)
    part = [(t, c, r, p) for t, c, r, p in S.ragged_stream(697, 1500, conns=3, seed=661)][:700]
    assert len(part) == 700
    with device_group(eng, n, L) as g:
        g.prologue()
        ty, co, ri, of, va = packed(part, g.leader.device, lead=40)
        if bad == "decrease":
            of[600] = of[599] - 1                       # block 2 (requests 512..699) only
            t0 = g.submit_device_packed(ty, co, ri, of, va)
        else:
            t0 = g.submit_device_packed(ty, co, ri, of, va[:-1])
        torch.cuda.synchronize(g.leader.device)
        assert g.leader.device_submit_status() == (len(part), t0)
        expect = [(O.NOOP, c_, r_, b"") for _, c_, r_, _ in part]
        more = [(t_, c_ + 10, r_, p_) for t_, c_, r_, p_ in S.ragged_stream(500, 1500, conns=2, seed=662)]
        submit_mixed_packed(g, more, rng, max_cut=300)
        expect += more
        g.run()
        c = EU.oracle_cluster(orc, n, L, expect)
        EU.compare_group_to_oracle(g, c, exact=True)
        assert g.leader.device_submit_status() == (len(part), t0)
        c.close()


@pytest.mark.parametrize("kind", ["ragged", "heavy"])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_packed_consumption_matches_oracle(eng, orc, mode, kind):
    """packed consumers in every follower mode while the kernels run, max_n from 1 up and values_cap on, one byte short
    of and one byte past the rows' cumulative boundaries: every row equals the stream and the oracle's log, nothing is
    written past offsets[count], and once everything is committed each call stops exactly where the capacity says; the
    final cursor is every follower's commit offset and forwarded apply offset"""
    n, L = 3, 1 << 22
    stream = _stream(kind, n)[:2500]
    reps = consumer_group(eng, n, L, MODES[mode])
    rng = np.random.default_rng(len(mode) * 13 + len(kind))
    try:
        cons = [PackedConsumer(r, [len(p) for *_, p in stream], seed=k) for k, r in enumerate(reps[1:])]
        EU.launch_each(eng, reps, FOREVER)
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = submit_all(lead, stream)
        last_idx = len(stream) + 1
        for cn in cons:
            # exact once this follower holds every entry as committed (and the CONFIG at idx 1 is behind the cursor)
            cn.exact = lambda cn=cn: (lead.committed() >= t and len(cn.rows) > 0 and
                                      cn.rep.offsets()["commit"] == lead.offsets()["end"])
            drain(cn, lambda st: st.next_idx == last_idx + 1, [1, 2, 7, 64, 333, 4096], rng)
        lead.wait_committed(t)
        wait_forwarded(reps)
        EU.stop_each(eng, reps)
        c = EU.oracle_cluster(orc, n, L, stream)
        EU.compare_group_to_oracle(T.SimpleNamespace(n=n, replicas=reps, leader_idx=0), c, exact=True)
        for j, cn in enumerate(cons, 1):
            check_rows(cn.rows, stream, first_idx=2)
            assert cn.rows == oracle_rows(c, j)
            st = reps[j].consume_status()
            assert st.cursor == reps[j].offsets()["commit"] == reps[j].offsets()["apply"] == c.offsets(j)["commit"]
            assert st.next_idx == last_idx + 1 and st.error == 0
        c.close()
    finally:
        close_all(eng, reps)


def test_capacity_stop(eng):
    """a values_cap smaller than the next cmd: count 0, need_stride is that cmd's length, the cursor stays; that
    capacity then delivers it.  A stop after rows were delivered is no error: need_stride stays 0"""
    n, L = 3, 1 << 22
    stream = [(S.CONNECT, 1, 1, b"")] + [(S.SEND, 1, 2 + k, bytes([k & 0xFF]) * (900 if k == 30 else 20 + k % 50))
                                         for k in range(400)]
    lens = [len(p) for *_, p in stream]
    reps = consumer_group(eng, n, L)
    try:
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        t = submit_all(lead, stream)
        EU.launch_each(eng, reps, t)
        for r in reps:
            r.wait(60_000)
        for r in reps[1:]:
            cn = PackedConsumer(r, lens)
            k, st = cn.step(1000, cap=sum(lens[:31]))            # rows up to the long one exactly
            assert k == 31 and st.need_stride == 0 and st.next_idx == 2 + 31
            k2, st2 = cn.step(1000, cap=899)
            assert k2 == 0 and st2.need_stride == 900 and st2.cursor == st.cursor and st2.next_idx == st.next_idx
            k3, st3 = cn.step(1000, cap=900)
            assert k3 == 1 and st3.need_stride == 0 and st3.next_idx == st.next_idx + 1
            k4, st4 = cn.step(300, cap=sum(lens[32:332]) - 1)      # one byte short, across a block boundary
            assert k4 == 299 and st4.need_stride == 0
            k5, st5 = cn.step(1000, cap=1 << 20)
            assert k5 == len(stream) - 331 and st5.need_stride == 0
            check_rows(cn.rows, stream, first_idx=2)
            assert [x[0] for x in cn.rows] == list(range(2, 2 + len(stream)))
            assert st5.cursor == r.offsets()["commit"]
            k6, st6 = cn.step(4, cap=0)                           # nothing left: count 0, offsets[0] = 0
            assert k6 == 0 and st6.need_stride == 0
    finally:
        close_all(eng, reps)


def test_jagged_round_trip(eng):
    """values + offsets on the leader (submit_device_packed), values + offsets on every follower (consume_device_packed):
    the same bytes and offsets; invalid requests become NOOP entries, skipped, whose idx shows the gap"""
    import torch
    from apus_b200 import engine as E
    n, L = 3, 1 << 22
    part = heavy_stream(1500, 650, conns=1, tail_every=100)[1:]
    part = [(S.SEND, 5, 2 + k, p) for k, (_, _, _, p) in enumerate(part)]
    bad = {17: 0, 400: 9}
    reps = consumer_group(eng, n, L, ring_mode=E.RING_DEVICE)
    try:
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        lead.submit(S.CONNECT, 5, 1, b"")
        ty, co, ri, of, va = packed(part, lead.device, lead=3)
        for k, v in bad.items():
            ty[k] = v
        t0 = lead.submit_device_packed(ty, co, ri, of, va)
        EU.launch_each(eng, reps, t0 + len(part) - 1)
        for r in reps:
            r.wait(60_000)
        keep = [k not in bad for k in range(len(part))]
        kept = [p for k, (*_, p) in enumerate(part) if keep[k]]
        for r in reps[1:]:
            dev = torch.device("cuda", r.device)
            cap = 1 + sum(len(p) for p in kept)
            out = r.consume_device_packed(4096, cap)
            torch.cuda.synchronize(r.device)
            k = int(out[6].cpu()[0])
            assert k == 1 + len(kept)
            idx, oty, oco, ori, oof, ova = out[:6]
            assert (int(oty[0]), int(ori[0])) == (S.CONNECT, 1) and int(idx[0]) == 2 and int(oof[1]) == 0
            kd = torch.tensor(keep, device=dev)
            assert torch.equal(oty[1:k], ty.to(dev)[kd]) and torch.equal(oco[1:k], co.to(dev)[kd])
            assert torch.equal(ori[1:k], ri.to(dev)[kd])
            lens_in = (of[1:] - of[:-1]).to(dev)[kd]
            assert torch.equal(oof[2:k + 1] - oof[1:k], lens_in)
            want = torch.cat([va[int(of[q]):int(of[q + 1])] for q in range(len(part)) if keep[q]]).to(dev)
            assert torch.equal(ova[:int(oof[k])], want)
            assert torch.equal(idx[1:k], torch.arange(3, 3 + len(part), device=dev)[kd])
            st = r.consume_status()
            assert st.error == 0 and st.next_idx == 3 + len(part) and st.cursor == r.offsets()["commit"]
    finally:
        close_all(eng, reps)


def test_packed_stream_order(eng):
    """a packed batch whose values a producer kernel on the caller's stream writes after the call returns is packed
    after it, and the inputs may be overwritten right after the call; a packed consume queued behind a long op runs
    after it, and work queued behind it sees its rows"""
    import torch
    n, L = 3, 1 << 22
    part = [(S.CONNECT, 3, 1, b"")] + [(S.SEND, 3, 2 + k, bytes([(k * 13 + i) & 0xFF for i in range(40 + 97 * k)]))
                                        for k in range(63)]
    reps = consumer_group(eng, n, L, ring_mode=eng.RING_DEVICE)
    try:
        lead = reps[0]
        lead.submit(O.CONFIG, 0, 0, O.cid_image(n))
        st = torch.cuda.Stream(device=lead.device)
        ty, co, ri, of, va = packed(part, lead.device)
        new_va = va.clone()
        va.zero_()
        torch.cuda.synchronize(lead.device)
        with torch.cuda.stream(st):
            torch.cuda._sleep(50_000_000)                 # the producer is still running when the call returns ...
            va.copy_(new_va)                              # ... and only then writes the values
            t0 = lead.submit_device_packed(ty, co, ri, of, va, stream=st)
            va.fill_(0xEE); of.fill_(0)                   # overwritten right after the call, in stream order
        EU.launch_each(eng, reps, t0 + len(part) - 1)
        for r in reps:
            r.wait(60_000)
        st.synchronize()
        r = reps[1]
        dev = torch.device("cuda", r.device)
        sa = torch.cuda.Stream(device=dev)
        out = r.consume_device_packed(8, 1 << 16, stream=sa)         # idx 1..8: the CONFIG, then part[0:7]
        sa.synchronize()
        o0 = out[4][:8].cpu().numpy()
        assert int(out[6].cpu()[0]) == 7
        assert [out[5][o0[q]:o0[q + 1]].cpu().numpy().tobytes() for q in range(7)] == [p for *_, p in part[:7]]
        with torch.cuda.stream(sa):
            torch.cuda._sleep(50_000_000)
            for x in out:
                x.fill_(0x5A) if x.dtype == torch.uint8 else x.fill_(-3)
            r.consume_device_packed(8, 1 << 16, out=out, stream=sa)
            seen_idx, seen_off = out[0].clone(), out[4].clone()
            done = torch.cuda.Event()
            done.record(sa)
        assert not done.query(), "the consume did not queue behind the long op"
        sa.synchronize()
        assert torch.equal(seen_idx, torch.arange(9, 17, device=dev)), seen_idx
        want = np.concatenate([[0], np.cumsum([len(p) for *_, p in part[7:15]])])
        assert seen_off.cpu().tolist() == want.tolist()
        rest = r.consume_device_packed(4096, 1 << 20)
        torch.cuda.synchronize(r.device)
        k = int(rest[6].cpu()[0])
        assert k == len(part) - 15
        oo = rest[4][:k + 1].cpu().numpy()
        vv = rest[5].cpu().numpy()
        rows = [vv[oo[q]:oo[q + 1]].tobytes() for q in range(k)]
        assert rows == [p for *_, p in part[15:]]
    finally:
        close_all(eng, reps)


def test_packed_argument_checks(eng):
    import torch
    from apus_b200 import engine as E
    n, L = 3, 1 << 20
    devs = devices_for(eng, n)
    reps = consumer_group(eng, n, L, ring_mode=E.RING_DEVICE, ring_slots=256)
    plain = E.Replica(devs[2], 2, n, 0, 1, L, flags=MODES["index_earlyack"])
    try:
        lead = reps[0]
        part = [(S.SEND, 1, 1 + k, b"x" * (k % 90)) for k in range(200)]
        ty, co, ri, of, va = packed(part, lead.device)
        with pytest.raises(E.ApusError):
            lead.submit_device_packed(ty, co, ri, of.to(torch.int32), va)                 # dtype
        with pytest.raises(E.ApusError):
            lead.submit_device_packed(ty, co, ri, of[:-1], va)                            # shape
        with pytest.raises(E.ApusError):
            lead.submit_device_packed(ty, co.cpu(), ri, of, va)                           # device
        with pytest.raises(E.ApusError):
            lead.submit_device_packed(ty, co, torch.stack([ri, ri], 1)[:, 0], of, va)     # contiguity
        s = torch.cuda.current_stream(lead.device).cuda_stream
        p = [ty.data_ptr(), co.data_ptr(), ri.data_ptr(), of.data_ptr(), va.data_ptr()]
        for k in range(5):                                                                # each array null in turn
            q = list(p)
            q[k] = None
            assert E.lib().apus_submit_device_packed(lead.h, 200, q[0], q[1], q[2], q[3], q[4], va.numel(), s,
                                                     None) == E.APUS_ERROR, k
        for k, sh in ((1, 1), (2, 4), (3, 4)):                                            # misaligned 2/8 B arrays
            q = list(p)
            q[k] += sh
            rc = E.lib().apus_submit_device_packed(lead.h, 200, q[0], q[1], q[2], q[3], q[4], va.numel(), s, None)
            assert rc == E.APUS_ERROR and b"misaligned" in E.lib().apus_last_error(), k
        big = [(S.SEND, 1, 1 + k, b"") for k in range(300)]
        with pytest.raises(E.ApusError, match="can never fit"):
            lead.submit_device_packed(*packed(big, lead.device))                          # 300 > 256 slots
        with pytest.raises(E.ApusError, match="follower"):
            reps[1].submit_device_packed(*packed(part, reps[1].device))
        with pytest.raises(E.ApusError, match="device submission ring"):
            plain_lead = E.Replica(devs[0], 0, n, 0, 1, L, flags=MODES["index_earlyack"])
            try:
                plain_lead.submit_device_packed(*packed(part, plain_lead.device))
            finally:
                plain_lead.close()
        assert lead.submit_device_packed(ty, co, ri, of, va) == 1
        with pytest.raises(BlockingIOError):
            lead.submit_device_packed(ty, co, ri, of, va)                                 # ring full: nothing reserved
        # consumption
        with pytest.raises(E.ApusError, match="follower"):
            lead.consume_device_packed(4, 16)
        with pytest.raises(E.ApusError, match="DEVICE_APPLY"):
            plain.consume_device_packed(4, 16)
        with pytest.raises(E.ApusError, match="max_n"):
            reps[1].consume_device_packed(0, 16)
        with pytest.raises(E.ApusError):
            reps[1].consume_device_packed(4, 16, out=reps[1].consume_device_packed(5, 16))   # shapes
        out = reps[1].consume_device_packed(4, 16)
        ptrs = [x.data_ptr() for x in out]
        s = torch.cuda.current_stream(reps[1].device).cuda_stream
        for k in range(7):
            q = list(ptrs)
            q[k] = None
            rc = E.lib().apus_consume_device_packed(reps[1].h, 4, q[0], q[1], q[2], q[3], q[4], q[5], 16, q[6], s)
            assert rc == E.APUS_ERROR, k
        for k, sh in ((0, 4), (2, 1), (3, 4), (4, 4), (6, 2)):
            q = list(ptrs)
            q[k] += sh
            rc = E.lib().apus_consume_device_packed(reps[1].h, 4, q[0], q[1], q[2], q[3], q[4], q[5], 16, q[6], s)
            assert rc == E.APUS_ERROR and b"misaligned" in E.lib().apus_last_error(), k
        # values may be null when values_cap is 0, and may have any alignment
        assert E.lib().apus_consume_device_packed(reps[1].h, 4, ptrs[0], ptrs[1], ptrs[2], ptrs[3], ptrs[4], None, 0,
                                                  ptrs[6], s) == E.APUS_OK
        assert E.lib().apus_consume_device_packed(reps[1].h, 4, ptrs[0], ptrs[1], ptrs[2], ptrs[3], ptrs[4],
                                                  ptrs[5] + 3, 13, ptrs[6], s) == E.APUS_OK
        torch.cuda.synchronize(reps[1].device)
        assert reps[1].consume_status().error == 0
    finally:
        plain.close()
        close_all(eng, reps)


def test_packed_destroy_right_after_enqueue(eng):
    """destroying a replica right after a packed consume was enqueued (behind a long op) completes, and nothing stays
    pending"""
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
        out = r.consume_device_packed(64, 4096, stream=st)
        st.synchronize()
        assert int(out[6].cpu()[0]) == 51
        with torch.cuda.stream(st):
            torch.cuda._sleep(20_000_000)
            r.consume_device_packed(64, 4096, out=out, stream=st)
            ev = torch.cuda.Event()
            ev.record(st)
        t0 = time.monotonic()
        r.close()
        assert time.monotonic() - t0 < 10
        st.synchronize()
        assert ev.query()
        assert int(out[6].cpu()[0]) == 0
    finally:
        close_all(eng, [x for x in reps if x.h])
