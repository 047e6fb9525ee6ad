"""Requests submitted straight from GPU memory (apus_submit_device) and stream-ordered commit waits
(apus_stream_wait_committed), against the CPU oracle: byte for byte, the logs a device batch leaves are the logs the
same request stream leaves when the host submits it.  Marked gpu."""
import time

import numpy as np
import pytest

import engine_util as EU
import orc as O
import streams as S
from engine_util import (MODES, device_group, devices_for, eng, hole_bytes, prune_both, submit_host,  # noqa: F401
                         tensors, torch_module, wrap_stream)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(180)]

FOREVER = EU.FOREVER


def submit_mixed(g, part, rng):
    """`part` cut into device batches of varied sizes, every third cut through apus_submit_batch instead; the tickets
    returned must follow one another"""
    k = 0
    while k < len(part):
        m = int(rng.integers(1, 300))
        cut = part[k:k + m]
        want = g.tickets + 1
        if rng.integers(0, 3) == 0:
            t0 = submit_host(g, cut)
        else:
            t0 = g.submit_device(*tensors(cut, g.leader.device))
        assert t0 == want and g.tickets == want + len(cut) - 1
        k += m


@pytest.mark.parametrize("n,seed", [(3, 401), (5, 402)])
def test_ragged_device_batches_match_oracle(eng, orc, n, seed):
    """ragged_stream (0..1500 B, CLOSE / CONNECT churn) in device batches of varied sizes, interleaved with host
    batches: the same logs as the oracle's for the same stream"""
    L = 1 << 22
    stream = S.ragged_stream(3000, 1500, conns=4, seed=seed, close_every=50)
    rng = np.random.default_rng(seed)
    with device_group(eng, n, L) as g:
        g.prologue()
        submit_mixed(g, stream, rng)
        g.run()
        c = EU.oracle_cluster(orc, n, L, stream)
        EU.compare_group_to_oracle(g, c, exact=True)
        assert g.leader.committed() == len(stream) + 1
        assert g.leader.device_submit_status() == (0, 0)
        c.close()


@pytest.mark.parametrize("kind,seed,ctas", [("ragged1500", 411, 2), ("u200", 412, 16), ("u960", 413, 4)])
def test_device_batches_lap_payload_ring_and_log(eng, orc, kind, seed, ctas):
    """The smallest payload ring the engine takes (128 KiB) and a 256 KiB log: device batches wrap the payload ring many
    times and the log more than four times, with HEAD entries at quiescent points as in test_wrap_laps_with_pruning"""
    n, L, R = 3, 1 << 18, 1 << 17
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
        total, written, prev, marks = 1, 0, c.offsets(0)["end"], []
        for k in range(0, len(stream), step):
            part = stream[k:k + step]
            for typ, clt, rid, payload in part:
                assert c.submit(typ, clt, rid, O.cmd_image(payload)) != 0
            c.round(); c.round()
            j = 0
            while j < len(part):
                cut = part[j:j + int(rng.integers(1, 60))]
                stride = max([len(p) for *_, p in cut] + [1])
                try:
                    g.submit_device(*tensors(cut, g.leader.device, stride))
                except BlockingIOError:                 # the payload ring is full: let the kernels consume it
                    g.run()
                    continue
                if 2 + stride > 80:
                    reserved += len(cut) * ((2 + stride + 15) & ~15)
                j += len(cut)
            total += len(part)
            g.run()
            if prune_both(g, c):
                total += 1
                c.round(); c.round()
                g.run()
            e = c.offsets(0)["end"]
            written += (e - prev) % L
            prev = e
            marks.append((written, e))
        EU.compare_group_to_oracle(g, c, exact=True)
        assert reserved >= 5 * R                                # payload-ring laps
        start = next(e for w, e in marks if written - w < L)
        img = c.image(0)
        ents = O.walk_entries(img, start, prev, L)
        holes = hole_bytes(img, ents)
        assert np.count_nonzero(holes) >= 0.5 * len(holes)
        assert g.leader.committed() == total
        assert g.leader.offsets()["head"] == c.offsets(0)["head"] != 0
    c.close()


def _order_case(eng, orc, overwrite_after):
    import torch
    n, L = 3, 1 << 20
    part = [(S.CONNECT, 3, 1, b"")] + [(S.SEND, 3, 2 + k, bytes([(k * 13 + i) & 0xFF for i in range(40 + 7 * k)]))
                                        for k in range(63)]
    old = [(t, c, r, bytes(len(p))) for t, c, r, p in part]
    with device_group(eng, n, L) as g:
        g.prologue()
        st = torch.cuda.Stream(device=g.leader.device)
        ty, co, ri, le, pl = tensors(part if overwrite_after else old, g.leader.device)
        new_pl = tensors(part, g.leader.device)[4]
        torch.cuda.synchronize(g.leader.device)
        with torch.cuda.stream(st):
            if not overwrite_after:
                torch.cuda._sleep(50_000_000)             # the producer is still running when the call returns ...
                pl.copy_(new_pl)                          # ... and only then writes the payloads
            g.submit_device(ty, co, ri, le, pl, stream=st)
            if overwrite_after:
                pl.fill_(0xEE); ty.fill_(0); le.fill_(0)  # overwritten right after the call, in stream order
        g.run()
        st.synchronize()
        c = EU.oracle_cluster(orc, n, L, part)
        EU.compare_group_to_oracle(g, c, exact=True)
        c.close()


def test_stream_order_read_side(eng, orc):
    """the packing sees what the caller's stream wrote before the call, with no host synchronisation"""
    _order_case(eng, orc, overwrite_after=False)


def test_stream_order_write_side(eng, orc):
    """the caller's stream may overwrite the input tensors right after the call"""
    _order_case(eng, orc, overwrite_after=True)


def test_invalid_requests_become_noops(eng, orc):
    """types 0, 2, 3, 9 and len > stride are written as the NOOP apus_submit would write at that ticket"""
    import torch
    n, L, stride = 3, 1 << 20, 120
    part = [(S.CONNECT, 5, 1, b"")] + [(S.SEND, 5, 2 + k, bytes([(k + i) & 0xFF for i in range(k % 110)])) for k in range(60)]
    bad = {7: 0, 13: 2, 21: 3, 30: 9}
    too_long = 44
    with device_group(eng, n, L) as g:
        g.prologue()
        ty, co, ri, le, pl = tensors(part, g.leader.device, stride)
        for k, t in bad.items():
            ty[k] = t
        le[too_long] = stride + 1
        t0 = g.submit_device(ty, co, ri, le, pl)
        g.run()
        torch.cuda.synchronize(g.leader.device)
        expect = [(O.NOOP, c, r, b"") if (k in bad or k == too_long) else (t, c, r, p) for k, (t, c, r, p) in enumerate(part)]
        c = EU.oracle_cluster(orc, n, L, expect)
        EU.compare_group_to_oracle(g, c, exact=True)
        assert g.leader.device_submit_status() == (5, t0 + 7)
        c.close()


def test_host_checks(eng):
    import torch
    part = [(S.SEND, 1, 1 + k, b"x" * 10) for k in range(200)]
    with device_group(eng, 3, 1 << 20, ring_slots=256) as g:
        dev = g.leader.device
        ty, co, ri, le, pl = tensors(part, dev)
        with pytest.raises(eng.ApusError):
            g.submit_device(ty.to(torch.int32), co, ri, le, pl)                  # dtype
        with pytest.raises(eng.ApusError):
            g.submit_device(ty, co.cpu(), ri, le, pl)                            # device
        with pytest.raises(eng.ApusError):
            g.submit_device(ty, co, torch.stack([ri, ri], 1)[:, 0], le, pl)      # contiguity
        with pytest.raises(eng.ApusError):
            g.submit_device(ty, co, ri, le[:-1], pl)                             # shape
        big = [(S.SEND, 1, 1 + k, b"") for k in range(300)]
        with pytest.raises(eng.ApusError):
            g.submit_device(*tensors(big, dev))                                  # can never fit 256 slots
        t0 = g.submit_device(ty, co, ri, le, pl)
        assert t0 == 1
        with pytest.raises(BlockingIOError):
            g.submit_device(ty, co, ri, le, pl)                                  # ring full: nothing reserved
        assert g.submit(S.SEND, 1, 999, b"next") == 201
    with eng.Group(3, devices=devices_for(eng, 3), log_size=1 << 20) as g:        # host-mapped ring
        with pytest.raises(eng.ApusError):
            g.submit_device(*tensors(part, g.leader.device))


class _Word:
    """the committed-tickets word (pinned, mapped) as a CUDA array torch can wrap"""

    def __init__(self, ptr):
        self.__cuda_array_interface__ = {"shape": (1,), "typestr": "<i8", "data": (ptr, False), "version": 3}


def test_wait_committed_on_stream(eng):
    """with resident kernels and the doorbell deferred, work enqueued after the wait runs only once the ticket has
    committed, and sees the committed count"""
    import torch
    n, L = 3, 1 << 20
    part = [(S.CONNECT, 2, 1, b"")] + [(S.SEND, 2, 2 + k, b"payload %d" % k) for k in range(100)]
    with device_group(eng, n, L) as g:
        dev = g.leader.device
        word = torch.as_tensor(_Word(g.leader.committed_word()), device=torch.device("cuda", dev))
        st = torch.cuda.Stream(device=dev)
        args = tensors(part, dev)
        word.clone()                      # load torch's copy kernel before the replica kernels are resident
        torch.cuda.synchronize(dev)
        g.launch(target=FOREVER)
        g.leader.wait_committed(g.prologue())
        g.leader.defer(True)
        with torch.cuda.stream(st):
            g.submit_device(*args, stream=st)
            g.leader.wait_committed_on_stream(g.tickets, stream=st)
            seen = word.clone()
            done = torch.cuda.Event()
            done.record(st)
        time.sleep(0.1)
        assert not done.query(), "the wait passed before the doorbell was rung"
        assert g.leader.committed() < g.tickets
        g.leader.flush()
        t = time.monotonic()
        while not done.query():
            assert time.monotonic() - t < 5, "the wait did not pass within 5 s of the commit"
            time.sleep(0.001)
        assert int(seen.item()) >= g.tickets
        g.leader.defer(False)
        g.stop()


def test_destroy_releases_pending_wait(eng):
    """a stream waiting on a ticket that cannot commit (no kernels) is released by destroy"""
    import torch
    g = device_group(eng, 3, 1 << 20)
    try:
        st = torch.cuda.Stream(device=g.leader.device)
        g.leader.wait_committed_on_stream(10, stream=st)
        ev = torch.cuda.Event()
        ev.record(st)
        time.sleep(0.05)
        assert not ev.query()
        t = time.monotonic()
        g.leader.close()
        while not ev.query():
            assert time.monotonic() - t < 1, "destroy did not release the wait"
            time.sleep(0.001)
        st.synchronize()
    finally:
        g.close()
