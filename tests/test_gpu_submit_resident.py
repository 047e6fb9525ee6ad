"""Resident submitters (apus_submitter_attach, include/apus_submitter.cuh) against the CPU oracle: an application's
own persistent kernel (tests/devicelogic/resident_submit.cu, one or several CTAs) reserves, writes and publishes
requests into the leader's HBM ring, and every replica's log equals the oracle's log of the same requests in ticket
order, byte for byte.  Also the hand-over to and from the host paths, a dropped reservation, rejected types, commit
waits, the refusals, and the whole loop on the device with resident consumers on every replica.  Marked gpu."""
import ctypes as C
import time

import pytest

import autoprune_replay as AR
import engine_util as EU
import orc as O
import resident
import streams as S
import submitter as SB
from apus_b200 import engine as E
from engine_util import MODES, device_group, devices_for, eng, submit_host, tensors, torch_module  # noqa: F401
from shadow import check_heads

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

FOREVER = EU.FOREVER
ANY = E.F_DEVICE_APPLY | E.F_APPLY_ANY_ROLE


@pytest.fixture(scope="module", autouse=True)
def loaded(eng):
    """the test kernels are loaded before any replica kernel is resident"""
    SB.lib()
    resident.lib()


def run_submitter(g, view, stream, requests, batch, ctas, mode=0, timeout_s=30.0):
    """launch the group for everything the submitter will publish, then the submitter; wait for both"""
    sub = SB.Submitter(view, stream, requests, batch=batch, ctas=ctas, mode=mode, timeout_s=timeout_s)
    g.tickets += len(requests)
    g.launch()
    sub.start()
    fail, pub, tickets = sub.result()
    assert fail is None and pub == len(requests), (fail, pub)
    g.wait(60_000)
    return tickets


def oracle_of(orc, n, L, stream):
    return EU.oracle_cluster(orc, n, L, stream)


@pytest.mark.parametrize("n,ctas", [(3, 1), (3, 4), (5, 1), (5, 4)])
def test_submitter_matches_oracle(eng, orc, n, ctas):
    """seeded requests of mixed types and sizes (0..1500 B, some up to 64 KiB, some rejected): the logs are the
    oracle's log of the same requests in ticket order; tickets are contiguous and the rejections are counted.  A SEND
    of 65535 B is written as it is; SENDs of 65536 and 70000 B, whose length the descriptor cannot carry, become counted
    NOOPs, and every entry after them stays byte-exact"""
    import torch
    L = 1 << 22
    reqs = SB.mixed_requests(2500, seed=500 + 10 * n + ctas, big_every=97)
    for k, ln in ((700, 65535), (701, 65536), (1500, 70000)):
        reqs[k] = (S.SEND, 1, reqs[k][2], bytes((7 * i + k) & 0xFF for i in range(ln)))
    with device_group(eng, n, L) as g:
        g.prologue()
        st = torch.cuda.Stream(device=g.leader.device)
        v = g.leader.submitter_attach(st)
        tickets = run_submitter(g, v, st, reqs, batch=32, ctas=ctas)
        assert sorted(tickets) == list(range(2, 2 + len(reqs)))
        assert g.leader.stats()["tickets_submitted"] == 1 + len(reqs)
        stream, _ = SB.ticket_order(reqs, tickets)
        rejected = [t for t, r in zip(tickets, reqs) if not SB.accepted(r)]
        assert {tickets[701], tickets[1500]} <= set(rejected) and tickets[700] not in rejected
        assert g.leader.device_submit_status() == (len(rejected), min(rejected))
        g.leader.submitter_detach()
        assert g.leader.device_submit_status() == (len(rejected), min(rejected))
        c = oracle_of(orc, n, L, stream)
        EU.compare_group_to_oracle(g, c, exact=True)
        assert g.leader.committed() == 1 + len(reqs)
        c.close()


@pytest.mark.parametrize("express", [True, False])
def test_submitter_laps_with_autoprune(eng, orc, express):
    """APUS_F_AUTOPRUNE over several laps of a 256 KiB log, a 2048-slot ring and a 128 KiB payload ring, with four
    submitting CTAs: every launch's entries replayed into the oracle (the leader's own HEAD entries included), every byte
    compared at the end"""
    import torch
    n, L = 3, 1 << 18
    flags = MODES["index_earlyack"] | E.F_AUTOPRUNE | (0 if express else E.F_NO_EXPRESS)
    reqs = SB.mixed_requests(7000, seed=77 if express else 78, max_len=300, reject_every=41, conns=3)
    step = 300                                          # ~ a quarter of the log per launch
    rp = AR.Replay(orc, n, L)
    try:
        with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=flags, leader_ctas=4, ring_mode=eng.RING_DEVICE,
                       ring_slots=1 << 11, ring_bytes=1 << 17) as g:
            g.prologue()
            st = torch.cuda.Stream(device=g.leader.device)
            v = g.leader.submitter_attach(st)
            ordered, prev, ext = [(O.CONFIG, 0, 0, b"")], 0, 0
            for k in range(0, len(reqs), step):
                part = reqs[k:k + step]
                tickets = run_submitter(g, v, st, part, batch=16, ctas=4)
                ordered += SB.ticket_order(part, tickets)[0]
                ext += sum(len(p) + 2 for t, _, _, p in SB.ticket_order(part, tickets)[0] if len(p) + 2 > 80)
                end = g.leader.offsets()["end"]
                rp.launch(AR.read_launch(g.leader, prev, end, L), ordered)
                prev = end
                check_heads(g.replicas, rp, f"after the launch ending at {end}")
            g.leader.submitter_detach()
            assert rp.pos == len(ordered)
            assert rp.written >= 4 * L and ext >= 4 * (1 << 17) and len(reqs) >= 3 * (1 << 11)
            EU.compare_group_to_oracle(g, rp.c, exact=True)
            assert g.leader.stats()["auto_heads"] == len(rp.heads) > 0
            assert g.leader.committed() == 1 + len(reqs)
    finally:
        rp.close()


def test_hand_over_to_and_from_the_host(eng, orc):
    """host apus_submit -> attach -> device submits -> detach -> apus_submit_device and apus_submit: contiguous
    tickets, and the log of all of them is the oracle's"""
    import torch
    n, L = 3, 1 << 22
    host1 = S.ragged_stream(200, 1500, conns=2, seed=61)
    dev = SB.mixed_requests(600, seed=62, first_req_id=5000)
    batch2 = S.ragged_stream(150, 900, conns=2, seed=63)
    host3 = S.ragged_stream(50, 1500, conns=2, seed=64)
    with device_group(eng, n, L) as g:
        g.prologue()
        submit_host(g, host1)
        assert g.tickets == 1 + len(host1)
        st = torch.cuda.Stream(device=g.leader.device)
        v = g.leader.submitter_attach(st)
        tickets = run_submitter(g, v, st, dev, batch=8, ctas=2)
        assert sorted(tickets) == list(range(2 + len(host1), 2 + len(host1) + len(dev)))
        g.leader.submitter_detach()
        t0 = g.submit_device(*tensors(batch2, g.leader.device))
        assert t0 == 2 + len(host1) + len(dev)
        for typ, conn, rid, p in host3:
            g.submit(typ, conn, rid, p)
        assert g.tickets == 1 + len(host1) + len(dev) + len(batch2) + len(host3)
        g.run()
        stream = host1 + SB.ticket_order(dev, tickets)[0] + batch2 + host3
        c = oracle_of(orc, n, L, stream)
        EU.compare_group_to_oracle(g, c, exact=True)
        c.close()


def test_dropped_reservation(eng, orc):
    """a reservation put but never published is dropped at detach: the next host ticket is P + 1, and the log holds
    the published requests, then the host's"""
    import torch
    n, L = 3, 1 << 22
    dev = SB.mixed_requests(40, seed=71, max_len=400, reject_every=0)
    host = S.ragged_stream(30, 1500, conns=2, seed=72)
    with device_group(eng, n, L) as g:
        g.prologue()
        st = torch.cuda.Stream(device=g.leader.device)
        v = g.leader.submitter_attach(st)
        sub = SB.Submitter(v, st, dev, batch=8, ctas=1, mode=SB.DROP_LAST).start()
        fail, pub, tickets = sub.result()
        assert fail is None and pub == 32
        assert g.leader.stats()["tickets_submitted"] == 33
        g.leader.submitter_detach()
        first = [g.leader.submit(typ, conn, rid, p) for typ, conn, rid, p in host][0]
        assert first == 34
        g.tickets = 33 + len(host)
        g.run()
        stream = SB.ticket_order(dev, tickets, upto=33)[0] + host
        c = oracle_of(orc, n, L, stream)
        EU.compare_group_to_oracle(g, c, exact=True)
        c.close()


def test_commit_waits_and_detach_ends_a_blocked_reserve(eng):
    """wait-committed ends OK at or past its ticket while the group runs, TIMED_OUT after apus_replicas_stop, and a
    reserve blocked on a full ring ends STOPPED when the submitter is detached"""
    import torch
    n, L = 3, 1 << 22
    with device_group(eng, n, L, ring_slots=1 << 11) as g:
        g.prologue()
        st = torch.cuda.Stream(device=g.leader.device)
        v = g.leader.submitter_attach(st)
        # every launch's arrays are made before the replica kernels are resident
        sub = SB.Submitter(v, st, SB.mixed_requests(64, seed=81, max_len=200, reject_every=0), batch=1, mode=SB.WAIT)
        one = SB.Submitter(v, st, SB.mixed_requests(1, seed=82, reject_every=0), batch=1, mode=SB.WAIT, timeout_s=0.05)
        many = SB.Submitter(v, st, SB.mixed_requests((1 << 11) + 256, seed=83, max_len=60, reject_every=0), batch=64,
                            timeout_s=60)
        g.launch(FOREVER)
        sub.start()
        fail, pub, tickets = sub.result()
        assert fail is None and pub == 64
        assert g.leader.committed() >= max(tickets) == 65
        lat = sub.latencies_ns()
        assert all(0 < x < 1_000_000_000 for x in lat), lat[:8]
        g.stop()
        one.start()
        assert one.result()[0] == (SB.STEP_WAIT, SB.TIMED_OUT)
        # the kernels are stopped: a submitter of more than the ring holds blocks in its reserve until detached
        many.start()
        t0 = time.time()
        while g.leader.stats()["tickets_submitted"] < (1 << 11) - 64 and time.time() - t0 < 30:
            time.sleep(0.01)
        time.sleep(0.2)
        t1 = time.time()
        g.leader.submitter_detach()
        assert time.time() - t1 < 5
        fail, pub, _ = many.result()
        assert fail == (SB.STEP_RESERVE, SB.STOPPED), fail
        assert g.leader.stats()["tickets_submitted"] == 66 + pub <= 65 + (1 << 11)


def test_refusals(eng):
    """a follower, a host-mapped ring, a second attach, a detach with nothing attached, set_role while attached and
    every call that writes the ring while attached (with nothing written); destroy with a submitter attached ends it"""
    import torch
    n, L = 3, 1 << 20
    lib = E.lib()
    with eng.Group(n, devices=devices_for(eng, n), log_size=L) as hm:
        with pytest.raises(E.ApusError, match="device submission ring"):
            hm.leader.submitter_attach()
        with pytest.raises(E.ApusError, match="follower"):
            hm.replicas[1].submitter_attach()
    g = device_group(eng, n, L)
    try:
        g.prologue()
        lead = g.leader
        with pytest.raises(E.ApusError, match="no resident submitter"):
            lead.submitter_detach()
        st = torch.cuda.Stream(device=lead.device)
        v = lead.submitter_attach(st)
        with pytest.raises(E.ApusError, match="attached already"):
            lead.submitter_attach(st)
        assert lib.apus_replica_set_role(lead.h, 0, 2) == E.APUS_ERROR
        assert b"detach first" in lib.apus_last_error()
        before = (lead.stats()["tickets_submitted"], lead.committed())
        assert before == (1, 0)
        a = (C.c_uint64 * 64)()
        p = C.addressof(a)
        t = C.byref(C.c_uint64())
        s = st.cuda_stream
        calls = {
            "apus_submit": (E.SEND, 1, 1, p, 4, t),
            "apus_submit_batch": (1, p, p, p, p, p, 8, t),
            "apus_submit_uniform": (1, E.SEND, 1, 1, 4, p, 4, t),
            "apus_submit_synth": (1, E.SEND, 1, 1, 4, 7, t),
            "apus_submit_device": (1, p, p, p, p, p, 8, s, t),
            "apus_submit_device_packed": (1, p, p, p, p, p, 8, s, t),
            "apus_submit_defer": (1,),
            "apus_submit_flush": (),
            "apus_submit_release": (1,),
            "apus_closed_loop": (1, 8, 1, 1, p),
        }
        for name, args in calls.items():
            assert getattr(lib, name)(lead.h, *args) == E.APUS_ERROR, name
            assert b"resident submitter is attached" in lib.apus_last_error(), (name, lib.apus_last_error())
        assert (lead.stats()["tickets_submitted"], lead.committed()) == before
        # destroy with a submitter attached: it is told to stop first; a launch blocked in its turn wait ends STOPPED
        sub = SB.Submitter(v, st, SB.mixed_requests(4, seed=91, reject_every=0), batch=1, mode=SB.WAIT,
                           timeout_s=60).start()
        time.sleep(0.1)
        t0 = time.time()
        g.close()
        assert time.time() - t0 < 10
        fail, _, _ = sub.result()
        assert fail == (SB.STEP_WAIT, SB.STOPPED), fail
    finally:
        g.close()


def test_whole_loop_on_the_device(eng):
    """APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE with the test submitter on the leader and resident_rows on every
    replica: every replica's rows are the same, in the same order, and equal the submitted stream in ticket order"""
    import torch
    n, L = 3, 1 << 22
    reqs = SB.mixed_requests(3000, seed=101, max_len=1200)
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES["index_earlyack"] | E.F_AUTOPRUNE | ANY,
                   ring_mode=eng.RING_DEVICE) as g:
        g.prologue()
        streams = [torch.cuda.Stream(device=r.device) for r in g.replicas]
        cons = [resident.Resident(r, s, stride=1200).start() for r, s in zip(g.replicas, streams)]
        st = torch.cuda.Stream(device=g.leader.device)
        v = g.leader.submitter_attach(st)
        tickets = run_submitter(g, v, st, reqs, batch=64, ctas=4)
        g.leader.submitter_detach()
        want = [r for r in SB.ticket_order(reqs, tickets)[0] if r[0] in SB.ACCEPTED]
        for c in cons:
            c.wait_rows(len(want))
        rows = []
        for c in cons:
            why, nrows, _ = c.detach()
            assert why == resident.END_STOP and nrows == len(want)
            rows.append(c.rows())
        for rr in rows[1:]:
            assert rr == rows[0]
        assert [(t, co, rq, p) for _, t, co, rq, p in rows[0]] == want
