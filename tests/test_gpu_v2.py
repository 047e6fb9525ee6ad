"""GPU parity, round 2: the express path (single warp, self-certifying publishes), device-generated and bulk
submission, the BASELINE config shapes that were missing (7 x 1 KiB, 5 x Redis-sized), follower apply semantics
under a slow host, abort during back-pressure, heartbeats and the term fence.  Bit-exact against the oracle
wherever the oracle can follow; through the C ABI; marked gpu.  Replicas are spread over every GPU the box has
(tests/test_gpu_parity.py: devices_for), so on a multi-GPU box every "peer" store crosses NVLink."""
import hashlib
import threading
import time

import numpy as np
import pytest

import engine_util as EU
import orc as O
import streams as S
from apus_b200 import engine as E
from engine_util import MODES, devices_for, eng, prune_both, settle  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(240)]

FOREVER = EU.FOREVER


def closed_loop(g, stream, timeout_us=5_000_000):
    t = 0
    for typ, clt, rid, payload in stream:
        t = g.submit(typ, clt, rid, payload)
        g.leader.wait_committed(t, timeout_us)
    return t


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("n", [3, 5])
def test_express_closed_loop_exact(eng, orc, n, mode):
    """One request in flight at a time on resident kernels: every entry takes the single-warp express path and
    reaches the followers under a self-certifying publish (no writer fence).  Every byte of every replica must
    still equal the oracle's -- reply bytes included."""
    L = 1 << 20
    stream = S.ragged_stream(700, 78, conns=3, seed=100 + n, close_every=90)
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES[mode]) as g:
        g.launch(target=FOREVER)
        t = g.prologue()
        g.leader.wait_committed(t)
        t = closed_loop(g, stream)
        settle(g, t)
        st = g.leader.stats()
        g.stop()
        c = EU.oracle_cluster(orc, n, L, stream)
        try:
            EU.compare_group_to_oracle(g, c, exact=True)
        finally:
            c.close()
        # the express counter (turn_ns[5]) says the path under test actually ran
        assert st["turn_ns"][5] >= len(stream) // 2, st["turn_ns"]


def test_express_off_is_the_same_log(eng, orc):
    """A/B: APUS_F_NO_EXPRESS (every publish fenced, tile machine only) leaves the identical image."""
    n, L = 3, 1 << 20
    stream = S.ragged_stream(300, 78, conns=2, seed=7)
    imgs = []
    for flags in (E.F_DEVICE_STATS, E.F_DEVICE_STATS | E.F_NO_EXPRESS):
        with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=flags) as g:
            g.launch(target=FOREVER)
            g.leader.wait_committed(g.prologue())
            t = closed_loop(g, stream)
            settle(g, t)
            st = g.leader.stats()
            g.stop()
            imgs.append([hashlib.sha256(r.image().tobytes()).hexdigest() for r in g.replicas])
            if flags & E.F_NO_EXPRESS:
                assert st["turn_ns"][5] == 0
    assert imgs[0] == imgs[1]


def test_express_across_wraps_with_pruning(eng, orc):
    """Closed loop around a small ring: the express path hands wraps, ghost headers and exact fits to the tile
    machine and takes over again behind them; HEAD entries are submitted at quiescent points on both sides."""
    n, L = 3, 16384
    stream = S.ragged_stream(1500, 78, conns=3, seed=41)
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, n, leader=0, term=1, length=L)
    c.prologue()
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=E.F_DEVICE_STATS) as g:
        g.launch(target=FOREVER)
        total = g.prologue()
        g.leader.wait_committed(total)
        step = 10
        for k in range(0, len(stream), step):
            part = stream[k:k + step]
            for typ, clt, rid, payload in part:
                assert c.submit(typ, clt, rid, O.cmd_image(payload)) != 0
            c.round(); c.round()
            total = closed_loop(g, part)
            settle(g, total)
            if prune_both(g, c):
                total += 1
                c.round(); c.round()
                g.leader.wait_committed(total, 5_000_000)
                settle(g, total)
        st = g.leader.stats()
        g.stop()
        EU.compare_group_to_oracle(g, c, exact=True)
        assert c.offsets(0)["head"] != 0
        assert st["turn_ns"][5] > 500
    c.close()


@pytest.mark.parametrize("n,payload,nreq", [(7, 1024, 6000), (5, 175, 20000), (3, 64, 50000)])
def test_config_shapes_exact(eng, orc, n, payload, nreq):
    """BASELINE config 4 shape (7 replicas x 1 KiB), config 3 shape (5 replicas, a Redis SET of a 128 B value is
    ~175 B on the wire) and config 1/2 shape, through the bulk submission call, byte for byte."""
    L = O.LOG_SIZE
    rng = np.random.default_rng(payload)
    pl = rng.integers(0, 256, size=nreq * payload, dtype=np.uint8)
    pb = pl.tobytes()
    stream = [(S.CONNECT, 0, 1, b"")] + [(S.SEND, 0, 2 + i, pb[i * payload:(i + 1) * payload]) for i in range(nreq)]
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, ring_mode=eng.RING_DEVICE, ring_slots=1 << 17,
                   ring_bytes=(nreq * ((payload + 2 + 15) // 16 * 16) + (1 << 20)) // 4096 * 4096) as g:
        g.prologue()
        g.submit(S.CONNECT, 0, 1, b"")
        t0 = g.leader.submit_uniform(nreq, S.SEND, 0, 2, payload, pl)
        g.tickets = t0 + nreq - 1
        g.run(timeout_ms=120_000)
        c = EU.oracle_cluster(orc, n, L, stream)
        try:
            EU.compare_group_to_oracle(g, c, exact=True)
            assert g.leader.stats()["bytes_replicated"] == c.bytes_replicated()
        finally:
            c.close()


@pytest.mark.parametrize("payload", [64, 1000])
def test_device_generated_requests_exact(eng, orc, payload):
    """apus_submit_synth: the fill kernel writes the requests straight into the HBM ring; the log must be what the
    same requests give when the host submits them (payload bytes recomputed on the host with numpy)."""
    n, L, nreq, seed = 5, O.LOG_SIZE, 5000, 0xC0FFEE
    stream = [(S.CONNECT, 0, 1, b"")] + [(S.SEND, 0, 2 + i, E.synth_payload(seed, 2 + i, payload)) for i in range(nreq)]
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, ring_mode=eng.RING_DEVICE, ring_slots=1 << 14,
                   ring_bytes=8 << 20) as g:
        g.prologue()
        g.submit(S.CONNECT, 0, 1, b"")
        t0 = g.leader.submit_synth(nreq, S.SEND, 0, 2, payload, seed)
        g.tickets = t0 + nreq - 1
        g.run(timeout_ms=60_000)
        c = EU.oracle_cluster(orc, n, L, stream)
        try:
            EU.compare_group_to_oracle(g, c, exact=True)
        finally:
            c.close()
        for k in (0, 1, 63, 64, 999):
            if k < payload:
                assert eng.lib().apus_synth_byte(seed, 77, k) == E.synth_payload(seed, 77, payload)[k]


def _replay_thread(r, L, expect, sink, stop, delay_s):
    try:
        _replay(r, L, expect, sink, stop, delay_s)
    except Exception as ex:                                  # noqa: BLE001 - surfaced by the test
        sink["error"] = f"{type(ex).__name__}: {ex}"


def _replay(r, L, expect, sink, stop, delay_s):
    """What follower_pump of libapus_dare.so does: read the committed range, walk it, 'apply', report the offset."""
    apply, next_idx = 0, 0
    h = hashlib.sha256()
    count = 0
    while not stop.is_set():
        off, _ = r.progress()
        if off == apply:
            time.sleep(0.0002)
            continue
        buf = r.read_range(apply, off, cap=1 << 20)
        o, p = apply, 0
        while p < len(buf):
            if L - o < 64:
                p += L - o; o = 0
                continue
            if len(buf) - p < 64:
                break
            typ = int(buf[p + 26])
            ln = int(buf[p + 48]) | (int(buf[p + 49]) << 8)
            stride = 64 if typ in (0, 2, 3) else 64 + ln
            if L - o < stride:
                p += L - o; o = 0
                continue
            if len(buf) - p < stride:
                break
            idx = int.from_bytes(buf[p:p + 8].tobytes(), "little")
            if next_idx and idx != next_idx:
                sink["error"] = (f"expected idx {next_idx}, found {idx} at {o}; batch [{apply}, {off}) of {len(buf)} bytes, p={p}; "
                                 f"follower offsets {r.offsets()}")
                return
            next_idx = idx + 1
            if typ == S.SEND:
                h.update(buf[p + 50:p + 50 + ln].tobytes())
                count += 1
            p += stride; o += stride
            if o == L:
                o = 0
        apply = o
        time.sleep(delay_s)                       # a slow application
        r.set_applied(apply)
        if count >= expect:
            break
    sink["sha"], sink["count"] = h.hexdigest(), count


def test_slow_follower_host_apply_many_laps(eng):
    """Followers whose HOST replays the log slowly (APUS_F_HOST_APPLY): the apply offset they report is the replayed
    one, the leader's pruning rule never lets the ring overwrite entries that were not replayed (it back-pressures
    instead), and after 10+ laps around a 1 MiB ring every follower has replayed exactly the submitted stream."""
    n, L, payload, per, rounds = 3, 1 << 20, 200, 10000, 5
    flags_l = E.F_DEVICE_STATS | E.F_AUTOPRUNE
    flags_f = E.F_DEVICE_STATS | E.F_AUTOPRUNE | E.F_HOST_APPLY
    devs = devices_for(eng, n)
    reps = [E.Replica(devs[i], i, n, 0, 1, L, eng.RING_HOST_MAPPED, 1 << 16, 16 << 20, flags_l if i == 0 else flags_f, 4)
            for i in range(n)]
    EU.connected(reps)
    import ctypes as C
    try:
        for dev in sorted(set(devs), key=lambda d: any(r.is_leader and r.device == d for r in reps)):
            rs = [r for r in reps if r.device == dev]
            arr = (C.c_void_p * len(rs))(*[r.h for r in rs])
            E._ck(eng.lib().apus_replicas_launch(arr, len(rs), FOREVER), "launch")
        rng = np.random.default_rng(9)
        expect_h = hashlib.sha256()
        total_req = per * rounds
        stop = threading.Event()
        sinks = [dict() for _ in range(n)]
        ths = [threading.Thread(target=_replay_thread, args=(reps[i], L, total_req, sinks[i], stop, 0.002 * i), daemon=True)
               for i in range(1, n)]
        for t in ths:
            t.start()
        lead = reps[0]
        lead.wait_committed(lead.submit(E.CONFIG, 0, 0, E.cid_image(n)))
        t = lead.submit(S.CONNECT, 0, 1, b"")
        req = 2
        for _ in range(rounds):
            pl = rng.integers(0, 256, size=per * payload, dtype=np.uint8)
            expect_h.update(pl.tobytes())
            done = 0
            while done < per:                      # the ring (64 Ki slots) is smaller than a round: feed it as it drains
                k = min(4096, per - done)
                try:
                    t0 = lead.submit_uniform(k, S.SEND, 0, req, payload, pl[done * payload:(done + k) * payload])
                except BlockingIOError:
                    time.sleep(0.001)
                    continue
                t = t0 + k - 1
                req += k; done += k
        t_end = time.time() + 150
        while lead.committed() < t:
            assert time.time() < t_end, f"stuck: committed {lead.committed()} of {t}; sinks {sinks}; leader {lead.offsets()} {lead.stats()}"
            if any("error" in s_ for s_ in sinks):
                raise AssertionError(f"{sinks}\nleader offsets {lead.offsets()}\nleader's view of the apply offsets "
                                     f"{lead.remote_apply_offsets()[:n]}\nleader stats {lead.stats()}")
            time.sleep(0.01)
        for th in ths:
            th.join(timeout=60)
        stop.set()
        st = lead.stats()
        assert (total_req * (64 + payload)) / L > 10          # laps
        assert st["auto_heads"] > 0
        for i in range(1, n):
            assert "error" not in sinks[i], sinks[i]
            assert sinks[i].get("count") == total_req, (i, sinks[i])
            assert sinks[i]["sha"] == expect_h.hexdigest(), f"follower {i} replayed something else"
    finally:
        arr = (C.c_void_p * n)(*[r.h for r in reps])
        eng.lib().apus_replicas_stop(arr, n)
        for r in reps:
            r.close()


def test_stop_while_blocked_on_a_full_log(eng):
    """ADVICE (medium): stop arrives while leader workers wait for free space / for their turns.  Nothing may be
    placed, stored or published with a stale placement: what the replicas hold afterwards is a clean common prefix."""
    n, L, payload = 3, 1 << 18, 200
    # followers never report an applied offset (HOST_APPLY with a host that replays nothing): head cannot move
    devs = devices_for(eng, n)
    flags = E.F_DEVICE_STATS | E.F_AUTOPRUNE
    reps = [E.Replica(devs[i], i, n, 0, 1, L, eng.RING_HOST_MAPPED, 1 << 14, 4 << 20,
                      flags if i == 0 else flags | E.F_HOST_APPLY, 4) for i in range(n)]
    EU.connected(reps)
    import ctypes as C
    try:
        for dev in sorted(set(devs), key=lambda d: any(r.is_leader and r.device == d for r in reps)):
            rs = [r for r in reps if r.device == dev]
            arr = (C.c_void_p * len(rs))(*[r.h for r in rs])
            E._ck(eng.lib().apus_replicas_launch(arr, len(rs), FOREVER), "launch")
        lead = reps[0]
        lead.submit(E.CONFIG, 0, 0, E.cid_image(n))
        lead.submit(S.CONNECT, 0, 1, b"")
        nreq = 3 * L // (64 + payload)                      # three rings' worth: must block
        pl = np.random.default_rng(1).integers(0, 256, size=4096 * payload, dtype=np.uint8)
        sent, req = 0, 2
        t_end = time.time() + 3.0
        while sent < nreq and time.time() < t_end:
            try:
                lead.submit_uniform(4096, S.SEND, 0, req, payload, pl)
                req += 4096; sent += 4096
            except BlockingIOError:
                time.sleep(0.01)
        time.sleep(0.2)
        committed_before = lead.committed()
        assert committed_before < sent + 2                  # it did block
    finally:
        arr = (C.c_void_p * n)(*[r.h for r in reps])
        rc = eng.lib().apus_replicas_stop(arr, n)
    try:
        assert rc in (0, 1)
        lo = reps[0].offsets()
        limg = reps[0].image()
        # the committed prefix [head, commit) parses cleanly with consecutive idx on the leader, and every follower
        # holds the same bytes for the part it has
        ents = O.walk_entries(limg, lo["head"], lo["commit"], L)
        idx = [int.from_bytes(limg[o:o + 8].tobytes(), "little") for o, _ in ents]
        assert idx == list(range(idx[0], idx[0] + len(idx)))
        lm = O.mask_replies(limg, ents)
        for i in range(1, n):
            fo = reps[i].offsets()
            fimg = O.mask_replies(reps[i].image(), ents)
            fents = O.walk_entries(fimg, lo["head"], fo["commit"], L) if fo["commit"] != lo["head"] else []
            for o, stride in fents:
                assert np.array_equal(fimg[o:o + stride], lm[o:o + stride]), (i, o)
    finally:
        for r in reps:
            r.close()


def test_heartbeats_and_failure_detector(eng):
    """The leader's commit warp beats into every follower (dare_ibv_rc.c:868-958); a follower whose leader kernel
    is gone reports the suspicion within its timeout, not before."""
    n, L = 3, 1 << 20
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=E.F_DEVICE_STATS, hb_period_us=100,
                   hb_timeout_us=20_000) as g:
        EU.launch_each(eng, g.replicas)
        g.leader.wait_committed(g.prologue())
        time.sleep(0.15)                                    # many timeouts' worth of beats
        for r in g.replicas[1:]:
            assert r.leader_suspect() == 0
        import ctypes as C
        arr = (C.c_void_p * 1)(g.leader.h)
        eng.lib().apus_replicas_stop(arr, 1)                # the leader's kernel goes away, followers stay
        t0 = time.time()
        while time.time() - t0 < 2.0 and any(r.leader_suspect() == 0 for r in g.replicas[1:]):
            time.sleep(0.001)
        dt = time.time() - t0
        for r in g.replicas[1:]:
            assert r.leader_suspect() == 1 + 1              # 1 + term
        assert dt < 0.5, dt


def test_term_fence_ignores_a_deposed_leader(eng, orc):
    """A follower that has moved to term 2 does not look at publishes stamped with term 1 (SURVEY H2, software form):
    it acks nothing and its `end` does not move, while the term-1 majority (leader + the other follower) commits."""
    import ctypes as C
    n, L = 3, 1 << 20
    devs = devices_for(eng, n)
    reps = [E.Replica(devs[i], i, n, 0, 2 if i == 2 else 1, L, eng.RING_HOST_MAPPED, 0, 0, E.F_DEVICE_STATS, 2)
            for i in range(n)]
    EU.connected(reps)
    try:
        for dev in sorted(set(devs), key=lambda d: any(r.is_leader and r.device == d for r in reps)):
            rs = [r for r in reps if r.device == dev]
            arr = (C.c_void_p * len(rs))(*[r.h for r in rs])
            E._ck(eng.lib().apus_replicas_launch(arr, len(rs), FOREVER), "launch")
        lead = reps[0]
        stream = S.ragged_stream(200, 100, conns=2, seed=3)
        fenced0 = reps[2].offsets()
        t = lead.submit(E.CONFIG, 0, 0, E.cid_image(n))
        for typ, clt, rid, payload in stream:
            t = lead.submit(typ, clt, rid, payload)
        lead.wait_committed(t, 10_000_000)
        time.sleep(0.05)
        assert reps[1].stats()["entries_acked"] == t
        assert reps[2].stats()["entries_acked"] == 0
        fo = reps[2].offsets()
        assert fo["end"] == L                               # still the empty-log sentinel
        # the deposed leader's commit offsets are fenced off too: the follower's commit and apply stay where they were
        assert (fo["commit"], fo["apply"]) == (fenced0["commit"], fenced0["apply"]), (fenced0, fo)
        assert reps[1].offsets()["commit"] == lead.offsets()["commit"]
    finally:
        arr = (C.c_void_p * n)(*[r.h for r in reps])
        eng.lib().apus_replicas_stop(arr, n)
        for r in reps:
            r.close()


@pytest.mark.parametrize("n,payload", [(2, 64), (2, 1000), (3, 64), (5, 1000)])
def test_multicast_replication_exact(eng, orc, n, payload):
    """Fabric mode: the replicas' regions are VMM allocations bound to an NVSwitch multicast object; the leader's T5 step
    (and the express push) issue ONE multimem.st per 16 B chunk and the switch fans it out.  Same bytes everywhere."""
    nd = eng.lib().apus_device_count()
    if nd < n:
        pytest.skip(f"needs {n} GPUs (one per replica), {nd} visible")
    L = 1 << 26                           # no pruning flag here: the whole stream (21 MB at 1000 B) has to fit
    nreq = 20000
    rng = np.random.default_rng(payload)
    pl = rng.integers(0, 256, size=nreq * payload, dtype=np.uint8)
    pb = pl.tobytes()
    stream = [(S.CONNECT, 0, 1, b"")] + [(S.SEND, 0, 2 + i, pb[i * payload:(i + 1) * payload]) for i in range(nreq)]
    with eng.Group(n, devices=list(range(n)), log_size=L, ring_mode=eng.RING_DEVICE, ring_slots=1 << 16,
                   ring_bytes=64 << 20, flags=E.F_DEVICE_STATS | E.F_FABRIC) as g:
        try:
            g.multicast()
        except E.ApusError as ex:
            pytest.skip(f"multicast unavailable: {ex}")
        g.prologue()
        g.submit(S.CONNECT, 0, 1, b"")
        t0 = g.leader.submit_uniform(nreq, S.SEND, 0, 2, payload, pl)
        g.tickets = t0 + nreq - 1
        g.run(timeout_ms=120_000)
        c = EU.oracle_cluster(orc, n, L, stream)
        try:
            EU.compare_group_to_oracle(g, c, exact=True)
        finally:
            c.close()
