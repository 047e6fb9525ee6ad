"""Device-side log pruning (APUS_F_AUTOPRUNE, the configuration bench.py measures and libapus_dare.so runs) byte for
byte against the CPU oracle.  Where an auto HEAD entry lands and what it carries depends on how far the followers had
applied, so the oracle replays the engine's own append sequence (tests/autoprune_replay.py): after every launch, which
stays under a third of a lap, the leader's new entries are read back, every HEAD entry is checked against the pruning
rule and appended to the oracle with the value it carries, the launch's bytes are compared, and at the end every byte
of every replica.  Marked gpu."""
import time

import numpy as np
import pytest

import autoprune_replay as AR
import engine_util as EU
import orc as O
import streams as S
from apus_b200 import engine as E
from engine_util import MODES, devices_for, eng, pin_and_wait, settle, submit_part, wrap_stream  # noqa: F401
from shadow import check_heads

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(240)]

FOREVER = EU.FOREVER


def check_final(g, rp):
    """every byte and offset of every replica against the replay, plus what compare_group_to_oracle leaves out"""
    EU.compare_group_to_oracle(g, rp.c, exact=True)
    check_heads(g.replicas, rp, "end")
    st = g.leader.stats()
    assert st["bytes_replicated"] == rp.c.bytes_replicated()
    assert st["auto_heads"] == len(rp.heads), (st["auto_heads"], len(rp.heads))
    assert len(rp.heads) >= int(rp.written / rp.L), (len(rp.heads), rp.written / rp.L)   # at least one per lap
    return st


def synth_stream(nreq, length, seed):
    return [(S.CONNECT, 0, 1, b"")] + [(S.SEND, 0, 2 + i, E.synth_payload(seed, 2 + i, length)) for i in range(nreq)]


def _case(n, L, kind, seed, mode, ctas, ring, id):
    return pytest.param(n, L, kind, seed, mode, ctas, ring, id=id)


LAP_CASES = [
    # the benchmark's own shape: 5 replicas, 64 B payloads written by the fill kernel into the HBM ring, 16 leader CTAs,
    # claims of 512 slots
    _case(5, 4 << 20, "synth64", 0xA070, "index_earlyack", 16, "synth", "bench-shape-n5-4M-synth-ctas16"),
    # stride 1024 from the HBM ring: the holes-only prefill, with the HEAD entry at j == 0; walking followers
    _case(5, 1 << 18, "u960", 95, "walk_fenced", 16, "device", "u960-n5-256K-walk_fenced-ctas16-device"),
    # stride 264: the full-sweep prefill, payloads staged as external images
    _case(3, 1 << 16, "u200", 96, "index_fenced", 4, "host", "u200-n3-64K-index_fenced-ctas4"),
    # 0..1500 B with connection churn on the drop-in's two CTAs: ghost headers, wraps, both prefills
    _case(3, 1 << 18, "ragged1500", 97, "walk_earlyack", 2, "host", "ragged1500-n3-256K-walk_earlyack-ctas2"),
]


@pytest.mark.parametrize("n,L,kind,seed,mode,ctas,ring", LAP_CASES)
def test_autoprune_laps_replayed(eng, orc, n, L, kind, seed, mode, ctas, ring):
    """4.5+ laps with the leader pruning on its own; every HEAD it appended checked and replayed, every byte compared"""
    if kind == "synth64":
        stream = synth_stream(int(4.6 * L / 128), 64, seed)
    elif kind == "ragged1500":                      # wrap_stream's shape, long enough for 4.5 laps
        stream = S.ragged_stream(int(4.8 * L / 814) + 1, 1500, conns=3, seed=seed, close_every=20)
    else:
        stream = wrap_stream(kind, seed, L)
    requests = [(O.CONFIG, 0, 0, b"")] + stream
    step = max(1, int(0.3 * L * len(stream) / S.stream_bytes(stream)))
    dev = dict(ring_mode=eng.RING_DEVICE, ring_slots=1 << 16, ring_bytes=8 << 20) if ring != "host" else {}
    rp = AR.Replay(orc, n, L)
    t_start = time.time()
    try:
        with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES[mode] | E.F_AUTOPRUNE, leader_ctas=ctas,
                       **dev) as g:
            g.prologue()
            prev = 0
            for k in range(0, len(stream), step):
                part = stream[k:k + step]
                if ring == "synth":
                    j = 0
                    if part[0][0] == S.CONNECT:
                        g.submit(*part[0])
                        j = 1
                    if j < len(part):
                        t0 = g.leader.submit_synth(len(part) - j, S.SEND, 0, part[j][2], 64, seed)
                        g.tickets = t0 + len(part) - j - 1
                else:
                    submit_part(g, part, ring == "device")
                g.run(timeout_ms=60_000)
                end = g.leader.offsets()["end"]
                rp.launch(AR.read_launch(g.leader, prev, end, L), requests)
                prev = end
                check_heads(g.replicas, rp, f"after the launch ending at {end}")
            assert rp.pos == len(requests)
            assert rp.written >= 4.5 * L
            st = check_final(g, rp)
            last = AR.parse_entries(rp.c.image(0), rp.c.offsets(0)["tail"], rp.c.offsets(0)["end"], L)[-1]
            assert last.idx == g.tickets + st["auto_heads"]
            assert g.leader.committed() == g.tickets
            teeth = AR.assert_heads_have_teeth(rp, rp.c.image(0))
            print(f"{len(rp.heads)} HEAD entries replayed over {rp.written / L:.2f} laps, {teeth} over earlier laps "
                  f"with non-zero holes, {time.time() - t_start:.1f} s")
    finally:
        rp.close()


def test_autoprune_head_is_the_lagging_application(eng, orc):
    """Followers whose host replays the log (APUS_F_HOST_APPLY) report pinned apply offsets: follower 1 the end of
    launch k-2, the others the end of launch k-1.  Every auto HEAD must carry exactly follower 1's offset.  Then a
    launch that needs more room than follower 1 leaves: the leader holds (rule E2) without touching what follower 1
    has not applied, and once the offsets are raised it prunes to the released value and completes."""
    n, L = 3, 1 << 18
    stream = wrap_stream("u200", 98, L)
    requests = [(O.CONFIG, 0, 0, b"")] + stream
    step = int(0.3 * L / 264)
    reps = EU.host_apply_replicas(eng, n, L, 0, eng.RING_HOST_MAPPED, 1 << 14, 4 << 20)
    lead = reps[0]

    class G:                                   # what EU.compare_group_to_oracle and settle() need of a Group
        replicas, leader_idx, leader = reps, 0, lead

    rp = AR.Replay(orc, n, L)
    try:
        EU.launch_each(eng, reps, FOREVER)
        ends = [0, 0]                          # leader's end after each launch (two zeros: before the first)
        t = 0
        pos = 0
        for k in range(12):
            pins = [0, ends[-2]] + [ends[-1]] * (n - 2)
            pin_and_wait(lead, reps, pins)
            part = requests[pos:pos + step]
            pos += len(part)
            lead.defer(True)
            for typ, clt, rid, payload in part:
                t = lead.submit(typ, clt, rid, payload) if typ != O.CONFIG else lead.submit(E.CONFIG, 0, 0, E.cid_image(n))
            lead.flush()
            lead.defer(False)
            lead.wait_committed(t, 10_000_000)
            settle(G, t)
            end = lead.offsets()["end"]
            lc = AR.read_launch(lead, ends[-1], end, L)
            rp.launch(lc, requests)
            heads = [e.value for e in lc.entries if e.typ == O.HEAD]
            assert all(v == pins[1] for v in heads), f"launch {k}: HEAD entries carry {heads}, follower 1 pinned {pins[1]}"
            check_heads(reps, rp, f"launch {k}")
            ends.append(end)
        assert len(rp.heads) >= 8, len(rp.heads)

        # ---- a launch that needs more room than follower 1 allows: back-pressure, then release
        pins = [0, ends[-2]] + [ends[-1]] * (n - 2)
        pin_and_wait(lead, reps, pins)
        kept = [r.read_range(pins[1], ends[-1], cap=L) for r in reps]     # follower 1 has not applied these
        part = requests[pos:pos + int(0.85 * L / 264)]
        pos += len(part)
        lead.defer(True)
        for typ, clt, rid, payload in part:
            t = lead.submit(typ, clt, rid, payload)
        lead.flush()
        lead.defer(False)
        t0, last, still = time.time(), -1, time.time()
        while time.time() - still < 0.3:                                   # committed() stopped moving
            assert time.time() - t0 < 5.0, "the leader kept committing: no back-pressure"
            c = lead.committed()
            if c != last:
                last, still = c, time.time()
            time.sleep(0.01)
        assert last < t, (last, t)
        time.sleep(0.5)                                                    # held, well below the kernels' watchdog
        assert lead.committed() == last
        for i, r in enumerate(reps):
            assert np.array_equal(r.read_range(pins[1], ends[-1], cap=L), kept[i]), \
                f"replica {i}: bytes follower 1 had not applied were overwritten while blocked"
        release = ends[-1]
        pin_and_wait(lead, reps, [0] + [release] * (n - 1))
        lead.wait_committed(t, 10_000_000)
        settle(G, t)
        end = lead.offsets()["end"]
        lc = AR.read_launch(lead, ends[-1], end, L)
        rp.launch(lc, requests)             # two HEADs in a row only where the placement blocked between them
        heads = [e.value for e in lc.entries if e.typ == O.HEAD]
        assert heads == [pins[1], release], (heads, pins[1], release)
        check_heads(reps, rp, "after the release")
        EU.stop_each(eng, reps)

        # everything against the replay; followers' apply is what their host reported
        for i, r in enumerate(reps):
            eo, oo = r.offsets(), rp.c.offsets(i)
            for key in ("end", "commit", "head"):
                assert eo[key] == oo[key], (i, key, eo, oo)
            assert eo["apply"] == (oo["apply"] if i == 0 else release), (i, eo)
            ei, oi = r.image(), rp.c.image(i)
            d = np.nonzero(ei != oi)[0]
            assert len(d) == 0, f"replica {i}: {len(d)} bytes differ, first at {int(d[0])}"
        assert lead.stats()["auto_heads"] == len(rp.heads)
        print(f"{len(rp.heads)} HEAD entries replayed over {rp.written / L:.2f} laps")
    finally:
        EU.stop_each(eng, reps)
        for r in reps:
            r.close()
        rp.close()


def test_express_closed_loop_with_autoprune(eng, orc):
    """One request in flight on resident kernels around a 64 KiB ring: the express path takes the requests until the
    ring is half used, the tile machine prunes and hands back.  Every chunk of ~50 requests is read back and replayed."""
    n, L = 3, 1 << 16
    stream = S.ragged_stream(int(4.6 * L / 103), 78, conns=3, seed=99, close_every=90)
    requests = [(O.CONFIG, 0, 0, b"")] + stream
    rp = AR.Replay(orc, n, L)
    try:
        with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=E.F_DEVICE_STATS | E.F_AUTOPRUNE) as g:
            g.launch(target=FOREVER)
            t = g.prologue()
            g.leader.wait_committed(t)
            prev = 0
            for k in range(0, len(stream), 50):
                for typ, clt, rid, payload in stream[k:k + 50]:
                    t = g.submit(typ, clt, rid, payload)
                    g.leader.wait_committed(t, 5_000_000)
                settle(g, t)
                end = g.leader.offsets()["end"]
                rp.launch(AR.read_launch(g.leader, prev, end, L), requests)
                prev = end
            st = g.leader.stats()
            g.stop()
            assert rp.pos == len(requests)
            assert rp.written >= 4 * L
            check_final(g, rp)
            assert st["turn_ns"][5] > 0, st["turn_ns"]
            assert st["auto_heads"] > 0
            print(f"{len(rp.heads)} HEAD entries replayed over {rp.written / L:.2f} laps, express {st['turn_ns'][5]}")
    finally:
        rp.close()
