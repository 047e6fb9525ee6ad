"""GPU parity: the CUDA engine (through the C ABI) against the CPU oracle and the
golden vectors.  Bit-exact: integer/byte work, no tolerance.  Marked gpu."""
import json
import os
import hashlib

import numpy as np
import pytest

import engine_util as EU
import orc as O
import streams as S
from engine_util import MODES, devices_for, eng, prune_both, wrap_case  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(180)]


def run_and_compare(eng, orc, n, L, stream, ring_mode=0, prologue=True, exact=True, devices=None, chunks=1,
                    mode="index_earlyack"):
    devices = devices or devices_for(eng, n)
    with eng.Group(n, devices=devices, log_size=L, ring_mode=ring_mode, flags=MODES[mode]) as g:
        if prologue:
            g.prologue()
        per = (len(stream) + chunks - 1) // chunks
        for k in range(chunks):                       # several launches: state carries over
            g.submit_stream(stream[k * per:(k + 1) * per])
            g.run()
        c = EU.oracle_cluster(orc, n, L, stream, prologue=prologue)
        try:
            eo, oo = EU.compare_group_to_oracle(g, c, exact=exact)
            st = g.leader.stats()
            total = len(stream) + (1 if (prologue and n > 1) else 0)
            assert st["tickets_committed"] == total == st["tickets_consumed"]
            assert g.leader.committed() == total
            # bytes accounted for the roofline = (N-1) * log bytes of the stream
            assert st["bytes_replicated"] == c.bytes_replicated()
            for i, r in enumerate(g.replicas):
                if i != g.leader_idx:
                    assert r.stats()["entries_acked"] == total
        finally:
            c.close()


def test_one_replica_degenerate(eng, orc):
    """group_size 1: no CONFIG prologue, the leader's own vote is the majority
    (dare_server.c:416-424)."""
    run_and_compare(eng, orc, 1, 1 << 20, S.uniform_stream(2000, 64), prologue=False)


@pytest.mark.parametrize("n", [3, 5, 7])
def test_uniform_64B(eng, orc, n):
    run_and_compare(eng, orc, n, 1 << 21, S.uniform_stream(6000, 64, conns=4))


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("n,seed", [(3, 11), (5, 12), (7, 13), (13, 14)])
def test_ragged_lengths(eng, orc, n, seed, mode):
    """0-length, odd and unaligned payloads: entries start at arbitrary byte offsets (H1)."""
    run_and_compare(eng, orc, n, 1 << 21, S.ragged_stream(3000, 300, conns=5, seed=seed, close_every=70), mode=mode)


def test_device_ring_mode(eng, orc):
    run_and_compare(eng, orc, 5, 1 << 21, S.ragged_stream(2500, 500, seed=21), ring_mode=1)


def test_multiple_launches_carry_state(eng, orc):
    run_and_compare(eng, orc, 3, 1 << 21, S.ragged_stream(2000, 128, seed=22), chunks=5)


@pytest.mark.parametrize("mode", ["index_earlyack", "walk_fenced"])
def test_large_payloads(eng, orc, mode):
    stream = [(S.CONNECT, 1, 1, b"")] + [(S.SEND, 1, 2 + i, bytes([(i * 7 + k) & 0xFF for k in range(256)]) * 16)
                                          for i in range(40)]
    stream += [(S.SEND, 1, 100 + i, np.random.default_rng(i).integers(0, 256, 65535, dtype=np.uint8).tobytes())
               for i in range(6)]
    stream += [(S.SEND, 1, 200, b""), (S.CLOSE, 1, 201, b"")]
    run_and_compare(eng, orc, 3, 1 << 21, stream, mode=mode)


def test_payload_ring_wraps(eng, orc):
    """External payload images wrap the (small) payload byte ring several times inside one run."""
    rng = np.random.default_rng(3)
    stream = [(S.CONNECT, 7, 1, b"")]
    for i in range(600):
        ln = int(rng.integers(100, 3000))
        stream.append((S.SEND, 7, 2 + i, rng.integers(0, 256, ln, dtype=np.uint8).tobytes()))
    n, L = 3, 1 << 21
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, ring_slots=1 << 16, ring_bytes=1 << 17) as g:
        g.launch(target=(1 << 64) - 1)          # resident: the ring drains while we submit
        g.prologue()
        for typ, clt, rid, payload in stream:
            while True:
                try:
                    t = g.submit(typ, clt, rid, payload)
                    break
                except BlockingIOError:
                    pass
        g.leader.wait_committed(t, 20_000_000)
        g.stop()
        c = EU.oracle_cluster(orc, n, L, stream)
        lo = g.leader.offsets()
        assert lo["end"] == c.offsets(0)["end"]
        ents = O.walk_entries(c.image(0), 0, lo["end"], L)
        assert np.array_equal(O.mask_replies(g.leader.image(), ents), O.mask_replies(c.image(0), ents))
        c.close()


def test_default_log_size_64MiB(eng, orc):
    """The reference's LOG_SIZE (dare_log.h:76), 4 KiB requests."""
    run_and_compare(eng, orc, 3, 0 or O.LOG_SIZE, S.uniform_stream(3000, 4096, conns=2))


def test_full_size_parity_run_2pow18_x_64B(eng, orc):
    """The parity run of SURVEY.md s8d at full size: 2^18 requests of 64 B behind the CONFIG prologue,
    32 MiB of the reference's 64 MiB ring at 5 replicas, every byte of every replica against the oracle."""
    n, L = 5, O.LOG_SIZE
    nreq = 1 << 18
    rng = np.random.default_rng(0xA5A50040)
    payloads = rng.integers(0, 256, size=nreq * 64, dtype=np.uint8)
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, n, leader=0, term=1, length=L)
    c.prologue()
    c.submit(S.CONNECT, 0, 1, O.cmd_image(b""))
    pb = payloads.tobytes()
    for i in range(nreq):
        assert c.submit(S.SEND, 0, 2 + i, O.cmd_image(pb[64 * i:64 * i + 64]))
        if i % 4096 == 4095:
            c.round()
    c.round(); c.round()
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, ring_mode=eng.RING_DEVICE, ring_slots=1 << 19,
                   ring_bytes=1 << 20) as g:
        g.prologue()
        g.submit(S.CONNECT, 0, 1, b"")
        g.submit_uniform(nreq, 64, 0, 2, payloads)
        g.run(timeout_ms=120_000)
        EU.compare_group_to_oracle(g, c, exact=True)
        assert g.leader.committed() == nreq + 2
        assert g.leader.stats()["bytes_replicated"] == c.bytes_replicated() == (n - 1) * (128 * nreq + 128)
    c.close()


def test_exact_fit_wrap_rule_E1(eng, orc):
    """An entry that ends exactly at len: the engine stores end = 0 (divergence E1; the
    reference's end == len would read as "log empty", SURVEY.md H11 iv)."""
    n, L = 3, 8192
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, n, leader=0, term=1, length=L)
    c.prologue()
    with eng.Group(n, devices=devices_for(eng, n), log_size=L) as g:
        g.prologue()
        part = S.uniform_stream(62, 64)                 # CONFIG 64 + CONNECT 64 + 62*128 = 8064
        for typ, clt, rid, payload in part:
            assert c.submit(typ, clt, rid, O.cmd_image(payload))
        c.round(); c.round()
        g.submit_stream(part); g.run()
        assert prune_both(g, c)                          # HEAD entry: 8064 -> 8128
        c.round(); c.round(); g.run()
        tail_part = [(S.SEND, 0, 64, b""),               # 64 B stride: ends exactly at 8192
                     (S.SEND, 0, 65, b"after the wrap" * 3), (S.SEND, 0, 66, b"x" * 100)]
        for typ, clt, rid, payload in tail_part[:1]:
            assert c.submit(typ, clt, rid, O.cmd_image(payload))
        c.round(); c.round()
        assert c.offsets(0)["end"] == 0
        g.submit_stream(tail_part[:1]); g.run()
        assert g.leader.offsets()["end"] == 0
        for typ, clt, rid, payload in tail_part[1:]:
            assert c.submit(typ, clt, rid, O.cmd_image(payload))
        c.round(); c.round()
        g.submit_stream(tail_part[1:]); g.run()
        EU.compare_group_to_oracle(g, c, exact=True)
    c.close()


WRAP_CASES = [
    # small ragged entries, a dozen per launch: ghost headers, header-does-not-fit jumps, tiny tiles (the original cases,
    # under their original ids)
    *[wrap_case(n, L, "ragged180", seed, mode, step=12, id=f"{n}-{L}-{seed}-{mode}")
      for mode in ("index_earlyack", "walk_fenced") for n, L, seed in ((3, 16384, 77), (5, 32768, 78), (3, 8192, 79))],
    # below: about a third of the ring per launch, so that a claim holds tens of entries
    # stride 1024: the 16 B register compose path with the holes-only prefill
    wrap_case(3, 1 << 16, "u960", 80, "index_earlyack", ctas=1),
    wrap_case(5, 1 << 18, "u960", 81, "walk_fenced", ctas=16),
    # stride 1065: byte-granular compose with the holes-only prefill; the slack hole straddles 16 B chunks
    wrap_case(3, 1 << 16, "u1001", 82, "walk_fenced", ctas=2),
    wrap_case(5, 1 << 18, "u1001", 83, "index_earlyack", ctas=4),
    # stride 264: whole-warp compose with the full-sweep prefill
    wrap_case(3, 1 << 16, "u200", 84, "index_earlyack", ctas=16),
    wrap_case(3, 1 << 18, "u200", 85, "walk_fenced", ctas=96),
    # 0..1500 B with connection churn: ghost headers of large entries, tiles switching between the two prefills
    wrap_case(3, 1 << 18, "ragged1500", 86, "index_earlyack", ctas=2),
    wrap_case(5, 1 << 16, "ragged1500", 87, "walk_fenced", ctas=16),
    wrap_case(3, 1 << 16, "ragged180", 88, "index_earlyack", ctas=1),
    # requests in HBM, one bulk call per launch: claims of 256 slots
    wrap_case(3, 1 << 18, "u200", 89, "index_earlyack", ctas=1, ring="device"),
]


@pytest.mark.parametrize("n,L,kind,seed,mode,step,ctas,ring", WRAP_CASES)
def test_wrap_laps_with_pruning(eng, orc, n, L, kind, seed, mode, step, ctas, ring):
    """Several laps around a small ring: ghost headers, header-does-not-fit jumps,
    stale bytes in entry holes, HEAD entries, for every compose path and prefill of the
    leader and 1..96 leader CTAs.  Pruning happens at quiescent points so that the
    stream of appends is identical on both sides."""
    EU.wrap_laps_with_pruning(eng, orc, n, L, kind, seed, mode, step, ctas, ring)


def test_persistent_service_mode_closed_loop(eng, orc):
    """Kernels stay resident (target = forever); a single client submits one request
    at a time and waits for its commit, like proxy.c:160."""
    n, L = 3, 1 << 20
    stream = S.ragged_stream(400, 100, conns=2, seed=31)
    with eng.Group(n, devices=devices_for(eng, n), log_size=L) as g:
        g.launch(target=(1 << 64) - 1)
        t = g.prologue()
        g.leader.wait_committed(t)
        for typ, clt, rid, payload in stream:
            t = g.submit(typ, clt, rid, payload)
            g.leader.wait_committed(t, 5_000_000)
            assert g.leader.committed() >= t
        g.stop()
        c = EU.oracle_cluster(orc, n, L, stream)
        # followers were stopped right after the last commit: their commit offset may lag
        lo = g.leader.offsets()
        assert lo["commit"] == lo["end"] == c.offsets(0)["end"]
        ents = O.walk_entries(c.image(0), 0, lo["end"], L)
        assert np.array_equal(O.mask_replies(g.leader.image(), ents), O.mask_replies(c.image(0), ents))
        for i in range(1, n):
            fo = g.replicas[i].offsets()
            assert fo["end"] == lo["end"]
            assert np.array_equal(O.mask_replies(g.replicas[i].image(), ents), O.mask_replies(c.image(i), ents))
        c.close()


def test_commit_is_monotone_prefix(eng, orc):
    """Observe the committed-ticket word while a long run is in flight: it only grows
    and never passes what was submitted (invariant I3)."""
    n, L = 5, 1 << 22
    stream = S.uniform_stream(20000, 64, conns=8)
    with eng.Group(n, devices=devices_for(eng, n), log_size=L) as g:
        g.prologue()
        g.submit_stream(stream)
        g.launch()
        seen = []
        while g.leader.committed() < g.tickets:
            seen.append(g.leader.committed())
            if len(seen) > 5_000_000:
                break
        g.wait()
        assert all(b >= a for a, b in zip(seen, seen[1:]))
        assert g.leader.committed() == g.tickets


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_golden.json")


@pytest.mark.parametrize("name,n,seed", [("cluster3_ragged", 3, 13), ("cluster5_ragged", 5, 15),
                                         ("cluster7_ragged", 7, 17), ("cluster1_ragged", 1, 11)])
def test_against_reference_golden(eng, name, n, seed):
    """No oracle at run time: SHA-256 of every replica's log image against the vectors
    generated from the COMPILED REFERENCE HEADER (tests/golden/gen_golden.py)."""
    gold = {g["name"]: g for g in json.load(open(GOLD))["scenarios"]}[name]
    stream = S.ragged_stream(500, 256, seed=seed, close_every=60)
    L = 1 << 20
    with eng.Group(n, devices=devices_for(eng, n), log_size=L) as g:
        g.prologue()
        g.submit_stream(stream)
        g.run()
        for i, r in enumerate(g.replicas):
            assert hashlib.sha256(r.image().tobytes()).hexdigest() == gold["sha"][i], f"replica {i}"
            o = r.offsets()
            assert o["end"] == gold["offsets"][i]["end"] and o["commit"] == gold["offsets"][i]["commit"]
        assert g.leader.stats()["bytes_replicated"] == gold["bytes_replicated"]


def check_replica_images_consistent(g, L, request=None):
    """Size-independent properties for runs too long for the oracle: every follower
    holds exactly the leader's live log bytes (modulo reply[]), entries parse from
    head to end with consecutive idx, HEAD entries carry offsets inside the ring.
    With `request` (ticket -> (type, clt_id, req_id, payload)) the live region is also
    checked against the submitted stream: counting tickets back from the last one,
    every entry that is not a HEAD must be its request; the last HEAD carries the
    leader's head, which every follower holds; every HEAD whose head lies in the region
    carries an entry boundary of it not past the HEAD itself; consecutive HEADs move
    the head by at least L/8.  The holes (bytes no append writes) and what the
    overwritten laps held cannot be checked without those laps: the replays of
    tests/test_gpu_prune_in_launch.py do that on smaller rings."""
    lo = g.leader.offsets()
    limg = g.leader.image()
    assert lo["commit"] == lo["end"]
    start = lo["head"]
    ents = O.walk_entries(limg, start, lo["end"], L)
    assert len(ents) > 0
    idx = [int.from_bytes(limg[o:o + 8].tobytes(), "little") for o, _ in ents]
    assert idx == list(range(idx[0], idx[0] + len(idx)))
    for o, _ in ents:
        if limg[o + 26] == 3:
            h = int.from_bytes(limg[o + 48:o + 56].tobytes(), "little")
            assert 0 <= h < L
        assert limg[o + 27] == g.leader_idx
    if request is not None:
        _check_live_region(g, L, limg, lo, ents, request)
    lm = O.mask_replies(limg, ents)
    for i, r in enumerate(g.replicas):
        if i == g.leader_idx:
            continue
        fo = r.offsets()
        assert fo["end"] == lo["end"] and fo["commit"] == lo["commit"] and fo["apply"] == lo["commit"]
        fimg = O.mask_replies(r.image(), ents)
        for o, stride in ents:
            assert np.array_equal(fimg[o:o + stride], lm[o:o + stride]), f"replica {i} entry at {o}"
        for o, _ in ents[-50:]:
            assert r.image(o + 28 + i, o + 29 + i)[0] == 1
    return len(ents), idx[-1]


def _check_live_region(g, L, limg, lo, ents, request):
    """check_replica_images_consistent's content checks of the leader's [head, end)"""
    head = lo["head"]
    rel = {o: (o - head) % L for o, _ in ents}                    # position in the region
    bounds = {head} | {o for o, _ in ents} | {(o + s) % L for o, s in ents}      # head: also where a wrap skipped
    ticket = g.tickets
    heads = []
    for o, stride in reversed(ents):
        typ = int(limg[o + 26])
        if typ == O.HEAD:
            heads.append((o, int.from_bytes(limg[o + 48:o + 56].tobytes(), "little")))
            continue
        want_typ, clt, rid, payload = request(ticket)
        got = (typ, int.from_bytes(limg[o + 24:o + 26].tobytes(), "little"),
               int.from_bytes(limg[o + 16:o + 24].tobytes(), "little"))
        assert got == (want_typ, clt, rid), f"entry at {o}: (type, clt_id, req_id) {got}, ticket {ticket} is {(want_typ, clt, rid)}"
        if typ != O.CONFIG:
            ln = int(limg[o + 48]) | int(limg[o + 49]) << 8
            assert ln == len(payload) and stride == 64 + ln, f"entry at {o}: len {ln}, ticket {ticket} has {len(payload)}"
            assert limg[o + 50:o + 50 + ln].tobytes() == payload, f"entry at {o}: data image of ticket {ticket}"
        ticket -= 1
    heads.reverse()
    assert heads, "no HEAD entry in the live region: the leader's head was carried by none"
    assert heads[-1][1] == head, f"the last HEAD carries {heads[-1][1]}, the leader's head is {head}"
    for k, (o, v) in enumerate(heads):
        if (v - head) % L <= rel[o]:                              # its head lies in the region
            assert v in bounds, f"HEAD at {o} carries {v}, not an entry boundary of [{head}, {lo['end']})"
        if k:
            pv, po = heads[k - 1][1], heads[k - 1][0]
            adv = (v - pv) % L
            assert L // 8 <= adv <= (o - pv) % L, f"HEAD at {o}: head {pv} -> {v} moves by {adv}"
    for i, r in enumerate(g.replicas):
        if i != g.leader_idx:
            assert r.offsets()["head"] == head, f"replica {i} head {r.offsets()['head']}, the last HEAD carries {head}"


@pytest.mark.parametrize("n,L,payload", [(3, 1 << 20, 64), (5, 1 << 20, 200), (3, 1 << 18, 1000),
                                         pytest.param(5, O.LOG_SIZE, 64, id="bench-shape-n5-64M-synth64-ctas16")])
def test_sustained_autoprune_many_laps(eng, n, L, payload):
    """Device-side pruning (APUS_F_AUTOPRUNE): 40+ laps around a small ring in a few
    launches, no host-side HEAD submission; the live region against the submitted
    requests.  The ring of the reference's LOG_SIZE runs the benchmark's configuration:
    five replicas, 16 leader CTAs, 2^20 device-generated 64 B requests per launch in
    the HBM ring, two launches (four laps)."""
    from apus_b200 import engine as E
    flags = E.F_DEVICE_STATS | E.F_AUTOPRUNE
    bench = L == O.LOG_SIZE
    per, rounds = (1 << 20, 2) if bench else (20000, 4)
    seed = 0xA5A50000 + payload
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, ring_mode=eng.RING_DEVICE,
                   ring_slots=(1 << 21) if bench else 1 << 17, ring_bytes=64 << 20, flags=flags,
                   leader_ctas=16 if bench else 0) as g:
        g.prologue()
        g.submit(S.CONNECT, 0, 1, b"")
        req = 2
        rng = np.random.default_rng(5)
        sent = {}                                    # first req_id of a round -> its payloads
        for _ in range(rounds):
            if bench:
                g.tickets = g.leader.submit_synth(per, S.SEND, 0, req, payload, seed) + per - 1
            else:
                pl = rng.integers(0, 256, size=per * payload, dtype=np.uint8)
                sent[req] = pl
                g.submit_uniform(per, payload, 0, req, pl)
            req += per
            g.run(timeout_ms=120_000)
        st = g.leader.stats()
        assert st["tickets_committed"] == g.tickets
        assert st["auto_heads"] > 0
        laps = (per * rounds * (64 + payload)) / L
        assert laps > (3.9 if bench else 4)

        def request(ticket):                         # ticket 1 the CONFIG prologue, 2 the CONNECT, then req_id + 1
            if ticket == 1:
                return (O.CONFIG, 0, 0, b"")
            if ticket == 2:
                return (S.CONNECT, 0, 1, b"")
            rid = ticket - 1
            if bench:
                return (S.SEND, 0, rid, E.synth_payload(seed, rid, payload))
            first = 2 + (rid - 2) // per * per
            k = rid - first
            return (S.SEND, 0, rid, sent[first][k * payload:(k + 1) * payload].tobytes())

        n_live, last_idx = check_replica_images_consistent(g, L, request)
        assert last_idx == g.tickets + st["auto_heads"]


# ---- golden vectors produced by the RUNNING reference (tests/golden/gen_refstack_golden.py) -----------------------
REFGOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refstack_golden.json")


def _refgold():
    with open(REFGOLD) as f:
        return json.load(f)["scenarios"]


@pytest.mark.parametrize("gold", _refgold(), ids=lambda g: g["name"])
def test_engine_reproduces_reference_run(eng, gold):
    """The logs the reference's own replicas held after its unmodified election / replication / commit code ran the
    scenario (leader index and term as its election produced them; SHA-256, followers under the H5 reply mask):
    the CUDA engine, led by the same replica in the same term, must leave the same bytes."""
    import refstack as R
    n, lead, end = gold["n"], gold["leader"], gold["end"]
    with eng.Group(n, devices=devices_for(eng, n), leader=lead, term=gold["term"], log_size=O.LOG_SIZE) as g:
        g.prologue()
        g.submit_stream(R.expected_stream(lead, gold["nconn"], gold["nreq"], gold["plen"]))
        g.run()
        ents = O.walk_entries(g.leader.image(0, end), 0, end, O.LOG_SIZE)
        assert len(ents) == gold["entries"] == g.leader.committed()
        for i in range(n):
            o = g.replicas[i].offsets()
            assert {k: o[k] for k in ("head", "apply", "commit", "end")} == gold["offsets"][i], (i, o)
            img = g.replicas[i].image(0, end)
            if i != lead:
                for off, _ in ents:
                    assert img[off + 28 + i] == 1            # I7: the follower's own ack byte
                img = O.mask_replies(img, ents)
            assert hashlib.sha256(img.tobytes()).hexdigest() == gold["sha256"][i], f"replica {i}"
