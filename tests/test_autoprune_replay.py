"""The replay harness of the device-side pruning tests (tests/autoprune_replay.py) checked on the CPU oracle alone: an
oracle run that prunes by the engine's rule at quiescent points, read back launch by launch and replayed into a fresh
cluster, must give back every replica byte for byte; a replay with one HEAD moved or dropped must not; and the
legality predicate must accept and refuse hand-built cases, one per clause of the rule."""
import numpy as np
import pytest

import autoprune_replay as R
import orc as O
import streams as S


def oracle_run(orc, n, L, stream, step):
    """The oracle on its own over several laps: `step` requests per launch, two quiescent rounds, then SIM(prune)
    where the engine's rule would prune (a quarter of the ring used, the head moving by an eighth).  Returns the
    cluster and the entries each launch appended, read back from the leader's image like the GPU tests do."""
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, n, leader=0, term=1, length=L)
    launches = []
    prev = 0
    cid = [0] * n
    requests = [(O.CONFIG, 0, 0, b"")] + stream
    for k in range(0, len(requests), step):
        for typ, clt, rid, payload in requests[k:k + step]:
            assert (c.prologue() if typ == O.CONFIG else c.submit(typ, clt, rid, O.cmd_image(payload))) != 0
        c.round(); c.round()
        o = c.offsets(0)
        if R.dist(o["head"], o["end"], L) >= L // 4 and R.dist(o["head"], o["tail"], L) >= L // 8:
            assert c.prune() != 0
            c.round(); c.round()
        R.poll_heads(c, cid)
        end = c.offsets(0)["end"]
        launches.append(R.launch_from_image(c.image(0), prev, end, L))
        prev = end
    return c, launches, requests


def replay(orc, n, L, launches, requests):
    rp = R.Replay(orc, n, L)
    for lc in launches:
        rp.launch(lc, requests)
    return rp


def same_cluster(a, b, n):
    """every byte and every offset of every replica"""
    for i in range(n):
        if a.offsets(i) != b.offsets(i):
            return f"replica {i}: offsets {a.offsets(i)} vs {b.offsets(i)}"
        d = np.nonzero(a.image(i) != b.image(i))[0]
        if len(d):
            return f"replica {i}: {len(d)} bytes differ, first at {int(d[0])}"
    if a.bytes_replicated() != b.bytes_replicated():
        return f"bytes_replicated {a.bytes_replicated()} vs {b.bytes_replicated()}"
    return None


CASES = {
    # 128 B strides: the benchmark's shape
    "u64": lambda L: S.uniform_stream(int(4.5 * L / 128) + 1, 64, seed=5),
    # 0..300 B with connection churn: ghost headers and header-does-not-fit jumps at the wraps
    "ragged300": lambda L: S.ragged_stream(int(4.5 * L / 214) + 1, 300, conns=3, seed=6, close_every=25),
}


@pytest.fixture(params=list(CASES))
def run(request, orc):
    n, L = 3, 1 << 16
    stream = CASES[request.param](L)
    step = max(1, int(0.3 * L * len(stream) / S.stream_bytes(stream)))
    c, launches, requests = oracle_run(orc, n, L, stream, step)
    yield n, L, c, launches, requests
    c.close()


def test_replay_reproduces_the_oracle(orc, run):
    n, L, c, launches, requests = run
    heads = sum(1 for lc in launches for e in lc.entries if e.typ == O.HEAD)
    rp = replay(orc, n, L, launches, requests)
    try:
        assert rp.written >= 4 * L                                   # laps
        assert len(rp.heads) == heads >= 4
        assert rp.pos == len(requests)
        assert same_cluster(c, rp.c, n) is None, same_cluster(c, rp.c, n)
        # every follower adopted the head of the last HEAD entry; the leader holds it
        for i in range(n):
            assert rp.c.offsets(i)["head"] == rp.last_committed_head() == c.offsets(0)["head"]
        R.assert_heads_have_teeth(rp, rp.c.image(0))
    finally:
        rp.close()


def _mutated(launches, how, L):
    """a copy of the launches with the middle HEAD entry moved to another legal head, or dropped; the leader's bytes
    stay what the unchanged run wrote"""
    where = [(k, j) for k, lc in enumerate(launches) for j, e in enumerate(lc.entries) if e.typ == O.HEAD]
    k, j = where[len(where) // 2]
    out = [R.Launch(lc.start, lc.end, lc.buf, list(lc.entries)) for lc in launches]
    h = out[k].entries[j]
    if how == "drop":
        del out[k].entries[j]
    else:
        # the next entry boundary past the carried head; when that is the HEAD entry's own position (a head at the
        # last entry, as at every quiescent point) the boundary before it, which is legal too
        flat = [e for lc in launches[:k] for e in lc.entries] + launches[k].entries[:j]
        at = [e for e in flat if e.off == h.value][-1]
        v = (at.off + at.stride) % L
        if v == h.off:
            v = [e for e in flat if (e.off + e.stride) % L == h.value][-1].off
        out[k].entries[j] = R.Entry(h.off, h.stride, h.typ, h.idx, h.req_id, h.clt_id, v)
    return out


def test_replay_with_a_moved_head_differs(orc, run):
    """a HEAD carrying another legal head passes the rule, and the launch's bytes tell it apart (long before a later
    lap overwrites it)"""
    n, L, c, launches, requests = run
    with pytest.raises(AssertionError, match="byte 4[89] of the HEAD entry"):
        replay(orc, n, L, _mutated(launches, "next_boundary", L), requests).close()


def test_replay_without_a_head_is_refused(orc, run):
    """without one of the engine's HEAD entries the oracle's end (and every idx behind it) falls behind the engine's"""
    n, L, c, launches, requests = run
    with pytest.raises(AssertionError, match="engine (end|idx)"):
        replay(orc, n, L, _mutated(launches, "drop", L), requests).close()


# ---- the pruning rule, one clause at a time: L = 1024 (L/4 = 256, L/8 = 128), 64 B entries ----------------------
L1K = 1024


def _b(head, end):
    """starts and ends of 64 B entries from head to end"""
    return {(head + 64 * k) % L1K for k in range(R.dist(head, end, L1K) // 64 + 1)}


@pytest.mark.parametrize("head,end,v,prev,nxt,expect", [
    (0, 512, 256, False, None, None),                                # legal
    (0, 512, 128, False, None, None),                                # exactly an eighth
    (0, 256, 128, False, None, None),                                # exactly a quarter used
    (0, 192, 128, False, None, "L/4"),                               # ring used below a quarter
    (0, L1K, 128, False, None, "L/4"),                               # empty log (end == len)
    (0, 512, 64, False, None, "L/8"),                                # head moves by less than an eighth
    (0, 512, 0, False, None, "L/8"),                                 # head does not move
    (0, 512, 300, False, None, "boundary"),                          # inside an entry
    (0, 512, 576, False, None, "past"),                              # beyond the HEAD entry's own position
    (0, 512, 512, False, None, None),                                # at the HEAD entry's own position
    (896, 384, 128, False, None, None),                              # across the wrap
    (896, 384, 960, False, None, "L/8"),
    (896, 384, 448, False, None, "past"),
    # right behind another HEAD entry: legal only when the next entry's placement blocked at this head and end.
    # No-wrap side (512 bytes used, 512 left): E2 keeps 1 + 64 bytes, so 447 fits and 448 blocks
    (0, 512, 256, True, None, "no entry behind"),
    (0, 512, 256, True, 447, "would have fit"),
    (0, 512, 256, True, 448, None),
    (0, 512, 256, True, 512, None),
    # wrap side (576 used, 64 left before the ring's end): 64 fits, 65..319 wrap (the skipped stretch counts), 320
    # blocks
    (384, 960, 512, True, 64, "would have fit"),
    (384, 960, 512, True, 65, "would have wrapped"),
    (384, 960, 512, True, 319, "would have wrapped"),
    (384, 960, 512, True, 320, None),
])
def test_head_violation_rules(head, end, v, prev, nxt, expect):
    why = R.head_violation(L1K, head, end, v, _b(head, end if end != L1K else head), prev, nxt)
    if expect is None:
        assert why is None, why
    else:
        assert why is not None and expect in why, why


# A HEAD is appended at the end or nowhere: never at 0 behind a wrapping entry's ghost header (128 B left before the
# ring's end) or behind the stretch skipped when even the header does not fit (32 B left).  Counting that stretch can
# put the ring over a quarter used where the end alone does not.
@pytest.mark.parametrize("head,end,v,at,expect", [
    (640, 896, 768, 896, None),                                      # legal at the end (256 used)
    (640, 896, 768, 0, "ghost/skip"),                                # the same HEAD behind the ghost
    (704, 896, 832, 896, "L/4"),                                     # 192 used: not due at the end ...
    (704, 896, 832, 0, "ghost/skip"),                                # ... named as such at 0, not as a used count
    (704, 960, 832, 960, None),                                      # 256 used, exactly one header left
    (704, 992, 832, 992, "does not fit"),                            # 288 used, but the header would cross len
    (704, 992, 832, 0, "ghost/skip"),
    (640, 0, 768, 0, None),                                          # end 0 after an exact fit (E1): 0 is the end
])
def test_head_between_a_wrap_and_its_entry(head, end, v, at, expect):
    why = R.head_violation(L1K, head, end, v, _b(head, end), False, None, at=at)
    if expect is None:
        assert why is None, why
    else:
        assert why is not None and expect in why, why


# ---- recordings of host-applying followers (replay_recordings), produced by the oracle alone -------------------------
def recorded_run(orc, n, L, stream, seed, step):
    """The oracle standing in for a launch that laps the ring with host-applying followers: requests appended in
    random chunks by the leader's own arithmetic (the pruning rule on the followers' reports before each entry, a HEAD
    pair only behind a blocked placement, E2 with one header kept), then follower 1's host reads and reports all that
    is committed, follower 2's at random times and at most `step` bytes (ending on an entry boundary).  Returns the
    cluster, the recordings, the requests and the number of HEAD pairs; time is a counter."""
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, n, leader=0, term=1, length=L)
    rng = np.random.default_rng(seed)
    requests = [(O.CONFIG, 0, 0, b"")] + stream
    recs = {j: R.Recording(j) for j in range(1, n)}
    rep = {j: 0 for j in recs}                       # absolute apply offset each host reported
    clock = iter(range(1, 1 << 62))
    written, pos, prev_head, blocked, pairs, cid = 0, 0, False, False, 0, [0] * n

    def append(fn):
        nonlocal written
        start = c.offsets(0)["end"]
        idx = fn()
        assert idx != 0, "the oracle refused an append the leader's arithmetic allows"
        written += R.dist(0 if start == L else start, c.offsets(0)["end"], L)

    def host_reads(final=False):
        for j, rec in recs.items():
            if rep[j] == written or (j > 1 and not final and rng.random() < 0.5):
                continue
            at = (rep[j] + np.arange(written - rep[j])) % L
            buf = c.image(j)[at]
            rec.segs.append((rep[j], buf, next(clock)))
            adv = len(buf) if j == 1 else R.boundary_within(buf, rep[j] % L, L, step)
            rep[j] += adv
            rec.reports.append((rep[j], next(clock)))

    while pos < len(requests):
        for _ in range(int(rng.integers(1, 12))):
            if pos == len(requests):
                break
            o = c.offsets(0)
            used = 0 if o["end"] == L else R.dist(o["head"], o["end"], L)
            if o["end"] != L and used >= L // 4 and (not prev_head or blocked) and L - o["end"] >= O.HDR:
                d = max(min(R.dist(rep[j] % L, o["end"], L), used) for j in recs) or R.dist(o["tail"], o["end"], L)
                if used - d >= L // 8:
                    pairs += prev_head
                    append(lambda: c.prune_to((o["end"] - d) % L))
                    prev_head, blocked = True, False
                    c.round(); c.round()
                    R.poll_heads(c, cid)
                    o = c.offsets(0)
            typ, clt, rid, payload = requests[pos]
            if R.placement_refusal(L, o["head"], o["end"], R.request_stride(requests[pos])) is None:
                blocked = True
                break
            append(lambda: c.prologue() if typ == O.CONFIG else c.submit(typ, clt, rid, O.cmd_image(payload)))
            pos += 1
            prev_head, blocked = False, False
        c.round(); c.round()
        R.poll_heads(c, cid)
        host_reads()
    while any(r != written for r in rep.values()):
        host_reads(final=True)
    return c, [recs[j] for j in sorted(recs)], requests, pairs


REC_CASES = {
    # 128 B strides: the benchmark's shape
    "u64": (1 << 16, lambda L: S.uniform_stream(int(6.5 * L / 128) + 1, 64, seed=7)),
    # 0..1500 B with connection churn: ghost headers and the stretches skipped at wraps
    "ragged1500": (1 << 16, lambda L: S.ragged_stream(int(7.5 * L / 814) + 1, 1500, conns=3, seed=8, close_every=20)),
    # 3..9 KiB on 32 KiB: most entries are larger than a prune of L/8 frees, so HEAD pairs behind blocked placements
    "sized3k9k": (1 << 15, lambda L: S.sized_stream(int(6.5 * L / 6200) + 1, 3072, 9216, seed=9)),
}


@pytest.fixture(params=list(REC_CASES))
def rec_run(request, orc):
    n, (L, stream) = 3, REC_CASES[request.param]
    c, recs, requests, pairs = recorded_run(orc, n, L, stream(L), seed=11, step=L // 64)
    yield n, L, c, recs, requests, pairs
    c.close()


def _replay_recs(orc, n, L, recs, requests, pieces=None):
    rp = R.Replay(orc, n, L)
    try:
        R.replay_recordings(rp, recs, requests, pieces)
    except BaseException:
        rp.close()
        raise
    return rp


def test_recordings_reproduce_the_oracle(orc, rec_run):
    """the pieces cut at every read, replayed, give back every replica byte for byte; every HEAD passes the rule and
    the reports before it was read"""
    n, L, c, recs, requests, pairs = rec_run
    rp = _replay_recs(orc, n, L, recs, requests)
    try:
        assert rp.written >= 6 * L
        assert len(rp.heads) >= 6
        assert rp.pos == len(requests)
        assert same_cluster(c, rp.c, n) is None, same_cluster(c, rp.c, n)
        R.assert_heads_have_teeth(rp, rp.c.image(0))
        assert rp.pairs == pairs
        assert pairs > 0 or L > 1 << 15
    finally:
        rp.close()


def _mid(segs, ok=lambda s, b: True):
    cand = [k for k, (s, b, _) in enumerate(segs) if ok(s, b)]
    assert cand
    return cand[len(cand) // 2]


def test_recording_with_a_changed_byte_is_refused(orc, rec_run):
    """one byte of an entry header in follower 2's recording: named by follower, entry idx and byte"""
    n, L, c, recs, requests, pairs = rec_run
    segs = recs[1].segs
    k = _mid(segs, lambda s, b: s % L + 1600 < L and len(b) > 64)
    s, b, t = segs[k]
    b = b.copy()
    b[16] ^= 0x5A                                                # req_id of the entry the read starts with
    segs[k] = (s, b, t)
    with pytest.raises(AssertionError, match=r"follower 2: 1 bytes of the read of \[\d+, \d+\) differ from the oracle, "
                                             r"first at \d+: byte 16 of the (HEAD|type \d+) entry idx \d+"):
        _replay_recs(orc, n, L, recs, requests).close()


def test_recording_read_after_a_later_lap_is_refused(orc, rec_run):
    """follower 2's read holding what the ring held one lap later: the leader overwrote it before the read"""
    n, L, c, recs, requests, pairs = rec_run
    _, flat, _, _ = R.recording_pieces(recs, L)
    segs = recs[1].segs
    k = _mid(segs, lambda s, b: s + len(b) + L <= len(flat) and len(b) > 256)
    s, b, t = segs[k]
    segs[k] = (s, flat[s + L:s + L + len(b)].copy(), t)
    with pytest.raises(AssertionError, match=r"follower 2: entry idx \d+ at \d+ was overwritten by lap \+1 before the "
                                             r"read of \[\d+, \d+\) returned: byte \d+ is"):
        _replay_recs(orc, n, L, recs, requests).close()


def test_head_past_a_report_is_refused(orc, rec_run):
    """follower 2's reports arriving only after every read: each HEAD carries a head it had not reported yet"""
    n, L, c, recs, requests, pairs = rec_run
    recs[1].reports = [(a, t + (1 << 40)) for a, t in recs[1].reports]
    with pytest.raises(AssertionError, match=r"follower 1's read: HEAD idx \d+ at \d+: head \d+ \(absolute \d+\) is "
                                             r"past follower 2's last report 0 before the HEAD was first read "
                                             r"\(byte 48 of the HEAD entry"):
        _replay_recs(orc, n, L, recs, requests).close()


def test_head_pair_that_was_not_blocked_is_refused(orc, rec_run):
    """a second HEAD right behind one, legal by every other clause, where the next entry would have been placed"""
    n, L, c, recs, requests, pairs = rec_run
    pieces, _, _, _ = R.recording_pieces(recs, L)
    flat = [(c0 + R.dist(lc.start, e.off, L), k, j, e) for k, (c0, lc) in enumerate(pieces)
            for j, e in enumerate(lc.entries)]
    ends = {a + e.stride for a, _, _, e in flat}
    for i, (a, k, j, h) in enumerate(flat):
        nxt = next((e for _, _, _, e in flat[i + 1:] if e.typ != O.HEAD), None)
        if h.typ != O.HEAD or nxt is None:
            continue
        v1 = a - R.dist(h.value, h.off, L)
        end = a + h.stride
        cands = sorted(x for x in ends if v1 + L // 8 <= x <= end)
        if end - v1 >= L // 4 and cands and R.placement_refusal(L, v1 % L, end % L, nxt.stride):
            break
    else:
        pytest.fail("no HEAD entry with room for a second one behind it")
    lc = pieces[k][1]
    extra = R.Entry(h.off + h.stride, O.HDR, O.HEAD, h.idx + 1, 0, 0, cands[0] % L)
    pieces[k] = (pieces[k][0], R.Launch(lc.start, lc.end, lc.buf, lc.entries[:j + 1] + [extra] + lc.entries[j + 1:]))
    with pytest.raises(AssertionError, match=rf"follower 1's read: HEAD idx {h.idx + 1} at {extra.off}: two HEAD entries "
                                             r"in a row, but the placement was not blocked: the next entry \(stride "
                                             r"\d+\) would have (fit|wrapped)"):
        _replay_recs(orc, n, L, recs, requests, pieces).close()


def test_recording_with_a_gap_is_refused(orc, rec_run):
    """one read of follower 1 missing: nothing else of it covers those bytes"""
    n, L, c, recs, requests, pairs = rec_run
    segs = recs[0].segs
    k = _mid(segs)
    del segs[k]
    with pytest.raises(AssertionError, match=r"follower 1: the recording has a gap \[\d+, \d+\): byte \d+ of the (HEAD|type \d+) "
                                             r"entry idx \d+ at \d+ was never read"):
        _replay_recs(orc, n, L, recs, requests).close()
