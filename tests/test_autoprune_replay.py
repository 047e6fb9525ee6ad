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


@pytest.mark.parametrize("head,end,v,prev,allow,expect", [
    (0, 512, 256, False, False, None),                               # legal
    (0, 512, 128, False, False, None),                               # exactly an eighth
    (0, 256, 128, False, False, None),                               # exactly a quarter used
    (0, 192, 128, False, False, "L/4"),                              # ring used below a quarter
    (0, L1K, 128, False, False, "L/4"),                              # empty log (end == len)
    (0, 512, 64, False, False, "L/8"),                               # head moves by less than an eighth
    (0, 512, 0, False, False, "L/8"),                                # head does not move
    (0, 512, 300, False, False, "boundary"),                         # inside an entry
    (0, 512, 576, False, False, "past"),                             # beyond the HEAD entry's own position
    (0, 512, 512, False, False, None),                               # at the HEAD entry's own position
    (0, 512, 256, True, False, "two HEAD"),                          # right behind another HEAD entry
    (0, 512, 256, True, True, None),                                 # ... which a blocked placement may do
    (896, 384, 128, False, False, None),                             # across the wrap
    (896, 384, 960, False, False, "L/8"),
    (896, 384, 448, False, False, "past"),
])
def test_head_violation_rules(head, end, v, prev, allow, expect):
    why = R.head_violation(L1K, head, end, v, _b(head, end if end != L1K else head), prev, allow)
    if expect is None:
        assert why is None, why
    else:
        assert why is not None and expect in why, why
