"""The leader's placement at the ring's end, edge by edge, against the oracle (plans: tests/ring_edges.py; the plans
themselves are checked on the CPU by tests/test_ring_edges_plan.py).  Marked gpu.

Wrap geometry: each edge request is placed at an exact `left` bytes before len -- 0 (exact fit of the entry before),
1, 15, 16, 17, 63 (the header does not fit), 64 (it fits exactly), 65, and the entry's stride - 1, stride, + 1 -- as
an empty SEND, a 841 B SEND, a maximal 65535 B cmd staged as an external image, a header-only CONNECT or a HEAD entry
the host submits, first, in the middle or last in its launch, after a lap has left stale bytes everywhere.  Every byte
and offset of every replica is compared with the oracle after each edge, for 1 and 16 leader CTAs and every follower
mode (the walking followers take the jump and ghost rules of their own walker).

Pruning at the ring's end (APUS_F_AUTOPRUNE, followers that report pinned apply offsets, one request per claim): the
rule where the skipped stretch would cross a quarter of the ring (C1), a HEAD ending exactly at len (C2), a HEAD
followed by a wrapping entry (C3), the used and advance thresholds to the byte (C4), the express path's hand-over at
half used, a HEAD carrying the tail when every replica applied up to the end right after a wrap (C5), and rule E2 to
the byte with the HEAD reserve, in place and wrapped, placed at L - 1 and held one byte later until the followers
release it (B).  Each is replayed into the oracle by autoprune_replay.Replay, which checks every HEAD entry against
the rule and every byte of every launch.  Some run at 5 replicas."""
import time

import numpy as np
import pytest

import autoprune_replay as AR
import engine_util as EU
import orc as O
import ring_edges as RE
import streams as S
from apus_b200 import engine as E
from engine_util import MODES, devices_for, eng, pin_and_wait, prune_both  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


@pytest.fixture(scope="module")
def plans(orc):
    """the tours of ring_edges.TOURS, planned once for the module"""
    out = {}
    yield lambda name: out[name] if name in out else out.setdefault(name, RE.make_tour(orc, name))
    for t in out.values():
        t.close()


TOUR_RUNS = [pytest.param("small", mode, ctas, id=f"small-{mode}-ctas{ctas}") for mode in MODES for ctas in (1, 16)]
TOUR_RUNS += [pytest.param("small-n5", "walk_fenced", 4, id="small-n5-walk_fenced-ctas4"),
              pytest.param("max", "index_earlyack", 1, id="max-index_earlyack-ctas1"),
              pytest.param("max", "walk_fenced", 16, id="max-walk_fenced-ctas16")]


@pytest.mark.parametrize("name,mode,ctas", TOUR_RUNS)
def test_wrap_edges_against_the_oracle(eng, orc, plans, name, mode, ctas):
    t = plans(name)
    n, L = t.n, t.L
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, n, leader=0, term=1, length=L)
    try:
        with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES[mode], leader_ctas=ctas) as g:
            for s in t.steps:
                if s[0] == "config":
                    g.prologue(); c.prologue()
                elif s[0] == "req":
                    typ, clt, rid, payload = s[1]
                    g.submit(typ, clt, rid, payload)
                    assert c.submit(typ, clt, rid, O.cmd_image(payload))
                elif s[0] == "run":
                    g.run(); c.round(); c.round()
                elif s[0] == "prune":
                    assert prune_both(g, c)
                else:
                    e = t.edges[s[1]]
                    what = f"{e.kind} at left {e.left} ({e.pos}, {e.expect})"
                    try:
                        EU.compare_group_to_oracle(g, c, exact=True)
                    except AssertionError as ex:
                        raise AssertionError(f"{what}: {ex}") from None
                    img = g.leader.image()
                    assert RE.u64(img, e.at) == e.idx, what
                    if e.ghost:
                        assert RE.u64(img, e.end_before) == e.idx, f"{what}: no ghost header at {e.end_before}"
                    # the launch's range through apus_log_read_range on a follower, across the wrap
                    end = g.leader.offsets()["end"]
                    buf = g.replicas[1].read_range(e.end_before, end, cap=L)
                    pos = (e.end_before + np.arange(AR.dist(e.end_before, end, L))) % L
                    assert np.array_equal(buf, c.image(1)[pos]), f"{what}: read_range [{e.end_before}, {end})"
            EU.compare_group_to_oracle(g, c, exact=True)
            assert g.leader.committed() == sum(1 for s in t.steps if s[0] in ("config", "req", "prune"))
    finally:
        c.close()


# ---- pruning at the ring's end ---------------------------------------------------------------------------------------
def settle(reps, lead, t, timeout=5.0):
    """resident kernels: every follower has acked `t` entries and holds the leader's commit offset, and the leader has
    applied up to its end (the pruning rule reads the leader's own apply offset too)"""
    t0 = time.time()
    while time.time() - t0 < timeout:
        lo = lead.offsets()
        if lo["apply"] == lo["end"] and all(r.stats()["entries_acked"] >= t and r.offsets()["commit"] == lo["commit"]
                                            for r in reps if r is not lead):
            return
        time.sleep(0.001)
    raise AssertionError(f"the group did not settle on {t} entries: leader {lead.offsets()}")


class AutoEngine:
    """ring_edges' driver on the engine: host-applying followers pinned by `pin`, every request in a claim of its own
    (submitted alone, committed and settled before the next), every launch replayed into the oracle.  `express`: the
    leader's express path on (it places single inline requests itself)."""

    def __init__(self, eng, orc, n, L, seed, mode, ctas, express=False):
        self.n, self.L = n, L
        self.express = express
        self.rng = np.random.default_rng(seed)
        self.rid = 1
        self.info = {}
        flags = MODES[mode] | (0 if express else E.F_NO_EXPRESS)
        self.reps = EU.host_apply_replicas(eng, n, L, flags, eng.RING_HOST_MAPPED, 1 << 12, 1 << 22, leader_ctas=ctas)
        self.lead = self.reps[0]
        self.eng = eng
        self.rp = AR.Replay(orc, n, L)
        self.requests = []
        self.prev = 0
        self.pinned = None
        EU.launch_each(eng, self.reps, EU.FOREVER)
        self.pin(0)
        self._put((O.CONFIG, 0, 0, b""), lambda: self.lead.submit(E.CONFIG, 0, 0, E.cid_image(n)))
        self.put((S.CONNECT, 0, 1, b""))

    def close(self):
        try:
            EU.stop_each(self.eng, self.reps)
        finally:
            for r in self.reps:
                r.close()
            self.rp.close()

    @property
    def heads(self):
        return [(h.off, h.value) for h in self.rp.heads]

    def offsets(self):
        return self.rp.c.offsets(0)

    def end(self):
        return self.offsets()["end"]

    def last_ended_at_len(self):
        return self.end() == 0

    def image(self):
        return self.rp.c.image(0)

    def pin(self, v):
        if v != self.pinned:
            pin_and_wait(self.lead, self.reps, [0] + [v] * (self.n - 1))
            self.pinned = v

    def _put(self, r, submit):
        self.requests.append(r)
        t = submit()
        self._done(t)

    def _done(self, t):
        self.lead.wait_committed(t, 10_000_000)
        settle(self.reps, self.lead, t)
        end = self.lead.offsets()["end"]
        self.rp.launch(AR.read_launch(self.lead, self.prev, end, self.L), self.requests)
        self.prev = end

    def put(self, r):
        self._put(r, lambda: self.lead.submit(*r))

    def request(self, stride):
        self.rid += 1
        return (S.SEND, 0, self.rid, self.rng.integers(1, 256, stride - RE.HDR, dtype=np.uint8).tobytes())

    def send(self, stride):
        self.put(self.request(stride))

    def put_held(self, r, release):
        """`r` is held by rule E2: committed() stops moving and the bytes from the head to the end stay as they are;
        then the followers report `release` and it completes"""
        o = self.lead.offsets()
        kept = [rep.read_range(o["head"], o["end"], cap=self.L) for rep in self.reps]
        self.requests.append(r)
        t = self.lead.submit(*r)
        t0, last, still = time.time(), -1, time.time()
        while time.time() - still < 0.3:
            assert time.time() - t0 < 5.0, "the leader kept committing: no back-pressure"
            c = self.lead.committed()
            if c != last:
                last, still = c, time.time()
            time.sleep(0.01)
        assert last == t - 1, (last, t)
        for i, rep in enumerate(self.reps):
            assert np.array_equal(rep.read_range(o["head"], o["end"], cap=self.L), kept[i]), \
                f"replica {i}: bytes of the live range changed while the placement was held"
        self.pin(release)
        self._done(t)

    def check_final(self):
        """every byte, and every offset but the followers' apply (what their host reported), against the replay"""
        EU.stop_each(self.eng, self.reps)
        for i, r in enumerate(self.reps):
            eo, oo = r.offsets(), self.rp.c.offsets(i)
            for key in ("end", "commit", "head"):
                assert eo[key] == oo[key], (i, key, eo, oo)
            d = np.nonzero(r.image() != self.rp.c.image(i))[0]
            assert len(d) == 0, f"replica {i}: {len(d)} bytes differ, first at {int(d[0])}"
        assert self.lead.stats()["auto_heads"] == len(self.rp.heads)


AUTO_L = 1 << 16
AUTO_RUNS = [pytest.param(c.name, 3, mode, ctas, id=f"{c.name}-{mode}-ctas{ctas}")
             for c in RE.auto_cases(AUTO_L) for mode, ctas in (("index_earlyack", 1), ("walk_fenced", 16))]
AUTO_RUNS += [pytest.param(name, 5, "walk_earlyack", 4, id=f"{name}-n5-walk_earlyack-ctas4")
              for name in ("c1-ghost", "c3-head-skip")]


@pytest.mark.parametrize("name,n,mode,ctas", AUTO_RUNS)
def test_pruning_at_the_ring_end(eng, orc, name, n, mode, ctas):
    """the same plan as on the model (test_ring_edges_plan.py), on the engine: the layout is the one the case claims,
    and no HEAD entry stands between a wrapping entry's ghost (or skipped stretch) and the entry"""
    case = next(c for c in RE.auto_cases(AUTO_L) if c.name == name)
    d = AutoEngine(eng, orc, n, AUTO_L, 0xC0 + len(name), mode, ctas)
    try:
        RE.scenario(d, case)
        assert case.got == case.expect, (case.got, case.expect, case.info)
        d.check_final()
    finally:
        d.close()


@pytest.mark.parametrize("name", [c.name for c in RE.e2_cases(AUTO_L)])
def test_e2_boundary_to_the_byte(eng, orc, name):
    """rule E2 with the HEAD reserve: used + stride + 64 (+ the skipped stretch when the entry wraps) == L - 1 places
    and commits; one byte more holds (committed() stops, the live bytes stay), and the followers' release completes it
    behind a HEAD entry, byte-equal to the oracle"""
    case = next(c for c in RE.e2_cases(AUTO_L) if c.name == name)
    d = AutoEngine(eng, orc, 3, AUTO_L, 0xB0 + len(name), "index_fenced", 4)
    try:
        RE.e2_scenario(d, case)
        E = AUTO_L - case.left
        wrap = case.stride > case.left
        assert d.offsets()["tail"] == (0 if wrap else E + (RE.HDR if case.held else 0)), (d.offsets(), case.info)
        d.check_final()
    finally:
        d.close()


def test_c5_head_becomes_the_tail(eng, orc):
    """every replica applied up to the end right after a wrap (d == 0): the HEAD carries the tail, the wrapped entry"""
    d = AutoEngine(eng, orc, 3, AUTO_L, 0xC5, "walk_fenced", 4)
    try:
        assert RE.c5_scenario(d) == (1500, 0, 0)
        d.check_final()
    finally:
        d.close()


@pytest.mark.parametrize("used,want", [(AUTO_L // 2 - 1, False), (AUTO_L // 2, True)], ids=["half-1", "half"])
def test_express_hand_over_at_half_used(eng, orc, used, want):
    """resident kernels, one request in flight, the express path on, the pruning rule due: an inline request at
    L/2 - 1 bytes used is placed by the express path without a HEAD; at L/2 the tile machine puts the HEAD first"""
    d = AutoEngine(eng, orc, 3, AUTO_L, 0xE5, "index_earlyack", 4, express=True)
    try:
        x0 = d.lead.stats()["turn_ns"][5]
        assert RE.express_scenario(d, used) == want
        assert d.lead.stats()["turn_ns"][5] > x0, "the express path placed nothing"
        d.check_final()
    finally:
        d.close()
