"""The ring-edge plans of tests/ring_edges.py on the oracle alone: every case lands on the edge it claims.  The GPU
file (tests/test_gpu_ring_edges.py) runs the same plans on the engine; a plan that drifted off its byte would pass
there without testing anything, so it fails here instead."""
import numpy as np
import pytest

import ring_edges as RE

@pytest.fixture(scope="module", params=list(RE.TOURS))
def tour(request, orc):
    t = RE.make_tour(orc, request.param)
    yield t
    t.close()


def test_tour_edges_land_where_planned(tour):
    L = tour.L
    assert tour.edges
    for e in tour.edges:
        what = f"{e.kind} at left {e.left} ({e.pos}): {e}"
        assert e.end_before == (L - e.left) % L, what                         # the planned left, exactly
        has_cmd = e.kind != "head"
        assert RE.klass(L, e.end_before, e.stride, has_cmd) == e.expect, what
        at, ghost = RE.landing(L, e.end_before, e.stride, has_cmd)
        assert (e.at, e.ghost) == (at, ghost), what                         # what the oracle did
        if e.expect == "e1":
            assert e.end == 0, what
        else:
            assert e.end == e.at + e.stride, what
        assert e.refusal is not None, what                                   # rule E2 lets it be placed
        if e.expect in ("ghost", "skip") and e.left >= 16:
            assert e.stale, f"the stretch an edge skips holds no bytes of an earlier lap: {what}"
    kinds = {(e.kind, e.expect) for e in tour.edges}
    assert len(kinds) >= 4, kinds
    assert {e.pos for e in tour.edges if e.kind != "head"} == {"first", "middle", "last"}


def test_tour_steps_replay_to_the_same_oracle(orc, tour):
    """the recorded steps alone rebuild the planner's cluster (the GPU test feeds the engine and a fresh oracle from
    them)"""
    import orc as O
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, tour.n, leader=0, term=1, length=tour.L)
    try:
        for s in tour.steps:
            if s[0] == "config":
                c.prologue()
            elif s[0] == "req":
                typ, clt, rid, payload = s[1]
                assert c.submit(typ, clt, rid, O.cmd_image(payload))
            elif s[0] == "run":
                c.round(); c.round()
            elif s[0] == "prune":
                assert c.prune()
        for i in range(tour.n):
            assert c.offsets(i) == tour.c.offsets(i)
            assert np.array_equal(c.image(i), tour.c.image(i))
    finally:
        c.close()


@pytest.mark.parametrize("name", [c.name for c in RE.auto_cases(1 << 16)])
def test_pruning_edge_cases_on_the_model(orc, name):
    """the APUS_F_AUTOPRUNE cases on the oracle with the engine's pruning rule: at the planned end, with the planned
    bytes in use and the followers the planned distance past the head, the append meets the planned edge"""
    L = 1 << 16
    case = next(c for c in RE.auto_cases(L) if c.name == name)
    d = RE.AutoModel(orc, 3, L, seed=0xC0 + len(name))
    try:
        RE.scenario(d, case)
        assert case.got == case.expect, (case.got, case.expect, case.info)
        E = L - case.left
        assert case.info["end_before"] == E
        if case.expect[1] in ("ghost", "skip"):
            assert case.info["at"] == 0
            assert case.info["stale"], "no bytes of an earlier lap at the ring's end"
        if name.startswith("c1"):
            # the rule is not due at the end, and would be if the skipped stretch counted
            assert case.used < L // 4 <= case.used + case.left
    finally:
        d.close()


@pytest.mark.parametrize("name", [c.name for c in RE.e2_cases(1 << 16)])
def test_e2_boundary_on_the_model(orc, name):
    """rule E2 with the HEAD reserve, to the byte: used + stride + 64 (+ the skipped stretch when wrapping) == L - 1
    is placed, one byte more is refused until a HEAD entry moves the head"""
    L = 1 << 16
    case = next(c for c in RE.e2_cases(L) if c.name == name)
    d = RE.AutoModel(orc, 3, L, seed=0xB0 + len(name))
    try:
        RE.e2_scenario(d, case)
        E = L - case.left
        assert case.info["end_before"] == E
        o = d.offsets()
        wrap = case.stride > case.left
        assert o["tail"] == (0 if wrap else E + (RE.HDR if case.held else 0)), (o, case.info)
        assert case.held == (case.extra == 1)
        if wrap:
            assert case.info["stale"]
    finally:
        d.close()


def test_e2_refusal_by_the_replay_predicate():
    """autoprune_replay.placement_refusal at the same bytes: None (the leader blocks) exactly one byte past L - 1"""
    import autoprune_replay as AR
    L = 1 << 16
    for case in RE.e2_cases(L):
        E = L - case.left
        wrap = case.stride > case.left
        used = L - 1 - RE.HDR - case.stride - (case.left if wrap else 0) + case.extra
        why = AR.placement_refusal(L, (E - used) % L, E, case.stride)
        assert (why is None) == (case.extra == 1), (case.name, why)


def test_c5_head_becomes_the_tail_on_the_model(orc):
    """every replica applied up to the end right after a wrap: the HEAD carries the tail, the wrapped entry at 0"""
    L = 1 << 16
    d = RE.AutoModel(orc, 3, L, seed=0xC5)
    try:
        off, v, at = RE.c5_scenario(d)
        assert (off, v, at) == (1500, 0, 0)
    finally:
        d.close()


@pytest.mark.parametrize("used,want", [((1 << 16) // 2 - 1, False), ((1 << 16) // 2, True)])
def test_express_hand_over_on_the_model(orc, used, want):
    """the express path places an inline request below half used without evaluating the rule; at half used it hands
    it to the tile machine, which puts the due HEAD first"""
    d = RE.AutoModel(orc, 3, 1 << 16, seed=0xE5, express=True)
    try:
        assert RE.express_scenario(d, used) == want
    finally:
        d.close()
