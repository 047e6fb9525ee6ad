"""Leader take-over and log adjustment in the oracle (SIM(take_over), SIM(adjust) in oracle/cluster_sim.inc): the
restatement of the reference's two log helpers (orc_log.h: log_entries_to_nc_buf, log_find_remote_end_offset) against
the compiled reference header, and the result of an adjustment against a brute-force reading of what it must leave.

The scripts (tests/scenarios.py: takeover) lap 16-64 KiB rings with ragged requests, so ghost headers and exact-fit ends
occur, then let followers lag, kill the leader and elect the most up-to-date member of a majority, one to three times in
a row, at 3-7 replicas.  The random scripts leave voters that lag or hold nothing uncommitted; the conflict scripts
(scenarios.CONFLICT_SCRIPTS) let a new term's entries reach a minority before its leader dies, so a later winner cuts
voters back where they hold an entry with its offset and idx but an older term."""
import numpy as np
import pytest

import orc as O
import scenarios


def entries(img, start, end, length):
    return O.walk_entries(img, start, end, length) if start != end else []


def brute_force_check(c, winner, voters, before, shared):
    """Right after the adjustment and the resend: every voter holds the winner's entries over the winner's [head, end)
    (reply bytes aside: each log holds its own), and its entries up to the shared end are the ones it held before the
    take-over, byte for byte."""
    L = c.len
    wo, wimg = c.offsets(winner), c.image(winner)
    went = entries(wimg, wo["head"], wo["end"], L)
    for v in voters:
        vo, vimg = c.offsets(v), c.image(v)
        assert vo["end"] == wo["end"], f"voter {v}: end {vo['end']}, winner's {wo['end']}"
        mv, mw = O.mask_replies(vimg, went), O.mask_replies(wimg, went)
        for off, stride in went:
            d = np.nonzero(mv[off:off + stride] != mw[off:off + stride])[0]
            assert len(d) == 0, (f"voter {v}: entry idx {int.from_bytes(wimg[off:off + 8].tobytes(), 'little')} at "
                                 f"{off}: byte {off + int(d[0])} differs from the winner's")
        bo, bimg = before[v]
        if bo["end"] == L:
            continue
        kept = entries(bimg, bo["head"], shared[v], L) if shared[v] != L else []
        for off, stride in kept:
            d = np.nonzero(vimg[off:off + stride] != bimg[off:off + stride])[0]
            assert len(d) == 0, (f"voter {v}: entry idx {int.from_bytes(bimg[off:off + 8].tobytes(), 'little')} at "
                                 f"{off}, inside the shared prefix, changed at byte {off + int(d[0])}")
        # the shared end is an entry boundary of the voter's old log, at or before its old end
        if shared[v] != bo["end"]:
            ends = {(o + s) % L for o, s in entries(bimg, bo["head"], bo["end"], L)} | {bo["head"]}
            starts = {o for o, _ in entries(bimg, bo["head"], bo["end"], L)}
            assert shared[v] in ends or shared[v] in starts, f"voter {v}: shared end {shared[v]} is no entry boundary"


@pytest.mark.parametrize("case", scenarios.TAKEOVER_CASES, ids=lambda t: f"n{t[0]}-{t[1] >> 10}k-s{t[2]}-x{t[3]}")
def test_takeover_restatement_equals_reference(orc, ref, case):
    """The same take-over script on both bindings: every offset, image byte, apply trace and shared end equal.
    (Where the reference tree is absent, tests/test_golden.py checks the restatement against the same scripts' vectors.)"""
    if not hasattr(ref.lib, "ref_take_over"):
        pytest.skip("oracle/_ref predates SIM(take_over): rebuild it (make -C oracle ref)")
    n, length, seed, t = case
    orc.set_rules(O.RULES_REFERENCE)
    a = scenarios.takeover(orc, "x", n, length, seed, takeovers=t)
    b = scenarios.takeover(ref, "x", n, length, seed, takeovers=t)
    assert a["n_takeovers"] == t
    assert a == b


@pytest.mark.parametrize("name,length,seed", scenarios.CONFLICT_CASES,
                         ids=[f"{nm}-{ln >> 10}k-s{sd}" for nm, ln, sd in scenarios.CONFLICT_CASES])
def test_truncation_restatement_equals_reference(orc, ref, name, length, seed):
    """Voters cut back across terms, on both bindings: every byte, offset and shared end equal, and the mismatch that
    decides the shared end is the term alone (same offset, same idx)."""
    if not hasattr(ref.lib, "ref_take_over"):
        pytest.skip("oracle/_ref predates SIM(take_over): rebuild it (make -C oracle ref)")
    orc.set_rules(O.RULES_REFERENCE)
    a = scenarios.conflict_scenario(orc, name, length, seed)
    b = scenarios.conflict_scenario(ref, name, length, seed)
    assert a["n_takeovers"] == 2 and a["kinds"]["term"] >= (1 if name == "n5" else 2), a["kinds"]
    assert a == b


@pytest.mark.parametrize("rules", [O.RULES_REFERENCE, O.RULES_ENGINE], ids=["reference", "engine"])
@pytest.mark.parametrize("case", scenarios.TAKEOVER_CASES, ids=lambda t: f"n{t[0]}-{t[1] >> 10}k-s{t[2]}-x{t[3]}")
def test_adjustment_leaves_the_winners_log(orc, case, rules):
    n, length, seed, t = case
    orc.set_rules(rules)
    r = scenarios.takeover(orc, "x", n, length, seed, takeovers=t, check=brute_force_check)
    assert r["n_takeovers"] == t


@pytest.mark.parametrize("rules", [O.RULES_REFERENCE, O.RULES_ENGINE], ids=["reference", "engine"])
@pytest.mark.parametrize("name,length,seed", scenarios.CONFLICT_CASES,
                         ids=[f"{nm}-{ln >> 10}k-s{sd}" for nm, ln, sd in scenarios.CONFLICT_CASES])
def test_truncated_voters_hold_the_winners_log(orc, name, length, seed, rules):
    """The brute-force reading on the conflict scripts: every kind of adjustment occurs (nothing uncommitted, a lagging
    prefix, a cut at a term-only mismatch), and after each one the voters hold exactly the winner's entries."""
    orc.set_rules(rules)
    r = scenarios.conflict_scenario(orc, name, length, seed, check=brute_force_check)
    assert r["n_takeovers"] == 2
    assert r["kinds"]["term"] >= 1 and r["kinds"]["empty"] >= 1 and r["kinds"]["lag"] >= 1, r["kinds"]


def _cluster_with(orc, n, L, plan):
    """a cluster of n, leader 0, term 1, blank CONFIG, then `plan`: [(k requests, live followers)]"""
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, n, leader=0, term=1, length=L)
    c.prologue()
    rid = 1
    for k, live in plan:
        for _ in range(k):
            rid += 1
            assert c.submit(O.SEND, 0, rid, O.cmd_image(bytes([rid & 0xFF]) * (rid % 70)))
        c.round(live=live)
        c.round(live=live)
    return c


def test_winner_adopts_a_voters_larger_commit(orc):
    """N = 5: followers 2-4 down, a burst acked by follower 1 alone; 1 goes down, 2 and 3 come back and the burst
    commits; the leader dies.  1 wins with voters 2 and 3, whose commit offsets lie past its own: it adopts the
    largest, and no follower's commit is ever ahead of the leader's.  The new term commits only with a majority."""
    c = _cluster_with(orc, 5, 1 << 16, [(5, [1, 2, 3, 4]), (8, [1])])
    try:
        c.round(live=[2, 3])
        c.round(live=[2, 3])
        o = {i: c.offsets(i) for i in range(5)}
        assert o[2]["commit"] == o[0]["commit"] == o[0]["end"]
        assert o[1]["commit"] < o[2]["commit"], "follower 1 must lag behind in commit"
        c.take_over(1, 2, {2: o[2]["commit"], 3: o[3]["commit"]})
        assert c.offsets(1)["commit"] == o[2]["commit"], "the winner adopts the largest voter commit"
        c.prologue()
        for v in (2, 3):
            assert c.adjust(v) == o[1]["end"]
        c.round(live=[2])                     # 3 is down: no majority in term 2
        c.round(live=[2])
        wc = c.offsets(1)["commit"]
        assert wc == o[2]["commit"]
        for i in (2, 3):
            assert c.offsets(i)["commit"] <= wc
        c.round(live=[2, 3])
        c.round(live=[2, 3])
        assert c.offsets(1)["commit"] == c.offsets(1)["end"]
    finally:
        c.close()


def test_old_term_entries_commit_with_the_first_new_term_entry(orc):
    """Entries of term 1 that no majority acked before the leader died commit as a prefix of the new leader's blank
    CONFIG, never on their own reply bytes."""
    c = _cluster_with(orc, 5, 1 << 16, [(4, [1, 2, 3, 4]), (6, [1])])
    try:
        o1 = c.offsets(1)
        assert o1["commit"] < o1["end"]
        c.take_over(1, 2, {2: c.offsets(2)["commit"], 3: c.offsets(3)["commit"]})
        c.round(live=[])                      # nothing of the new term yet: the old-term entries stay uncommitted
        assert c.offsets(1)["commit"] == o1["commit"]
        c.prologue()
        for v in (2, 3):
            assert c.adjust(v) == c.offsets(v)["end"]
        c.round(live=[2])                     # the CONFIG held by two of five
        c.round(live=[2])
        assert c.offsets(1)["commit"] == o1["commit"]
        c.round(live=[2, 3])
        c.round(live=[2, 3])
        assert c.offsets(1)["commit"] == c.offsets(1)["end"]
        assert c.offsets(2)["commit"] == c.offsets(1)["end"]
    finally:
        c.close()
