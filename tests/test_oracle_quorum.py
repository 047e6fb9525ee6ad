"""The oracle's round with only some followers up (orc.Cluster.round(live=...)): the expected-value generator of the
GPU quorum tests (tests/test_gpu_quorum.py), pinned here against a brute-force reading of the commit rule
(dare_ibv_rc.c:1725-1758: an entry commits when its reply bytes plus the leader's own vote reach size/2+1, and the
commit offset is a prefix)."""
import numpy as np
import pytest

import orc as O
import streams as S


def brute_force_commit(img, end, n, leader, L):
    """Offset of the first entry (walking from 0) that fewer than n//2+1 replicas hold, else `end`."""
    for off, _ in O.walk_entries(img, 0, end, L):
        votes = 1 + sum(1 for i in range(n) if i != leader and img[off + 28 + i] == 1)
        if votes < n // 2 + 1:
            return off
    return end


@pytest.mark.parametrize("leader_at", ["first", "last"])
@pytest.mark.parametrize("n", list(range(1, 14)))
def test_partial_round_commits_what_a_majority_holds(orc, n, leader_at):
    leader = 0 if leader_at == "first" else n - 1
    followers = [i for i in range(n) if i != leader]
    L = 1 << 16
    orc.set_rules(O.RULES_ENGINE)
    rng = np.random.default_rng(1000 * n + leader)
    for k in range(len(followers) + 1):                     # every size of live set
        c = O.Cluster(orc, n, leader=leader, term=1, length=L)
        try:
            c.prologue()
            stream = S.ragged_stream(60, 40, conns=2, leader=leader, seed=7 * n + k)
            for typ, clt, rid, payload in stream[:20]:
                assert c.submit(typ, clt, rid, O.cmd_image(payload))
            c.round(); c.round()
            lo = c.offsets(leader)
            assert lo["commit"] == lo["end"]
            # three partial rounds, each with its own live set of size k: entries end up acked by different subsets
            for step in range(3):
                live = set(int(x) for x in rng.choice(followers, size=k, replace=False)) if k else set()
                before = {i: c.offsets(i) for i in followers}
                imgs = {i: c.image(i) for i in followers if i not in live}
                for typ, clt, rid, payload in stream[20 + 10 * step:30 + 10 * step]:
                    assert c.submit(typ, clt, rid, O.cmd_image(payload))
                c.round(live=live)
                lo = c.offsets(leader)
                limg = c.image(leader)
                assert lo["commit"] == brute_force_commit(limg, lo["end"], n, leader, L), (k, step, live)
                if k + 1 >= n // 2 + 1:
                    assert lo["commit"] == lo["end"]
                for i in followers:
                    fo = c.offsets(i)
                    if i in live:
                        assert fo["end"] == lo["end"]
                        assert fo["commit"] == lo["commit"]
                    else:                                   # down: nothing of it moves
                        assert fo == before[i]
                        assert np.array_equal(c.image(i), imgs[i])
                    # invariant I4: a follower's commit never passes its end (no wrap in this ring)
                    assert fo["commit"] <= fo["end"]
        finally:
            c.close()


def test_partial_round_without_live_set_is_the_full_round(orc):
    """round(live=every follower) and round() leave the same cluster."""
    n, L = 5, 1 << 16
    orc.set_rules(O.RULES_ENGINE)
    stream = S.ragged_stream(80, 100, conns=3, seed=5)
    cs = [O.Cluster(orc, n, leader=2, term=1, length=L) for _ in range(2)]
    try:
        for j, c in enumerate(cs):
            c.prologue()
            for typ, clt, rid, payload in stream:
                assert c.submit(typ, clt, rid, O.cmd_image(payload))
            for _ in range(2):
                c.round() if j == 0 else c.round(live={0, 1, 3, 4})
        for i in range(n):
            assert cs[0].offsets(i) == cs[1].offsets(i)
            assert np.array_equal(cs[0].image(i), cs[1].image(i))
    finally:
        for c in cs:
            c.close()
