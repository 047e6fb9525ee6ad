"""Scenario scripts shared by the golden generator (run against the compiled
reference header) and test_golden.py (run against the restatement, anywhere)."""
import hashlib

import numpy as np

import orc as O
import streams as S


def _h(obj) -> str:
    return hashlib.sha256(repr(obj).encode()).hexdigest()[:16]


def single_log(oracle, name, length, stream, term=1, head_follows=0):
    log = O.Log(oracle, length)
    rets = []
    for k, (typ, clt, rid, payload) in enumerate(stream):
        rets.append(log.append(term, rid, clt, typ, O.cmd_image(payload)))
        if head_follows and k % head_follows == 0:
            o = log.offsets()
            if o["end"] != o["len"]:
                log.set_offsets(head=o["tail"], apply=o["tail"], commit=o["tail"])
    off = log.offsets()
    img = log.image()
    log.close()
    return dict(name=name, offsets=off, rets=_h(rets), n_rets=len(rets), last_ret=rets[-1],
                fnv=f"{O.fnv1a(img) if length <= (1 << 20) else 0:016x}",
                sha=hashlib.sha256(img.tobytes()).hexdigest())


def cluster(oracle, name, n, length, stream, prune_every=0):
    c = O.Cluster(oracle, n, leader=0, term=1, length=length)
    c.prologue()
    cido = [(O.u64)(0) for _ in range(n)]
    heads = []
    for k, (typ, clt, rid, payload) in enumerate(stream):
        c.submit(typ, clt, rid, O.cmd_image(payload))
        if k % 3 == 2:
            c.round()
        if prune_every and k % prune_every == prune_every - 1:
            c.round()
            heads.append(int(c.prune()))
            c.round()
            for i in range(1, n):
                c.poll_head(i, cido[i])
    c.round()
    out = dict(name=name, n=n,
               offsets=[c.offsets(i) for i in range(n)],
               sha=[hashlib.sha256(c.image(i).tobytes()).hexdigest() for i in range(n)],
               applied=[_h(c.applied(i)) for i in range(n)],
               n_applied=[len(c.applied(i)) for i in range(n)],
               heads=_h(heads), bytes_replicated=int(c.bytes_replicated()),
               update_state=int(c.update_state_calls()))
    c.close()
    return out


def last_entry(c, i):
    """(term, idx) of the last entry replica i holds, walking its log from head to end: what it votes on"""
    o = c.offsets(i)
    if o["end"] == o["len"]:
        return (0, 0)
    img = c.image(i)
    ents = O.walk_entries(img, o["head"], o["end"], o["len"])
    if not ents:
        return (0, 0)
    off = ents[-1][0]
    return (int.from_bytes(img[off + 8:off + 16].tobytes(), "little"), int.from_bytes(img[off:off + 8].tobytes(), "little"))


def adjustment_kind(before, c, winner, v, shared):
    """what SIM(adjust) did to voter v: "empty" (it held nothing uncommitted), "lag" (it holds a prefix of the winner's
    log: the shared end is its old end), "term" (cut back where it holds an entry with the winner's offset and idx but
    another term), "cut" (cut back where offset or idx differ too)"""
    bo, bimg = before
    if bo["commit"] == bo["end"]:
        return "empty"
    if shared == bo["end"]:
        return "lag"
    wimg = c.image(winner)
    same_idx = bimg[shared:shared + 8].tobytes() == wimg[shared:shared + 8].tobytes()
    other_term = bimg[shared + 8:shared + 16].tobytes() != wimg[shared + 8:shared + 16].tobytes()
    return "term" if same_idx and other_term else "cut"


def takeover(oracle, name, n, length, seed, laps=2, takeovers=1, max_len=200, check=None, script=None):
    """Leader take-over and log adjustment on a cluster (SIM(take_over), SIM(adjust)).

    Term 1 laps the ring `laps` times with every follower up and the reference's pruning every 5 requests.  Then, per
    take-over: bursts, each received by a subset of the followers (lagging and diverging logs, commit offsets that
    differ); the leader dies; a majority of the survivors elects the most up-to-date of them (last (term, idx)), which
    adopts its voters' commit offsets, appends the blank CONFIG and adjusts every voter: SIM(adjust), then the resend
    (SIM(replicate)).  Then the new term's first requests, again each burst received by a subset.
    Without `script` the subsets and the majority are random, every survivor votes while more take-overs are to come,
    and after a take-over the voters are all up (survivors that did not vote, possible in the last take-over only,
    leave the group).  `script`: per take-over a dict of "bursts" [(requests, live followers)] before the leader dies,
    "group" (the survivors that vote, winner included) and "after" [(requests, live followers)] in the new term --
    a new term's entries can then reach a minority only, and a later winner from the other side truncates them.
    `check(c, winner, voters, before, shared)` runs right after the resend (before: {voter: (offsets, image)} taken
    before the take-over, shared: {voter: the shared end SIM(adjust) returned})."""
    rng = np.random.default_rng(seed)
    it = iter(S.ragged_stream(100_000, max_len, conns=3, seed=seed))

    def submit():
        typ, clt, rid, payload = next(it)
        assert c.submit(typ, clt, rid, O.cmd_image(payload))
        return 64 + len(payload)

    def burst(k, live):
        for _ in range(k):
            submit()
        c.round(live=live)
        c.round(live=live)

    c = O.Cluster(oracle, n, leader=0, term=1, length=length)
    c.prologue()
    cido = [O.u64(0) for _ in range(n)]
    written, k = 0, 0
    while written < laps * length:
        written += submit()
        k += 1
        if k % 3 == 0:
            c.round()
        if k % 5 == 0:
            c.round()
            c.prune()
            c.round()
            for i in range(n):
                if i != c.leader:
                    c.poll_head(i, cido[i])
    c.round()
    takeovers = len(script) if script else takeovers
    alive, term, log = list(range(n)), 1, []
    kinds = {"empty": 0, "lag": 0, "term": 0, "cut": 0}
    for x in range(takeovers):
        lead = c.leader
        others = [i for i in alive if i != lead]
        if script:
            for k, live in script[x]["bursts"]:
                burst(k, live)
        else:
            for _ in range(int(rng.integers(2, 5))):
                live = [int(s) for s in rng.permutation(others)[:int(rng.integers(0, len(others) + 1))]]
                burst(int(rng.integers(1, 8)), live)
        alive.remove(lead)
        q = n // 2 + 1
        if len(alive) < q:
            break
        if script:
            group = script[x]["group"]
            assert set(group) <= set(alive) and len(group) >= q, (group, alive)
        else:
            # every survivor votes while more take-overs are to come (each one costs the group a member)
            size = len(alive) if x < takeovers - 1 else int(rng.integers(q, len(alive) + 1))
            group = [int(s) for s in rng.permutation(alive)[:size]]
        winner = max(group, key=lambda i: (last_entry(c, i), -i))
        voters = sorted(v for v in group if v != winner)
        before = {v: (c.offsets(v), c.image(v)) for v in voters}
        commits = {v: c.offsets(v)["commit"] for v in voters}
        term += 1
        c.take_over(winner, term, commits)
        c.prologue()
        shared = {v: c.adjust(v) for v in voters}
        for v in voters:
            c.replicate(v)
        adj = {v: adjustment_kind(before[v], c, winner, v, shared[v]) for v in voters}
        for v in voters:
            kinds[adj[v]] += 1
        log.append(dict(winner=winner, voters=voters, commits=commits, shared=shared, kinds=adj,
                        last=[last_entry(c, i) for i in range(n)], commit=c.offsets(winner)["commit"]))
        if check:
            check(c, winner, voters, before, shared)
        if script:
            for k, live in script[x]["after"]:
                burst(k, live)
        else:
            burst(0, voters)
            burst(int(rng.integers(3, 12)), voters)
            alive = [winner] + voters
    out = dict(name=name, n=n, takeovers=_h(log), n_takeovers=len(log), kinds=kinds,
               offsets=[c.offsets(i) for i in range(n)],
               sha=[hashlib.sha256(c.image(i).tobytes()).hexdigest() for i in range(n)],
               applied=[_h(c.applied(i)) for i in range(n)], n_applied=[len(c.applied(i)) for i in range(n)])
    c.close()
    return out


TAKEOVER_CASES = [(n, length, seed, takeovers) for n, length, seed, takeovers in
                  [(3, 1 << 14, 1, 1), (3, 1 << 15, 2, 1), (4, 1 << 16, 3, 1), (5, 1 << 14, 4, 2), (5, 1 << 16, 5, 2),
                   (6, 1 << 15, 6, 2), (7, 1 << 14, 7, 3), (7, 1 << 16, 8, 3)]]

# New-term entries that reach a minority only, then a winner from the other side.
#   n5: term 1 ends with a burst that only follower 1 holds; 2 wins term 2 with voters 3 and 4 (1 does not vote), and
#       its blank CONFIG and a burst reach 3 only; 3 wins term 3 with voters 1 and 4.  Follower 1 holds term-1 entries
#       where 3 holds the term-2 CONFIG: same offset, same idx, another term -- cut back, then overwritten.
#   n7: the same with two such followers (1 and 2) and a lagging voter in the third term (the issue's N = 7 case).
CONFLICT_SCRIPTS = {
    "n5": (5, [dict(bursts=[(3, [1, 2, 3, 4]), (5, [1])], group=[2, 3, 4], after=[(2, [3])]),
               dict(bursts=[], group=[1, 3, 4], after=[(0, [1, 4]), (4, [1, 4])])]),
    "n7": (7, [dict(bursts=[(3, [1, 2, 3, 4, 5, 6]), (6, [1, 2])], group=[3, 4, 5, 6], after=[(3, [4])]),
               dict(bursts=[], group=[1, 2, 4, 5], after=[(0, [1, 2, 5]), (5, [1, 2, 5])])]),
}
CONFLICT_CASES = [(name, length, seed) for name in CONFLICT_SCRIPTS for length, seed in ((1 << 14, 21), (1 << 16, 22))]


def conflict_scenario(oracle, name, length, seed, check=None):
    n, script = CONFLICT_SCRIPTS[name]
    return takeover(oracle, f"conflict_{name}_{length >> 10}k_s{seed}", n, length, seed, script=script, check=check)


def takeover_scenarios(oracle):
    return ([takeover(oracle, f"takeover{n}_{length >> 10}k_s{seed}", n, length, seed, takeovers=t)
             for n, length, seed, t in TAKEOVER_CASES] +
            [conflict_scenario(oracle, name, length, seed) for name, length, seed in CONFLICT_CASES])


def all_scenarios(oracle):
    res = []
    res.append(single_log(oracle, "kat7", O.LOG_SIZE,
                          [(O.SEND, 0x0100, i + 1, S.payload_kat(i, ln))
                           for i, ln in enumerate([64, 64, 64, 100, 4096])]
                          + [(O.CONNECT, 0x0100, 6, b"")]))
    res.append(single_log(oracle, "uniform64_x4096", O.LOG_SIZE, S.uniform_stream(4096, 64)))
    res.append(single_log(oracle, "uniform1024_x512_c16", O.LOG_SIZE, S.uniform_stream(512, 1024, conns=16)))
    res.append(single_log(oracle, "ragged300_x2000", O.LOG_SIZE, S.ragged_stream(2000, 300, seed=5, close_every=100)))
    res.append(single_log(oracle, "ragged_wrap_16k", 16384, S.ragged_stream(1500, 200, seed=6), head_follows=5))
    res.append(single_log(oracle, "ragged_wrap_4k", 4096, S.ragged_stream(800, 90, seed=7), head_follows=3))
    res.append(single_log(oracle, "max_len_65535", O.LOG_SIZE,
                          [(O.CONNECT, 1, 1, b"")] + [(O.SEND, 1, 2 + i, bytes([i]) * 65535) for i in range(3)]))
    for n in (1, 3, 5, 7):
        res.append(cluster(oracle, f"cluster{n}_ragged", n, 1 << 20, S.ragged_stream(500, 256, seed=10 + n, close_every=60)))
    res.append(cluster(oracle, "cluster5_uniform64", 5, 1 << 20, S.uniform_stream(2000, 64, conns=4)))
    res.append(cluster(oracle, "cluster3_wrap_prune", 3, 16384, S.ragged_stream(900, 150, conns=2, seed=77), prune_every=5))
    res.append(cluster(oracle, "cluster5_wrap_prune", 5, 32768, S.ragged_stream(1200, 333, conns=3, seed=78), prune_every=7))
    res.extend(takeover_scenarios(oracle))
    return res
