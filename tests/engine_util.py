"""Helpers for the GPU parity tests: run one request stream through the CUDA
engine (via the C ABI) and through the CPU oracle, then compare everything
observable (SURVEY.md s8c "Masking rule for parity")."""
import ctypes as C

import numpy as np

import orc as O

FOREVER = (1 << 64) - 1


def launch_each(eng, reps, target=FOREVER):
    """one launch per replica (followers first): a replica can then be stopped on its own even when several share a GPU"""
    from apus_b200 import engine as E
    for r in sorted(reps, key=lambda r: r.is_leader):
        arr = (C.c_void_p * 1)(r.h)
        E._ck(eng.lib().apus_replicas_launch(arr, 1, target), "apus_replicas_launch")


def stop_each(eng, reps):
    """stop the launches of `reps` (each launched on its own by launch_each)"""
    from apus_b200 import engine as E
    arr = (C.c_void_p * len(reps))(*[r.h for r in reps])
    E._ck(eng.lib().apus_replicas_stop(arr, len(reps)), "apus_replicas_stop")


def oracle_cluster(orc, n, length, stream, rules=O.RULES_ENGINE, prologue=True, leader=0, term=1):
    orc.set_rules(rules)
    c = O.Cluster(orc, n, leader=leader, term=term, length=length)
    if prologue:
        c.prologue()
    for typ, clt, rid, payload in stream:
        idx = c.submit(typ, clt, rid, O.cmd_image(payload))
        assert idx != 0, "oracle refused an append (ring full): shorten the stream or prune"
    for _ in range(2):
        c.round()
    return c


def compare_group_to_oracle(group, c, exact=True):
    """group: apus_b200.Group at quiescence; c: orc.Cluster at quiescence."""
    n, L = group.n, group.replicas[0].log_len
    lead = group.leader_idx
    oo = [c.offsets(i) for i in range(n)]
    eo = [r.offsets() for r in group.replicas]
    for i in range(n):
        assert eo[i]["len"] == oo[i]["len"] == L
        assert eo[i]["end"] == oo[i]["end"], f"replica {i} end {eo[i]} vs {oo[i]}"
        assert eo[i]["commit"] == oo[i]["commit"], f"replica {i} commit {eo[i]} vs {oo[i]}"
        assert eo[i]["apply"] == oo[i]["apply"], f"replica {i} apply {eo[i]} vs {oo[i]}"
    assert eo[lead]["tail"] == oo[lead]["tail"]
    assert eo[lead]["commit"] == eo[lead]["end"], "leader: commit == end at quiescence"
    for i in range(n):
        ei = group.replicas[i].image()
        oi = c.image(i)
        if exact:
            if not np.array_equal(ei, oi):
                d = np.nonzero(ei != oi)[0]
                raise AssertionError(f"replica {i}: {len(d)} bytes differ, first at {int(d[0])} "
                                     f"(engine {ei[d[0]]} oracle {oi[d[0]]}); offsets {eo[i]}")
        else:
            ents = O.walk_entries(oi, 0, oo[i]["end"], L) if oo[i]["end"] != L else []
            assert np.array_equal(O.mask_replies(ei, ents), O.mask_replies(oi, ents))
    # invariant I7: at quiescence the leader holds reply[i]==1 for every follower,
    # follower i holds at least its own byte
    limg = group.replicas[lead].image()
    end = eo[lead]["end"]
    if end != L and eo[lead]["head"] == 0 and end > 0:
        ents = O.walk_entries(limg, 0, end, L)
        for off, _ in ents[-64:]:
            for i in range(n):
                if i != lead:
                    assert limg[off + 28 + i] == 1
    return eo, oo


def host_apply_replicas(eng, n, L, mode, ring_mode, ring_slots, ring_bytes, leader_ctas=4):
    """n connected replicas that prune on the device (APUS_F_AUTOPRUNE) with followers whose host applies the log
    (APUS_F_HOST_APPLY): what a follower's host reports as applied is the apply offset the leader's pruning rule
    reads.  `mode`: the follower mode flags, given to every replica."""
    from apus_b200 import engine as E
    nd = eng.lib().apus_device_count()
    base = E.F_DEVICE_STATS | E.F_AUTOPRUNE | mode
    reps = [E.Replica(i % nd, i, n, 0, 1, L, ring_mode, ring_slots, ring_bytes,
                      base if i == 0 else base | E.F_HOST_APPLY, leader_ctas) for i in range(n)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    return reps
