"""Helpers for the GPU tests: build and warm the engine, build, run and settle groups, run one request stream through
the CUDA engine (via the C ABI) and through the CPU oracle, then compare everything observable (SURVEY.md s8c "Masking
rule for parity").  Importing this module starts no CUDA context: torch and the library are loaded where they are
used."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import orc as O
import streams as S
from apus_b200 import engine as E

FOREVER = (1 << 64) - 1
QUIET_S = 0.1                    # how long "nothing commits" is watched

MODES = {
    # default: offset index, ack on tail observation
    "index_earlyack": E.F_DEVICE_STATS,
    # reference-like follower: parse the bytes, reply bytes before the ack
    "walk_fenced": E.F_DEVICE_STATS | E.F_FENCED_ACK | E.F_FOLLOWER_WALK,
    "index_fenced": E.F_DEVICE_STATS | E.F_FENCED_ACK,
    "walk_earlyack": E.F_DEVICE_STATS | E.F_FOLLOWER_WALK,
}


# ---- fixtures: a test module imports the ones it uses ----------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    import apus_b200
    if apus_b200.lib().apus_device_count() < 1:
        pytest.fail("no CUDA device visible on a gpu-marked test")
    return apus_b200


def warm_torch():
    """load torch's kernels on every device before replica kernels are resident: a kernel loaded lazily while replica
    kernels run waits for them to end.  PackedConsumer fills int64 offsets and uint8 values."""
    import torch
    for d in range(torch.cuda.device_count()):
        for dt in (torch.uint8, torch.int16, torch.int32, torch.int64):
            x = torch.zeros(16, dtype=dt, device=torch.device("cuda", d))
            x.fill_(1)
            x.clone()
        torch.cuda.synchronize(d)


@pytest.fixture(scope="module", autouse=True)
def torch_module(eng):
    """for the modules that use torch: its kernels warmed before the first test, and the memory it cached handed back to
    the driver after the last (later tests run several replica processes on the same GPU)"""
    warm_torch()
    yield
    import gc
    import torch
    gc.collect()
    if torch.cuda.is_initialized():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


# ---- groups --------------------------------------------------------------------------------------------------------
def devices_for(eng, n):
    nd = eng.lib().apus_device_count()
    return [i % nd for i in range(n)]


def device_group(eng, n, L, **kw):
    """a Group whose requests come through the HBM ring (RING_DEVICE)"""
    return eng.Group(n, devices=devices_for(eng, n), log_size=L, ring_mode=eng.RING_DEVICE, **kw)


def connected(reps):
    """connect every replica of `reps` to every other; returns `reps`"""
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    return reps


def launch_each(eng, reps, target=FOREVER):
    """one launch per replica (followers first): a replica can then be stopped on its own even when several share a GPU"""
    for r in sorted(reps, key=lambda r: r.is_leader):
        arr = (C.c_void_p * 1)(r.h)
        E._ck(eng.lib().apus_replicas_launch(arr, 1, target), "apus_replicas_launch")


def stop_each(eng, reps):
    """stop the launches of `reps` (each launched on its own by launch_each)"""
    arr = (C.c_void_p * len(reps))(*[r.h for r in reps])
    E._ck(eng.lib().apus_replicas_stop(arr, len(reps)), "apus_replicas_stop")


def host_apply_replicas(eng, n, L, mode, ring_mode, ring_slots, ring_bytes, leader_ctas=4):
    """n connected replicas that prune on the device (APUS_F_AUTOPRUNE) with followers whose host applies the log
    (APUS_F_HOST_APPLY): what a follower's host reports as applied is the apply offset the leader's pruning rule
    reads.  `mode`: the follower mode flags, given to every replica."""
    devs = devices_for(eng, n)
    base = E.F_DEVICE_STATS | E.F_AUTOPRUNE | mode
    return connected([E.Replica(devs[i], i, n, 0, 1, L, ring_mode, ring_slots, ring_bytes,
                                base if i == 0 else base | E.F_HOST_APPLY, leader_ctas) for i in range(n)])


def wait_for(cond, what, timeout=10.0):
    t_end = time.time() + timeout
    while not cond():
        assert time.time() < t_end, f"timed out waiting for {what}"
        time.sleep(0.001)


def settle(g, t, timeout=5.0):
    """resident kernels: wait until every follower has acked `t` entries and holds the leader's commit offset (the
    commit push is lazy)"""
    t0 = time.time()
    lo = g.leader.offsets()
    while time.time() - t0 < timeout:
        if all(r.stats()["entries_acked"] >= t and r.offsets()["commit"] == lo["commit"]
               for i, r in enumerate(g.replicas) if i != g.leader_idx):
            return
        time.sleep(0.002)
    raise AssertionError(f"followers did not settle on {t} entries / commit {lo['commit']}")


def pin_and_wait(lead, reps, pins, timeout=5.0):
    """report `pins[i]` as follower i's applied offset (APUS_F_HOST_APPLY) and wait until the leader's pruning rule
    sees them"""
    for i, r in enumerate(reps):
        if i:
            r.set_applied(pins[i])
    t0 = time.time()
    while True:
        seen = lead.remote_apply_offsets()
        if all(seen[i] == pins[i] for i in range(1, len(reps))):
            return
        assert time.time() - t0 < timeout, f"the leader sees apply offsets {seen[:len(reps)]}, pinned {pins}"
        time.sleep(0.001)


# ---- requests ------------------------------------------------------------------------------------------------------
def submit_all(lead, stream):
    """the requests (CONNECT first, then runs of SENDs through apus_submit_uniform where they share a shape)"""
    t, k = 0, 0
    while k < len(stream):
        typ, clt, rid, payload = stream[k]
        j = k + 1
        while (typ == S.SEND and j < len(stream) and stream[j][0] == S.SEND and stream[j][1] == clt and
               stream[j][2] == rid + (j - k) and len(stream[j][3]) == len(payload)):
            j += 1
        while True:
            try:
                if j - k > 1:
                    pl = np.frombuffer(b"".join(p for _, _, _, p in stream[k:j]), dtype=np.uint8)
                    t = lead.submit_uniform(j - k, S.SEND, clt, rid, len(payload), pl) + (j - k) - 1
                else:
                    t = lead.submit(typ, clt, rid, payload)
                break
            except BlockingIOError:                 # a ring smaller than the stream drains while the kernels run
                time.sleep(0.0005)
        k = j
    return t


def tensors(part, device, stride=None):
    """the tailq_entry_t fields of `part` as the CUDA tensors submit_device takes"""
    import torch
    n = len(part)
    if stride is None:
        stride = max([len(p) for *_, p in part] + [1])
    pl = np.zeros((n, stride), dtype=np.uint8)
    for k, (_, _, _, p) in enumerate(part):
        pl[k, :len(p)] = np.frombuffer(p, dtype=np.uint8)
    dev = torch.device("cuda", device)
    return (torch.from_numpy(np.array([t for t, *_ in part], dtype=np.uint8)).to(dev),
            torch.from_numpy(np.array([c for _, c, _, _ in part], dtype=np.uint16).view(np.int16)).to(dev),
            torch.from_numpy(np.array([r for _, _, r, _ in part], dtype=np.uint64).view(np.int64)).to(dev),
            torch.from_numpy(np.array([len(p) for *_, p in part], dtype=np.uint16).view(np.int16)).to(dev),
            torch.from_numpy(pl).to(dev))


def submit_host(g, part):
    """one apus_submit_batch call for `part`"""
    stride = max([len(p) for *_, p in part] + [1])
    pl = np.zeros(len(part) * stride, dtype=np.uint8)
    for k, (_, _, _, p) in enumerate(part):
        pl[k * stride:k * stride + len(p)] = np.frombuffer(p, dtype=np.uint8)
    t0 = g.leader.submit_batch([t for t, *_ in part], [c for _, c, _, _ in part], [r for _, _, r, _ in part],
                               [len(p) for *_, p in part], pl, stride)
    g.tickets = t0 + len(part) - 1
    return t0


# ---- the oracle ----------------------------------------------------------------------------------------------------
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


def _oracle():
    O.build_oracle()
    return O.Oracle("orc")


# ---- laps around a small ring with pruning at quiescent points, against the oracle --------------------------------
def prune_both(g, c):
    """log_pruning (dare_server.c:1996-2067) on both sides: head := min apply, HEAD entry."""
    idx = c.prune()
    if not idx:
        return False
    head = c.offsets(0)["head"]
    g.leader.set_head(head)
    g.submit(E.HEAD, 0, 0, head.to_bytes(8, "little"))
    return True


def wrap_stream(kind, seed, L):
    """ragged<max>: lengths 0..max (ragged1500 with connection churn); u<len>: uniform, enough for 4.5 laps"""
    if kind == "ragged180":
        return S.ragged_stream(max(1500, int(4.5 * L / 150)), 180, conns=3, seed=seed)
    if kind == "ragged1500":
        return S.ragged_stream(int(4.5 * L / 814) + 1, 1500, conns=3, seed=seed, close_every=20)
    size = int(kind[1:])
    return S.uniform_stream(int(4.5 * L / (64 + size)) + 1, size, conns=1, seed=seed)


def submit_part(g, part, uniform):
    """the requests of one launch: one deferred flush, or (uniform) runs of SENDs through apus_submit_uniform"""
    if not uniform:
        g.submit_stream(part)
        return
    k = 0
    while k < len(part):
        typ, clt, rid, payload = part[k]
        j = k + 1
        while (typ == S.SEND and j < len(part) and part[j][0] == S.SEND and part[j][1] == clt and
               part[j][2] == rid + (j - k) and len(part[j][3]) == len(payload)):
            j += 1
        if j - k > 1:
            pl = np.frombuffer(b"".join(p for _, _, _, p in part[k:j]), dtype=np.uint8)
            g.tickets = g.leader.submit_uniform(j - k, S.SEND, clt, rid, len(payload), pl) + (j - k) - 1
        else:
            g.submit(typ, clt, rid, payload)
        k = j


def hole_bytes(img, ents):
    """the bytes no append writes: header bytes 41..47 and the slack behind the data image of every entry"""
    out = []
    for off, stride in ents:
        typ = int(img[off + 26])
        nb = {O.NOOP: 0, O.CONFIG: 16, O.HEAD: 8}.get(typ, 2 + int(img[off + 48]) + 256 * int(img[off + 49]))
        out.append(img[off + 41:off + 48])
        out.append(img[off + 48 + nb:off + stride])
    return np.concatenate(out)


def wrap_case(n, L, kind, seed, mode, step=None, ctas=0, ring="host", id=None):
    return pytest.param(n, L, kind, seed, mode, step, ctas, ring,
                        id=id or f"{kind}-n{n}-{L >> 10}K-{mode}-ctas{ctas or 4}" + ("-device" if ring == "device" else ""))


def wrap_laps_with_pruning(eng, orc, n, L, kind, seed, mode, step, ctas, ring, stream_of=wrap_stream):
    """stream_of(kind, seed, L) over 4+ laps of an L-byte ring, `step` requests a launch (None: about a third of the
    ring), pruned on both sides at quiescent points; every byte against the oracle, and the holes of the last lap
    non-zero"""
    stream = stream_of(kind, seed, L)
    if step is None:
        step = max(1, int(0.3 * L * len(stream) / S.stream_bytes(stream)))
    assert S.stream_bytes(stream) >= 4 * L, (S.stream_bytes(stream), L)          # laps
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, n, leader=0, term=1, length=L)
    c.prologue()
    dev = dict(ring_mode=eng.RING_DEVICE, ring_slots=1 << 12, ring_bytes=1 << 20) if ring == "device" else {}
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=MODES[mode], leader_ctas=ctas, **dev) as g:
        g.prologue()
        total = 1
        marks = []                                          # (log bytes appended so far, leader's end) per launch
        written, prev = 0, c.offsets(0)["end"]
        for k in range(0, len(stream), step):
            part = stream[k:k + step]
            for typ, clt, rid, payload in part:
                assert c.submit(typ, clt, rid, O.cmd_image(payload)) != 0, f"the oracle refused request {rid}"
            c.round(); c.round()
            submit_part(g, part, ring == "device")
            total += len(part)
            g.run()
            if prune_both(g, c):
                total += 1
                c.round(); c.round()
                g.run()
            e = c.offsets(0)["end"]
            written += (e - prev) % L
            prev = e
            marks.append((written, e))
        compare_group_to_oracle(g, c, exact=True)
        # teeth: the entries of the last lap (all still in the ring) keep bytes of earlier laps in their holes, so a
        # prefill that stored zeros or loaded the wrong chunk would have shown in the comparison above
        start = next(e for w, e in marks if written - w < L)
        img = c.image(0)
        ents = O.walk_entries(img, start, prev, L)
        holes = hole_bytes(img, ents)
        assert len(ents) >= 4 * step // 3 or len(ents) >= 100, len(ents)
        assert np.count_nonzero(holes) >= 0.5 * len(holes), (np.count_nonzero(holes), len(holes))
        assert g.leader.committed() == total, (g.leader.committed(), total)
        assert c.offsets(0)["head"] != 0, c.offsets(0)
        # every follower adopted the head carried by the last committed HEAD entry
        # (poll_config_entries, dare_server.c:2163-2186)
        lh = g.leader.offsets()["head"]
        assert lh == c.offsets(0)["head"], (lh, c.offsets(0))
        for i, r in enumerate(g.replicas[1:], 1):
            assert r.offsets()["head"] == lh, (i, r.offsets(), lh)
    c.close()


# ---- worker processes ----------------------------------------------------------------------------------------------
def run_case(path, name, **params):
    """run case `name` of the test module at `path` in a worker process of its own (worker_main)"""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(path), name,
                                                                         json.dumps(params)]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=840)
    print(p.stdout[-4000:])
    assert p.returncode == 0, f"{name} {params}: exit {p.returncode}\n{p.stdout[-3000:]}\n{p.stderr[-6000:]}"


def _engine():
    import apus_b200
    warm_torch()
    return apus_b200


def worker_main(namespace):
    """the worker process of a test module: `python <module> <name> '<json params>'` runs the module's
    case_<name>(eng, orc, **params)"""
    import faulthandler
    name, params = sys.argv[1], json.loads(sys.argv[2]) if len(sys.argv) > 2 else {}
    faulthandler.dump_traceback_later(float(os.environ.get("APUS_CASE_TIMEOUT_S", "780")), exit=True)  # where it hung
    eng_, orc_ = _engine(), _oracle()
    namespace["case_" + name](eng_, orc_, **params)
    print(f"{name} {params}: ok")
