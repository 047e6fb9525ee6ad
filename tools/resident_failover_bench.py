"""How long a group that writes and applies in GPU memory takes to write again after its leader stops: three replicas in
one process on GPU 0 (APUS_RING_DEVICE, APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE), a resident consumer
(tests/devicelogic/resident_rows.cu) on every replica, and a device-side closed loop from the leader's resident submitter
(tests/devicelogic/takeover_submit.cu: one 64 B request in flight, each waiting for its commit).

The leader's application stops (its submitter is detached) once 2000 of its requests have committed; then replica 1
takes over with replica 2's vote, driven as dare_entry.c drives an election (stop, disconnect the dead leader, vote,
set_role, adjust the voter, set_role, the blank CONFIG through the host, launch).  Two arms, alternating trial by trial:

  dormant  replica 1's submitter kernel was launched once, before the group's first launch, and has waited out
           NOT_LEADER since; the winner's first launch hands it the ring
  fresh    replica 1 has no submitter until the take-over: after its launch the host attaches one and launches a new
           submitter kernel

Two gaps on the device clock (%globaltimer, one GPU):
  commit   from the old leader's last commit (apus_last_commit_ns) to the winner's submitter seeing its first ticket
           committed
  applied  from the same point to the first of the winner's rows applied on both surviving consumers (their cursor logs)

Prints JSON lines: the card's name and power limit, read in the same run, one line per trial, one summary per arm.

  python tools/resident_failover_bench.py [--trials 5] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")     # before CUDA starts: a stream per resident kernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import apus_b200 as A  # noqa: E402
import engine_util as EU  # noqa: E402
import resident as R  # noqa: E402
import takeover_submit as TS  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consume_bench import card  # noqa: E402
from consumers import new_stream  # noqa: E402
from shadow import sid  # noqa: E402

N, L = 3, 1 << 24
OLD, NEW = 1 << 16, 4000          # requests handed to the old leader's and to the winner's kernel
STOP_AFTER = 2000                 # the old leader's application stops once this many of its requests committed
PAYLOAD = 64
FLAGS = E.F_DEVICE_STATS | E.F_DEVICE_APPLY | E.F_APPLY_ANY_ROLE


def requests(n, conn, first):
    rng = np.random.default_rng(first)
    return [(E.SEND, conn, first + k, rng.integers(0, 256, PAYLOAD, dtype=np.uint8).tobytes()) for k in range(n)]


def take_over(reps, winner=1, voter=2, dead=0, term=2):
    """dare_entry.c's elect() on stopped replicas: the winner leads in `term` with the voter's vote"""
    lib = E.lib()
    EU.stop_each(A, reps)
    for i in (winner, voter):
        E._ck(lib.apus_replica_disconnect(reps[i].h, dead), "apus_replica_disconnect")
    idx, tm, commit, end = (C.c_uint64() for _ in range(4))
    E._ck(lib.apus_ctl_last_entry(reps[voter].h, C.byref(idx), C.byref(tm), C.byref(commit), C.byref(end)),
          "apus_ctl_last_entry")
    E._ck(lib.apus_ctl_send_vote_ack(reps[voter].h, winner, commit.value), "apus_ctl_send_vote_ack")
    E._ck(lib.apus_replica_set_role(reps[winner].h, winner, term), "apus_replica_set_role (winner)")
    got = C.c_uint64()
    E._ck(lib.apus_ctl_adjust_follower(reps[winner].h, voter, sid(term, 1, winner), C.byref(got)),
          "apus_ctl_adjust_follower")
    E._ck(lib.apus_replica_set_role(reps[voter].h, winner, term), "apus_replica_set_role (voter)")
    for r in reps:
        r.leader = winner
    reps[winner].submit(E.CONFIG, 0, 0, E.cid_image(N))          # the blank CONFIG, before the hand-over
    EU.launch_each(A, [reps[voter], reps[winner]])


def first_row_ns(log, row):
    """the %globaltimer ns of the first pass after which the consumer had written more than `row` rows"""
    return next(t for _, n, t in log if n > row)


def trial(arm):
    reps = EU.connected([E.Replica(0, i, N, 0, 1, L, E.RING_DEVICE, 1 << 16, 1 << 22, FLAGS, 4) for i in range(N)])
    cons, views = [], {}
    try:
        # every array and stream exists before the replica kernels are resident
        subs = {0: TS.Submitter(new_stream(0), requests(OLD, 1, 1), batch=1, mode=TS.WAIT, timeout_s=60),
                1: TS.Submitter(new_stream(0), requests(NEW, 2, 1 << 30), batch=1, mode=TS.WAIT, timeout_s=60)}
        cons = [R.Resident(r, new_stream(0), stride=PAYLOAD, row_cap=1 << 17, log_cap=1 << 17).start() for r in reps]
        if arm == "dormant":
            views[1] = reps[1].submitter_attach(subs[1].stream)
            subs[1].start(views[1])
        EU.launch_each(A, reps)
        base = reps[0].submit(E.CONFIG, 0, 0, E.cid_image(N))
        reps[0].wait_committed(base)
        views[0] = reps[0].submitter_attach(subs[0].stream)
        subs[0].start(views[0])
        EU.wait_for(lambda: reps[0].committed() >= base + STOP_AFTER, "the old leader's requests", timeout=60)
        reps[0].submitter_detach()                                 # the old leader's application stops
        views.pop(0)
        P = reps[0].stats()["tickets_submitted"]
        EU.wait_for(lambda: reps[0].committed() >= P, "the old leader's last ticket", timeout=60)
        EU.wait_for(lambda: all(x.rows_so_far() >= P - base for x in cons), "the old rows", timeout=60)
        t_stop = int(A.lib().apus_last_commit_ns(reps[0].h))
        take_over(reps)
        if arm == "fresh":
            views[1] = reps[1].submitter_attach(subs[1].stream)
            subs[1].start(views[1])
        fail, pub, _ = subs[1].result()
        assert fail is None and pub == NEW, (fail, pub)
        t_commit = subs[1].first_commit_ns()
        for x in cons[1:]:
            x.wait_rows(P - base + NEW)
        applied = max(first_row_ns(x.detach()[2], P - base) for x in cons[1:])
        cons[0].detach()
        reps[1].submitter_detach()
        views.pop(1)
        return {"arm": arm, "old_requests": P - base, "not_leader_polls": subs[1].not_leader(),
                "commit_gap_us": (t_commit - t_stop) / 1e3, "applied_gap_us": (applied - t_stop) / 1e3}
    finally:
        for i in list(views):
            reps[i].submitter_detach()
        for x in cons:
            try:
                x.rep.consumer_detach()
            except E.ApusError:
                pass
        try:
            EU.stop_each(A, reps)
        finally:
            for r in reps:
                r.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available() or A.lib().apus_device_count() < 1:
        raise SystemExit("resident_failover_bench.py: no CUDA device; the engine has no CPU fallback")
    TS.lib()
    R.lib()
    EU.warm_torch()
    lines = [json.dumps({"card": card(), "torch": torch.__version__, "replicas": N, "log_size": L,
                         "payload": PAYLOAD, "old_leader_stops_after": STOP_AFTER, "trials": args.trials})]
    print(lines[0], flush=True)
    got = {"dormant": [], "fresh": []}
    trial("dormant")                                               # warm-up
    for _ in range(args.trials):
        for arm in ("dormant", "fresh"):                           # alternating
            d = trial(arm)
            got[arm].append(d)
            lines.append(json.dumps(d))
            print(lines[-1], flush=True)
    for arm, ds in got.items():
        s = {"arm": arm, "trials": len(ds)}
        for k in ("commit_gap_us", "applied_gap_us"):
            x = np.asarray([d[k] for d in ds])
            s[k + "_median"], s[k + "_min"], s[k + "_max"] = float(np.median(x)), float(x.min()), float(x.max())
        lines.append(json.dumps(s))
        print(lines[-1], flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
