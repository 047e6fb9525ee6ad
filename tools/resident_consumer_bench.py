"""Resident consumers (apus_consumer_attach) against consumers that wait for commits in stream order
(apus_consume_wait), in bench.py's placement: five replicas on GPU 0, 16 leader CTAs, a 64 MiB log with device-side
pruning, 64 B requests, one resident launch for the whole run.  Every follower consumes on the device.

  waited    consume_wait_bench.py's waited leg: a host thread per follower enqueues K iterations of
            consume_wait(1) -> consume_device -> apply ahead, and the apply kernel stamps %globaltimer when rows came
  resident  tests/devicelogic/resident_rows.cu on every follower, attached for the round: one persistent CTA that
            polls the consumer record, writes the rows and moves the cursor; its cursor log stamps %globaltimer
            when each row lands

Three measurements, the legs alternating round by round (one warm-up round, then the timed ones):
  step     2^20 requests from apus_submit_synth, host clock from the submit until every follower has examined every
           entry (its consume status) and its consumer has ended
  latency  single 64 B requests in a closed loop (apus_submit, then wait until every follower has applied it): the
           follower's stamp minus the leader's apus_last_commit_ns, both %globaltimer on the one GPU
  group    the leader's own closed loop (apus_closed_loop: host clock, and the device-side commit latency samples)
           with the four resident consumers attached and polling, against none: their back-off must not cost the
           replica kernels

Prints JSON lines: the card's name and power limit, read in the same run, then one line per leg and measurement.

  python tools/resident_consumer_bench.py [--steps 3] [--warmup 1] [--lat 1000] [--k 8] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import apus_b200 as A  # noqa: E402
import consume_wait_bench as CW  # noqa: E402
import resident as R  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consume_bench import CTAS, N_REQ, PAYLOAD, REPLICAS, card  # noqa: E402

GROUP_LAT = 2000          # closed-loop requests of the leader's own loop per round and leg


def resident_start(res):
    for x in res:
        x.start()


def resident_stop(res):
    out = []
    for x in res:
        why, n, lg = x.detach()
        assert why == R.END_STOP, why
        out.append((n, lg))
    return out


def all_examined(lead, reps, t):
    lead.wait_committed(t, 60_000_000)
    last = lead.stats()["entries_published"]
    while any(r.consume_status().next_idx <= last for r in reps):
        time.sleep(0.0001)
    for r in reps:
        assert r.consume_status().error == 0


def step_round(leg, lead, fol, res, req, seed, k):
    if leg == "waited":
        stop, lock, th = CW.start("waited", fol, k)
    else:
        resident_start(res)
    t0 = time.perf_counter()
    t = lead.submit_synth(N_REQ, E.SEND, 0, req, PAYLOAD, seed) + N_REQ - 1
    all_examined(lead, [f.rep for f in fol], t)
    if leg == "waited":
        CW.finish("waited", fol, stop, lock, th)
    else:
        got = resident_stop(res)
        assert all(n == N_REQ for n, _ in got), [n for n, _ in got]
    return time.perf_counter() - t0


def latency_round(leg, lead, fol, res, stamps, req, n, k):
    """commit-to-applied of n single requests, ns on %globaltimer, one list per request (one value per follower)"""
    pl = bytes(PAYLOAD)
    commit_ns = []
    if leg == "waited":
        stop, lock, th = CW.start("waited", fol, k)
        out = []
        for i in range(n):
            before = stamps.copy()
            t = lead.submit(E.SEND, 1, req + i, pl)
            lead.wait_committed(t, 10_000_000)
            c_ns = lead.last_commit_ns()
            t_end = time.time() + 10
            while np.any(stamps == before):
                assert time.time() < t_end, "a follower did not apply a committed request within 10 s"
                time.sleep(0.00005)
            out.append([int(s) - c_ns for s in stamps])
        all_examined(lead, [f.rep for f in fol], t)
        CW.finish("waited", fol, stop, lock, th)
        return out
    resident_start(res)
    for i in range(n):
        t = lead.submit(E.SEND, 1, req + i, pl)
        lead.wait_committed(t, 10_000_000)
        commit_ns.append(lead.last_commit_ns())
        t_end = time.time() + 10
        while any(x.rows_so_far() < i + 1 for x in res):
            assert time.time() < t_end, "a follower did not apply a committed request within 10 s"
            time.sleep(0.00005)
    all_examined(lead, [x.rep for x in res], t)
    got = resident_stop(res)
    out = [[0] * len(res) for _ in range(n)]
    for j, (rows, lg) in enumerate(got):
        assert rows == n, rows
        prev = 0
        for _, r, ns in lg:                      # the advance that brought row r lands it at ns
            if r > prev:
                out[r - 1][j] = ns - commit_ns[r - 1]
                prev = r
    return out


def group_round(lead, res, req, attached):
    if attached:
        resident_start(res)
    host = lead.closed_loop(GROUP_LAT, PAYLOAD, 2, req)
    dev = lead.latency_ns(GROUP_LAT)
    if attached:                                   # (the rows of the round without consumers come first)
        for n, _ in resident_stop(res):
            assert n >= GROUP_LAT, n
    return host.astype(np.float64), np.asarray(dev, dtype=np.float64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--lat", type=int, default=1000, help="closed-loop requests per round and leg")
    ap.add_argument("--k", type=int, default=8, help="waited leg: iterations per batch")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available() or A.lib().apus_device_count() < 1:
        raise SystemExit("resident_consumer_bench.py: no CUDA device; the engine has no CPU fallback")
    CW.APPLY = CW.load_apply()
    R.lib()
    for dt in (torch.uint8, torch.int16, torch.int32, torch.int64):
        torch.zeros(16, dtype=dt, device="cuda:0").clone()
    torch.cuda.synchronize()
    lines = [json.dumps({"card": card(), "torch": torch.__version__, "replicas": REPLICAS, "leader_ctas": CTAS,
                         "log_size": A.LOG_SIZE, "requests_per_step": N_REQ, "payload": PAYLOAD, "k_ahead": args.k,
                         "latency_requests": args.lat, "group_latency_requests": GROUP_LAT})]
    print(lines[0], flush=True)
    reps = [E.Replica(0, i, REPLICAS, 0, 1, A.LOG_SIZE, E.RING_DEVICE, 1 << 21, 1 << 20,
                      E.F_DEVICE_STATS | (E.F_AUTOPRUNE if i == 0 else E.F_DEVICE_APPLY), CTAS) for i in range(REPLICAS)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    stamps_t = torch.zeros(REPLICAS - 1, dtype=torch.int64).pin_memory()
    stamps = stamps_t.numpy()
    fol = [CW.Follower(r, stamps_t.data_ptr() + 8 * k) for k, r in enumerate(reps[1:])]
    res = [R.Resident(r, CW.new_stream(r.device), stride=PAYLOAD, row_cap=N_REQ + 4096, log_cap=N_REQ + 4096)
           for r in reps[1:]]
    lead = reps[0]
    arr = (E.C.c_void_p * REPLICAS)(*[r.h for r in reps])
    E._ck(E.lib().apus_replicas_launch(arr, REPLICAS, E.UINT64_MAX), "apus_replicas_launch")
    legs = ("waited", "resident")
    out = {w: {"step_s": [], "lat_ns": []} for w in legs}
    grp = {a: {"host": [], "dev": []} for a in ("none", "attached")}
    try:
        lead.wait_committed(lead.submit(E.CONFIG, 0, 0, E.cid_image(REPLICAS)))
        req = 1
        for s in range(args.warmup + args.steps):
            for w in legs:                                          # alternating
                dt = step_round(w, lead, fol, res, req, 0xE0 + s, args.k)
                req += N_REQ
                lat = latency_round(w, lead, fol, res, stamps, req, args.lat, args.k)
                req += args.lat
                p50 = np.percentile(np.asarray(lat), 50) / 1e3
                print(f"[{w}] round {s}: step {dt * 1e3:.1f} ms, commit-to-applied p50 {p50:.2f} us", file=sys.stderr,
                      flush=True)
                if s >= args.warmup:
                    out[w]["step_s"].append(dt)
                    out[w]["lat_ns"].extend(lat)
            for a in ("none", "attached"):
                host, dev = group_round(lead, res, req, a == "attached")
                req += GROUP_LAT
                print(f"[group, consumers {a}] round {s}: host p50 {np.percentile(host, 50) / 1e3:.2f} us, device p50 "
                      f"{np.percentile(dev, 50) / 1e3:.2f} us", file=sys.stderr, flush=True)
                if s >= args.warmup:
                    grp[a]["host"].extend(host.tolist())
                    grp[a]["dev"].extend(dev.tolist())
    finally:
        E._ck(E.lib().apus_replicas_stop(arr, REPLICAS), "apus_replicas_stop")
    for w in legs:
        r = out[w]
        lat = np.asarray(r["lat_ns"], dtype=np.float64)
        lines.append(json.dumps({
            "leg": w, "rounds": args.steps,
            "step_ms": [round(x * 1e3, 3) for x in r["step_s"]],
            "step_ms_median": float(np.median(r["step_s"])) * 1e3,
            "commit_to_applied_samples": int(lat.size),
            "commit_to_applied_p50_us": float(np.percentile(lat, 50)) / 1e3,
            "commit_to_applied_p99_us": float(np.percentile(lat, 99)) / 1e3}))
        print(lines[-1], flush=True)
    for a in ("none", "attached"):
        h, d = np.asarray(grp[a]["host"]), np.asarray(grp[a]["dev"])
        lines.append(json.dumps({
            "group_closed_loop": a, "resident_consumers": 0 if a == "none" else REPLICAS - 1, "rounds": args.steps,
            "host_samples": int(h.size), "host_p50_us": float(np.percentile(h, 50)) / 1e3,
            "host_p99_us": float(np.percentile(h, 99)) / 1e3,
            "device_samples": int(d.size), "device_p50_us": float(np.percentile(d, 50)) / 1e3,
            "device_p99_us": float(np.percentile(d, 99)) / 1e3}))
        print(lines[-1], flush=True)
    for r in reps:
        r.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
