"""Resident submitters (apus_submitter_attach) against the host-driven device submit paths, in bench.py's placement:
five replicas on GPU 0, 16 leader CTAs, a 64 MiB log with device-side pruning, 64 B requests, one resident launch of
the replica kernels for the whole run.

  synth        apus_submit_synth from a host loop (chunks of 32768 requests, retried while the ring is full)
  device512    apus_submit_device in 512-request batches from a host loop (the same tensors each time)
  resident     tests/devicelogic/resident_submit.cu attached for the round: C CTAs reserving B requests at a time,
               writing the slots and publishing the doorbell, with no host call

Two measurements, the legs alternating round by round (one warm-up round, then the timed ones):
  step     2^20 requests, host clock from the first submit until the leader's committed-tickets word reaches the last;
           for the resident legs also until the submitter kernel has ended (its stream synchronised), and its thread 0s'
           %globaltimer ns per phase (size sums, reserves, puts, publishes), summed over the CTAs
  closed   one request in flight: the resident submitter's device clock from before its reserve until it sees its
           ticket committed (its commit poll crosses PCIe), against apus_closed_loop's host clock and the leader's
           device-side commit latency samples

Prints JSON lines: the card's name and power limit, read in the same run, then one line per leg and measurement.

  python tools/resident_submitter_bench.py [--steps 3] [--warmup 1] [--lat 2000] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import apus_b200 as A  # noqa: E402
import submitter as SB  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consume_bench import CTAS, N_REQ, PAYLOAD, REPLICAS, card  # noqa: E402

RESIDENT = [(1, 32), (4, 32), (16, 32), (16, 512), (16, 1)]      # (CTAs, requests per reservation)


def wait_commit(lead, ticket, timeout=120.0):
    t = time.time()
    while lead.committed() < ticket:
        assert time.time() - t < timeout, (lead.committed(), ticket)


def step_synth(lead, req):
    t0 = time.perf_counter()
    k, last = 0, 0
    while k < N_REQ:
        m = min(32768, N_REQ - k)
        try:
            last = lead.submit_synth(m, E.SEND, 2, req + k, PAYLOAD, 7) + m - 1
        except BlockingIOError:
            continue
        k += m
    wait_commit(lead, last)
    return time.perf_counter() - t0, last


def step_device(lead, tens, req):
    t0 = time.perf_counter()
    k, last = 0, 0
    while k < N_REQ:
        try:
            last = lead.submit_device(*tens) + 511
        except BlockingIOError:
            continue
        k += 512
    wait_commit(lead, last)
    return time.perf_counter() - t0, last


def step_resident(lead, sub):
    sub.view = lead.submitter_attach(sub.stream)
    t0 = time.perf_counter()
    sub.start()
    sub.stream.synchronize()
    t_kernel = time.perf_counter() - t0
    wait_commit(lead, lead.stats()["tickets_submitted"])       # the doorbell: the last ticket published
    dt = time.perf_counter() - t0
    fail, pub, _ = sub.result()                                 # (checked outside the timed window)
    assert fail is None and pub == sub.n, (fail, pub)
    lead.submitter_detach()
    return dt, t_kernel, sub.phase_ns()


def closed_resident(lead, sub):
    sub.view = lead.submitter_attach(sub.stream)
    sub.start()
    fail, pub, _ = sub.result()
    assert fail is None and pub == sub.n, (fail, pub)
    lat = sub.latencies_ns()
    lead.submitter_detach()
    return np.asarray(lat, dtype=np.float64)


def pct(x, q):
    return float(np.percentile(np.asarray(x, dtype=np.float64), q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--lat", type=int, default=2000, help="closed-loop requests per round and leg")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available() or A.lib().apus_device_count() < 1:
        raise SystemExit("resident_submitter_bench.py: no CUDA device; the engine has no CPU fallback")
    SB.lib()
    for dt in (torch.uint8, torch.int16, torch.int32, torch.int64):
        torch.zeros(16, dtype=dt, device="cuda:0").clone()
    torch.cuda.synchronize()
    lines = [json.dumps({"card": card(), "torch": torch.__version__, "replicas": REPLICAS, "leader_ctas": CTAS,
                         "log_size": A.LOG_SIZE, "requests_per_step": N_REQ, "payload": PAYLOAD,
                         "closed_loop_requests": args.lat, "resident_configs": RESIDENT})]
    print(lines[0], flush=True)
    reps = [E.Replica(0, i, REPLICAS, 0, 1, A.LOG_SIZE, E.RING_DEVICE, 1 << 21, 1 << 20,
                      E.F_DEVICE_STATS | (E.F_AUTOPRUNE if i == 0 else 0), CTAS) for i in range(REPLICAS)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    lead = reps[0]
    stream = torch.cuda.Stream(device=0)
    rng = np.random.default_rng(5)
    pay = [rng.integers(0, 256, PAYLOAD, dtype=np.uint8).tobytes() for _ in range(64)]
    reqs = [(E.SEND, 2, 0, pay[k & 63]) for k in range(N_REQ)]
    closed = [(E.SEND, 2, 0, pay[k & 63]) for k in range(args.lat)]
    import engine_util as EU
    tens = EU.tensors(reqs[:512], 0)
    # every launch's arrays are made before the replica kernels are resident (the view is set at each attach)
    subs = {(c, b): SB.Submitter(E.SubmitterView(), stream, reqs, batch=b, ctas=c, timeout_s=60) for c, b in RESIDENT}
    closed_sub = SB.Submitter(E.SubmitterView(), stream, closed, batch=1, ctas=1, mode=SB.WAIT, timeout_s=60)
    arr = (E.C.c_void_p * REPLICAS)(*[r.h for r in reps])
    E._ck(E.lib().apus_replicas_launch(arr, REPLICAS, E.UINT64_MAX), "apus_replicas_launch")
    legs = ["synth", "device512"] + [f"resident_c{c}_b{b}" for c, b in RESIDENT]
    step = {w: [] for w in legs}
    kern = {w: [] for w in legs}
    phases = {w: [] for w in legs}
    lat = {w: [] for w in ("resident", "closed_loop_host", "closed_loop_device")}
    try:
        lead.wait_committed(lead.submit(E.CONFIG, 0, 0, E.cid_image(REPLICAS)))
        req = 1
        for s in range(args.warmup + args.steps):
            for w in legs:                                          # alternating
                if w == "synth":
                    dt, _ = step_synth(lead, req)
                elif w == "device512":
                    dt, _ = step_device(lead, tens, req)
                else:
                    c, b = (int(x[1:]) for x in w.split("_")[1:])
                    dt, tk, ph = step_resident(lead, subs[(c, b)])
                    print(f"[{w}] round {s}: submitter kernel ended after {tk * 1e3:.1f} ms, phases {ph}",
                          file=sys.stderr, flush=True)
                    if s >= args.warmup:
                        kern[w].append(tk)
                        phases[w].append(ph)
                req += N_REQ
                print(f"[{w}] round {s}: step {dt * 1e3:.1f} ms", file=sys.stderr, flush=True)
                if s >= args.warmup:
                    step[w].append(dt)
            res = closed_resident(lead, closed_sub)
            host = lead.closed_loop(args.lat, PAYLOAD, 2, req).astype(np.float64)
            dev = np.asarray(lead.latency_ns(args.lat), dtype=np.float64)
            req += args.lat
            print(f"[closed] round {s}: resident p50 {pct(res, 50) / 1e3:.2f} us, apus_closed_loop host p50 "
                  f"{pct(host, 50) / 1e3:.2f} us, device p50 {pct(dev, 50) / 1e3:.2f} us", file=sys.stderr, flush=True)
            if s >= args.warmup:
                lat["resident"].extend(res.tolist())
                lat["closed_loop_host"].extend(host.tolist())
                lat["closed_loop_device"].extend(dev.tolist())
    finally:
        E._ck(E.lib().apus_replicas_stop(arr, REPLICAS), "apus_replicas_stop")
    for w in legs:
        d = {"leg": w, "rounds": args.steps, "step_ms": [round(x * 1e3, 3) for x in step[w]],
             "step_ms_median": float(np.median(step[w])) * 1e3,
             "requests_per_s_median": N_REQ / float(np.median(step[w]))}
        if kern[w]:
            d["submitter_kernel_ms"] = [round(x * 1e3, 3) for x in kern[w]]
            d["thread0_phase_ms_summed_over_ctas"] = [{k: round(v / 1e6, 3) for k, v in ph.items()} for ph in phases[w]]
        lines.append(json.dumps(d))
        print(lines[-1], flush=True)
    for w, x in lat.items():
        lines.append(json.dumps({"closed_loop": w, "samples": len(x), "p50_us": pct(x, 50) / 1e3,
                                 "p99_us": pct(x, 99) / 1e3}))
        print(lines[-1], flush=True)
    for r in reps:
        r.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
