"""Follower-side consumption of committed entries, device against host, in bench.py's placement: five replicas on GPU 0,
16 leader CTAs, a 64 MiB ring, 2^20 requests of 64 B per step from apus_submit_synth, device-side pruning.

  device  every follower is created with APUS_F_DEVICE_APPLY; a host thread per follower calls apus_consume_device
          (max_n 2^16, stride 64) in a loop on its own stream, with CUDA events around each call
  host    every follower is created with APUS_F_HOST_APPLY; a host thread per follower does what follower_pump does:
          apus_log_read_range of [apply, commit), a walk over the entries in C (log_get_entry / log_fit_entry /
          log_entry_len, reading the fields do_action takes; compiled into a temporary directory at start-up),
          apus_set_applied

Each step is one bounded launch; the consumers run beside it, and the leader prunes behind what they have applied.
The two ways alternate, step by step.  Prints JSON lines: per way, the replica kernel time per launch (CUDA events of
the launch), and for `device` the entries/s and GB/s per follower from the events around the consume calls (bytes from
shapes: the 64 B header and the cmd read, the row written); the card's name and power limit read in the same run.

  python tools/consume_bench.py [--steps 3] [--warmup 1] [--out FILE]

--leg any_role: what APUS_F_APPLY_ANY_ROLE costs the latency path.  Two groups of five replicas on GPU 0, device
consumers on every follower; the leader of one is created with APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE (the express
path's fence before its publish record, the commit warp's acquire and consumer record), the other's without.  Each
round resident-launches one group, runs apus_closed_loop (one 64 B request in flight: the express path), stops it; the
groups alternate.  Prints per group the host-clock p50 / p99 of the closed loop and the device-clock commit latency
(APUS_F_DEVICE_STATS samples), and checks afterwards that the flagged leader's own consumer delivers every request.

  python tools/consume_bench.py --leg any_role [--steps 5] [--warmup 1] [--out FILE]
"""
import argparse
import json
import os
import ctypes
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

if any("any_role" in a for a in sys.argv[1:]):
    # two groups' streams beside resident launches (the default consume leg keeps the default 8 queues it was measured with)
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import numpy as np  # noqa: E402
import torch  # noqa: E402

import apus_b200 as A  # noqa: E402
from apus_b200 import engine as E  # noqa: E402

N_REQ = 1 << 20
REPLICAS, CTAS, PAYLOAD = 5, 16, 64
MAX_N = 1 << 16
ROW_BYTES = 8 + 1 + 2 + 8 + 2 + PAYLOAD          # idx, type, conn, req_id, len, cmd


WALK_C = r"""
#include <stdint.h>
#include <string.h>
/* the entries in buf[0, n), ring bytes read from ring offset `start` of a ring of L bytes: the walk of follower_pump
 * (a header that does not fit before the ring's end, or an entry that would cross it, continues at 0).  Returns the
 * entries walked; *fold gathers the fields do_action takes so that the reads are not optimised away. */
uint64_t walk(const uint8_t *buf, uint64_t n, uint64_t start, uint64_t L, uint64_t *fold)
{
    uint64_t off = 0, cnt = 0, f = 0;
    while (off < n) {
        const uint64_t pos = (start + off) % L;
        if (L - pos < 64) { off += L - pos; continue; }
        if (off + 64 > n) break;
        const uint8_t *e = buf + off;
        const uint32_t ty = e[26];
        uint16_t len = 0;
        if (ty != 0 && ty != 2 && ty != 3) memcpy(&len, e + 48, 2);
        const uint64_t es = 64u + len;
        if (L - pos < es) { off += L - pos; continue; }
        if (off + es > n) break;
        uint64_t req; uint16_t clt;
        memcpy(&req, e + 16, 8); memcpy(&clt, e + 24, 2);
        f += req ^ clt ^ ty ^ (len ? e[50] ^ e[49 + len] : 0);
        off += es;
        cnt++;
    }
    *fold += f;
    return cnt;
}
"""


def load_walk():
    d = tempfile.mkdtemp(prefix="consume_bench_")
    src, so = os.path.join(d, "walk.c"), os.path.join(d, "walk.so")
    with open(src, "w") as f:
        f.write(WALK_C)
    subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-o", so, src], check=True)
    lib = ctypes.CDLL(so)
    lib.walk.restype = ctypes.c_uint64
    lib.walk.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64,
                         ctypes.POINTER(ctypes.c_uint64)]
    return lib


WALK = None
APPLIED = {}      # host route: the offset each follower's pump has reported, carried from launch to launch


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def make_group(way):
    base = E.F_DEVICE_STATS
    fl = E.F_DEVICE_APPLY if way == "device" else E.F_HOST_APPLY
    reps = [E.Replica(0, i, REPLICAS, 0, 1, A.LOG_SIZE, E.RING_DEVICE, 1 << 21, 1 << 20,
                      base | E.F_AUTOPRUNE if i == 0 else base | fl, CTAS) for i in range(REPLICAS)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    return reps


def host_pump(r, stop, counts, k):
    """follower_pump's route: read the committed range through the pinned bounce buffer, walk the entries, report"""
    L = r.log_len
    apply = APPLIED.get(r.idx, 0)
    fold = ctypes.c_uint64(0)
    while True:
        commit, _ = r.progress()
        if commit == apply:
            if stop.is_set():
                APPLIED[r.idx] = apply
                return
            time.sleep(0.0001)
            continue
        buf = r.read_range(apply, commit, cap=L)
        n = WALK.walk(buf.ctypes.data, len(buf), apply, L, ctypes.byref(fold))
        apply = (apply + len(buf)) % L                      # the read ended on a commit offset: an entry boundary
        r.set_applied(apply)
        counts[k] += n


def device_pump(r, stop, counts, k, times):
    st = torch.cuda.Stream(device=0)
    out = None
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        out = r.consume_device(MAX_N, PAYLOAD, out=out, stream=st)
        e1.record(st)
        st.synchronize()
        got = int(out[6].cpu()[0])
        if got:
            times[k].append((got, e0.elapsed_time(e1)))
            counts[k] += got
        elif stop.is_set():
            return
        assert r.consume_status().error == 0


def run_step(way, reps, req, seed):
    lead = reps[0]
    t = lead.submit_synth(N_REQ, E.SEND, 0, req, PAYLOAD, seed) + N_REQ - 1
    stop = threading.Event()
    counts = [0] * (REPLICAS - 1)
    times = [[] for _ in range(REPLICAS - 1)]
    if way == "device":
        th = [threading.Thread(target=device_pump, args=(r, stop, counts, k, times)) for k, r in enumerate(reps[1:])]
    else:
        th = [threading.Thread(target=host_pump, args=(r, stop, counts, k)) for k, r in enumerate(reps[1:])]
    for x in th:
        x.start()
    arr = (E.C.c_void_p * REPLICAS)(*[r.h for r in reps])
    E._ck(E.lib().apus_replicas_launch(arr, REPLICAS, t), "apus_replicas_launch")
    for r in reps:
        r.wait(300_000)
    stop.set()
    for x in th:
        x.join(300)
    return t, lead.last_launch_ms(), counts, times


LOOP_N = 20000        # closed-loop requests per round (--leg any_role)


def any_role_group(flagged):
    ff = E.F_DEVICE_STATS | E.F_DEVICE_APPLY | (E.F_APPLY_ANY_ROLE if flagged else 0)
    reps = [E.Replica(0, i, REPLICAS, 0, 1, A.LOG_SIZE, E.RING_HOST_MAPPED, 0, 0,
                      ff if (i != 0 or flagged) else E.F_DEVICE_STATS, 0) for i in range(REPLICAS)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    return reps


def any_role_leg(args):
    lines = [json.dumps({"leg": "any_role", "card": card(), "torch": torch.__version__, "replicas": REPLICAS,
                         "requests_per_round": LOOP_N, "payload": PAYLOAD})]
    print(lines[0], flush=True)
    groups = {w: any_role_group(w == "any_role") for w in ("plain", "any_role")}
    res = {w: {"host_ns": [], "dev_ns": []} for w in groups}
    rid = {w: 1 for w in groups}
    for w, reps in groups.items():
        reps[0].submit(E.CONFIG, 0, 0, E.cid_image(REPLICAS))
    for s in range(args.warmup + args.steps):
        for w in ("plain", "any_role"):                           # alternating
            reps = groups[w]
            arr = (E.C.c_void_p * REPLICAS)(*[r.h for r in reps])
            E._ck(E.lib().apus_replicas_launch(arr, REPLICAS, E.UINT64_MAX), "apus_replicas_launch")
            n0 = reps[0].stats()["lat_samples"]
            lat = reps[0].closed_loop(LOOP_N, PAYLOAD, 7, rid[w])
            rid[w] += LOOP_N
            dev = reps[0].latency_ns(LOOP_N)
            E._ck(E.lib().apus_replicas_stop(arr, REPLICAS), "apus_replicas_stop")
            for r in reps:
                r.wait(60_000)
            got = reps[0].stats()["lat_samples"] - n0
            print(f"[{w}] round {s}: host p50 {np.percentile(lat, 50) / 1e3:.2f} us, device samples {got}",
                  file=sys.stderr, flush=True)
            if s >= args.warmup:
                res[w]["host_ns"].extend(int(x) for x in lat)
                res[w]["dev_ns"].extend(int(x) for x in dev[-min(got, LOOP_N):])
    # the flagged leader's own consumer: every request it committed, in order
    lead = groups["any_role"][0]
    rows, out = 0, None
    while True:
        out = lead.consume_device(MAX_N, PAYLOAD, out=out)
        torch.cuda.synchronize(0)
        k = int(out[6].cpu()[0])
        rows += k
        if k == 0:
            break
    st = lead.consume_status()
    assert st.error == 0 and rows == rid["any_role"] - 1, (rows, rid["any_role"] - 1, st)
    for w in ("plain", "any_role"):
        h, d = np.asarray(res[w]["host_ns"]), np.asarray(res[w]["dev_ns"])
        lines.append(json.dumps({"group": w, "rounds": args.steps, "requests": int(len(h)),
                                 "host_p50_us": float(np.percentile(h, 50)) / 1e3,
                                 "host_p99_us": float(np.percentile(h, 99)) / 1e3,
                                 "device_p50_us": float(np.percentile(d, 50)) / 1e3 if len(d) else None,
                                 "device_p99_us": float(np.percentile(d, 99)) / 1e3 if len(d) else None,
                                 "leader_rows_consumed": rows if w == "any_role" else None}))
        print(lines[-1], flush=True)
    for reps in groups.values():
        for r in reps:
            r.close()
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    ap.add_argument("--leg", choices=["consume", "any_role"], default="consume")
    args = ap.parse_args()
    if not torch.cuda.is_available() or A.lib().apus_device_count() < 1:
        raise SystemExit("consume_bench.py: no CUDA device; the engine has no CPU fallback")
    if args.leg == "any_role":
        torch.zeros(1, device="cuda:0").clone()
        torch.cuda.synchronize()
        lines = any_role_leg(args)
        if args.out:
            with open(args.out, "w") as f:
                f.write("\n".join(lines) + "\n")
        return
    global WALK
    WALK = load_walk()
    torch.zeros(1, device="cuda:0").clone()
    torch.cuda.synchronize()
    lines = [json.dumps({"card": card(), "torch": torch.__version__, "replicas": REPLICAS, "leader_ctas": CTAS,
                         "log_size": A.LOG_SIZE, "requests_per_step": N_REQ, "payload": PAYLOAD, "max_n": MAX_N})]
    print(lines[0], flush=True)
    groups = {w: make_group(w) for w in ("device", "host")}
    for w, reps in groups.items():
        reps[0].submit(E.CONFIG, 0, 0, E.cid_image(REPLICAS))
        reps[0].submit(E.CONNECT, 0, 1, b"")
    req = {w: 2 for w in groups}
    res = {w: {"launch_ms": [], "entries": [], "calls": []} for w in groups}
    for s in range(args.warmup + args.steps):
        for w in ("device", "host"):                              # alternating
            t, ms, counts, times = run_step(w, groups[w], req[w], 0xC0 + s)
            req[w] += N_REQ
            print(f"[{w}] step {s}: tickets {t}, launch {ms:.1f} ms, entries per follower {counts}", file=sys.stderr,
                  flush=True)
            if s >= args.warmup:
                res[w]["launch_ms"].append(ms)
                res[w]["entries"].append(counts)
                res[w]["calls"].append(times)
    for w in ("device", "host"):
        r = res[w]
        out = {"way": w, "steps": args.steps, "launch_ms": r["launch_ms"],
               "launch_ms_median": float(np.median(r["launch_ms"]))}
        if w == "device":
            per = []
            for k in range(REPLICAS - 1):
                n = sum(g for st in r["calls"] for g, _ in st[k])
                ms = sum(m for st in r["calls"] for _, m in st[k])
                calls = sum(len(st[k]) for st in r["calls"])
                per.append({"follower": k + 1, "entries": n, "calls": calls, "consume_ms": ms,
                            "entries_per_s": n / (ms / 1e3) if ms else None,
                            "gb_per_s": n * (64 + PAYLOAD + ROW_BYTES) / (ms / 1e3) / 1e9 if ms else None})
            out["per_follower"] = per
        else:
            out["entries_walked_per_follower"] = [sum(c[k] for c in r["entries"]) for k in range(REPLICAS - 1)]
        lines.append(json.dumps(out))
        print(lines[-1], flush=True)
    for reps in groups.values():
        for r in reps:
            r.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
