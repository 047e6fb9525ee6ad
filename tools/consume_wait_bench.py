"""Device consumers that wait for commits on the device (apus_consume_wait) against consumers polled by the host, in
bench.py's placement: five replicas on GPU 0, 16 leader CTAs, a 64 MiB log with device-side pruning, 64 B requests,
one resident launch for the whole run.  Every follower consumes on the device (APUS_F_DEVICE_APPLY) and runs a small
apply kernel after each consume call: one thread adds the call's row count to an applied counter and, when rows came,
stamps %globaltimer into a pinned word.

  polled  consume_bench.py's device_pump, plus the apply kernel: a host thread per follower calls consume_device
          (max_n 2^16, stride 64), then synchronises the stream and reads the count, in a loop
  waited  a host thread per follower enqueues K iterations of consume_wait(1) -> consume_device -> apply ahead, keeps
          two such batches in flight and synchronises once per batch

Two measurements per leg, the legs alternating round by round:
  step     2^20 requests from apus_submit_synth, host clock from the submit until every follower has examined every
           entry (its consume status) and its pump has ended in a synchronise; and the host CPU time of the pump
           threads (time.thread_time)
  latency  single 64 B requests in a closed loop (apus_submit, then wait until every follower's stamp moved): the
           stamp minus the leader's apus_last_commit_ns, both %globaltimer on the one GPU

The apply kernel is compiled with nvcc into a temporary directory at start-up.  Prints JSON lines: the card's name
and power limit, read in the same run, then one line per leg.

  python tools/consume_wait_bench.py [--steps 3] [--warmup 1] [--lat 1000] [--k 8] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

# four follower pump streams and the engine's three streams per replica beside a resident launch (DESIGN.md s2)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import apus_b200 as A  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consume_bench import CTAS, MAX_N, N_REQ, PAYLOAD, REPLICAS, card  # noqa: E402

WAIT_TIMEOUT_US = 1_000_000

APPLY_CU = r"""
#include <cuda_runtime.h>
#include <stdint.h>
__global__ void apply_kernel(const uint32_t *count, unsigned long long *applied, volatile unsigned long long *stamp)
{
    const uint32_t c = *count;
    if (!c) return;
    *applied += c;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    *stamp = t;
}
extern "C" int apply(const uint32_t *count, unsigned long long *applied, unsigned long long *stamp, void *stream)
{
    apply_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(count, applied, stamp);
    return (int)cudaGetLastError();
}
extern "C" int apply_load(void)
{
    cudaFuncAttributes fa;
    return (int)cudaFuncGetAttributes(&fa, apply_kernel);
}
"""


def load_apply():
    d = tempfile.mkdtemp(prefix="consume_wait_bench_")
    src, so = os.path.join(d, "apply.cu"), os.path.join(d, "apply.so")
    with open(src, "w") as f:
        f.write(APPLY_CU)
    subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared", "-Xcompiler", "-fPIC",
                    "-o", so, src], check=True)
    lib = ctypes.CDLL(so)
    lib.apply.argtypes = [ctypes.c_void_p] * 4
    # loaded before any replica kernel is resident: a lazy load beside them may wait for them
    assert lib.apply_load() == 0
    return lib


def new_stream(device):
    """a stream created with the runtime, not taken from torch's pool: the pool creates dozens of streams at once, and
    those wrap around the hardware queues onto the replicas' own streams, where a pending consume wait would hold up
    the leader (DESIGN.md s2)"""
    try:
        rt = ctypes.CDLL("libcudart.so.12")
    except OSError:
        import nvidia.cuda_runtime as ncr
        rt = ctypes.CDLL(os.path.join(list(ncr.__path__)[0], "lib", "libcudart.so.12"))
    s = ctypes.c_void_p()
    assert rt.cudaSetDevice(device) == 0
    assert rt.cudaStreamCreateWithFlags(ctypes.byref(s), 1) == 0          # cudaStreamNonBlocking
    return torch.cuda.ExternalStream(s.value, device=torch.device("cuda", device))


class Follower:
    """one follower's consumer: its stream, output tensors, applied counter (device) and stamp word (pinned)"""

    def __init__(self, rep, stamp_word):
        dev = torch.device("cuda", rep.device)
        self.rep = rep
        self.stream = new_stream(rep.device)
        with torch.cuda.stream(self.stream):
            self.out = (torch.empty(MAX_N, dtype=torch.int64, device=dev), torch.empty(MAX_N, dtype=torch.uint8, device=dev),
                        torch.empty(MAX_N, dtype=torch.int16, device=dev), torch.empty(MAX_N, dtype=torch.int64, device=dev),
                        torch.empty(MAX_N, dtype=torch.int16, device=dev),
                        torch.empty((MAX_N, PAYLOAD), dtype=torch.uint8, device=dev),
                        torch.zeros(1, dtype=torch.int32, device=dev))
            self.applied = torch.zeros(1, dtype=torch.int64, device=dev)
        self.stamp = stamp_word
        self.cpu = 0.0

    def consume_and_apply(self):
        self.rep.consume_device(MAX_N, PAYLOAD, out=self.out, stream=self.stream)
        APPLY.apply(self.out[6].data_ptr(), self.applied.data_ptr(), self.stamp, self.stream.cuda_stream)


def polled_pump(f, stop):
    """device_pump (consume_bench.py) with the apply kernel after each call"""
    c0 = time.thread_time()
    while True:
        f.consume_and_apply()
        f.stream.synchronize()
        got = int(f.out[6].cpu()[0])
        if not got and stop.is_set():
            break
    f.cpu += time.thread_time() - c0


def waited_pump(f, stop, lock, k_ahead):
    """K iterations of consume_wait(1) -> consume -> apply per batch, two batches in flight, one synchronise per batch"""
    c0 = time.thread_time()
    prev = None
    while True:
        with lock:                    # a stop and its release happen together: no batch is enqueued after the release
            if stop.is_set():
                break
            for _ in range(k_ahead):
                f.rep.consume_wait(1, WAIT_TIMEOUT_US, stream=f.stream)
                f.consume_and_apply()
            ev = torch.cuda.Event(blocking=True)       # the thread sleeps while the batch waits on the device
            ev.record(f.stream)
        if prev is not None:
            prev.synchronize()
        prev = ev
    f.stream.synchronize()
    f.cpu += time.thread_time() - c0


def start(leg, fol, k_ahead):
    stop, lock = threading.Event(), threading.Lock()
    if leg == "polled":
        th = [threading.Thread(target=polled_pump, args=(f, stop)) for f in fol]
    else:
        th = [threading.Thread(target=waited_pump, args=(f, stop, lock, k_ahead)) for f in fol]
    for x in th:
        x.start()
    return stop, lock, th


def finish(leg, fol, stop, lock, th):
    with lock:
        stop.set()
        if leg == "waited":
            for f in fol:
                f.rep.consume_wait_release()
    for x in th:
        x.join(300)
        assert not x.is_alive()


def all_examined(lead, fol, t):
    lead.wait_committed(t, 60_000_000)
    last = lead.stats()["entries_published"]
    while any(f.rep.consume_status().next_idx <= last for f in fol):
        time.sleep(0.0001)
    for f in fol:
        assert f.rep.consume_status().error == 0


def step_round(leg, lead, fol, req, seed, k_ahead):
    for f in fol:
        f.cpu = 0.0
    stop, lock, th = start(leg, fol, k_ahead)
    t0 = time.perf_counter()
    t = lead.submit_synth(N_REQ, E.SEND, 0, req, PAYLOAD, seed) + N_REQ - 1
    all_examined(lead, fol, t)
    finish(leg, fol, stop, lock, th)
    return time.perf_counter() - t0, sum(f.cpu for f in fol)


def latency_round(leg, lead, fol, stamps, req, n, k_ahead):
    stop, lock, th = start(leg, fol, k_ahead)
    out = []
    pl = bytes(PAYLOAD)
    for i in range(n):
        before = stamps.copy()
        t = lead.submit(E.SEND, 1, req + i, pl)
        lead.wait_committed(t, 10_000_000)
        c_ns = lead.last_commit_ns()
        t_end = time.time() + 10
        while np.any(stamps == before):
            assert time.time() < t_end, "a follower did not apply a committed request within 10 s"
            time.sleep(0.00005)       # lets the pump threads have the GIL (the latency itself is on the device clock)
        out.append([int(s) - c_ns for s in stamps])
    all_examined(lead, fol, t)
    finish(leg, fol, stop, lock, th)
    return out


def main():
    global APPLY
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--lat", type=int, default=1000, help="closed-loop requests per round and leg")
    ap.add_argument("--k", type=int, default=8, help="waited leg: iterations per batch")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available() or A.lib().apus_device_count() < 1:
        raise SystemExit("consume_wait_bench.py: no CUDA device; the engine has no CPU fallback")
    APPLY = load_apply()
    for dt in (torch.uint8, torch.int16, torch.int32, torch.int64):
        torch.zeros(16, dtype=dt, device="cuda:0").clone()
    torch.cuda.synchronize()
    lines = [json.dumps({"card": card(), "torch": torch.__version__, "replicas": REPLICAS, "leader_ctas": CTAS,
                         "log_size": A.LOG_SIZE, "requests_per_step": N_REQ, "payload": PAYLOAD, "max_n": MAX_N,
                         "k_ahead": args.k, "wait_timeout_us": WAIT_TIMEOUT_US, "latency_requests": args.lat})]
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
    fol = [Follower(r, stamps_t.data_ptr() + 8 * k) for k, r in enumerate(reps[1:])]
    lead = reps[0]
    arr = (E.C.c_void_p * REPLICAS)(*[r.h for r in reps])
    E._ck(E.lib().apus_replicas_launch(arr, REPLICAS, E.UINT64_MAX), "apus_replicas_launch")
    res = {w: {"step_s": [], "cpu_s": [], "lat_ns": []} for w in ("polled", "waited")}
    try:
        lead.wait_committed(lead.submit(E.CONFIG, 0, 0, E.cid_image(REPLICAS)))
        req = 1
        for s in range(args.warmup + args.steps):
            for w in ("polled", "waited"):                        # alternating
                dt, cpu = step_round(w, lead, fol, req, 0xD0 + s, args.k)
                req += N_REQ
                lat = latency_round(w, lead, fol, stamps, req, args.lat, args.k)
                req += args.lat
                p50 = np.percentile(np.asarray(lat), 50) / 1e3
                print(f"[{w}] round {s}: step {dt * 1e3:.1f} ms, pump cpu {cpu * 1e3:.1f} ms, "
                      f"commit-to-applied p50 {p50:.2f} us", file=sys.stderr, flush=True)
                if s >= args.warmup:
                    res[w]["step_s"].append(dt)
                    res[w]["cpu_s"].append(cpu)
                    res[w]["lat_ns"].extend(lat)
        applied = [int(f.applied.cpu()[0]) for f in fol]
        want = (args.warmup + args.steps) * 2 * (N_REQ + args.lat)
        assert applied == [want] * len(fol), (applied, want)
    finally:
        E._ck(E.lib().apus_replicas_stop(arr, REPLICAS), "apus_replicas_stop")
    for w in ("polled", "waited"):
        r = res[w]
        lat = np.asarray(r["lat_ns"], dtype=np.float64)
        lines.append(json.dumps({
            "leg": w, "rounds": args.steps,
            "step_ms": [round(x * 1e3, 3) for x in r["step_s"]],
            "step_ms_median": float(np.median(r["step_s"])) * 1e3,
            "pump_cpu_ms": [round(x * 1e3, 3) for x in r["cpu_s"]],
            "pump_cpu_ms_median": float(np.median(r["cpu_s"])) * 1e3,
            "commit_to_applied_samples": int(lat.size),
            "commit_to_applied_p50_us": float(np.percentile(lat, 50)) / 1e3,
            "commit_to_applied_p99_us": float(np.percentile(lat, 99)) / 1e3,
            "applied_per_follower": applied[0]}))
        print(lines[-1], flush=True)
    for r in reps:
        r.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


APPLY = None

if __name__ == "__main__":
    main()
