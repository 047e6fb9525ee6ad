"""Replace a lost follower of a group that applies in GPU memory, and time it: five replicas on GPU 0 (bench.py's
placement), 16 leader CTAs, a 64 MiB log with device-side pruning, every replica consuming on the device
(APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE) into a device state of --state-mib MiB.  A host thread keeps 64 B requests
coming (batches of 4096 through apus_submit_uniform) the whole time.

  1. steady state with five replicas: commits per second over --window seconds ("before")
  2. follower 4 is lost: every replica stops, the others disconnect it, its region is freed, the rest run on
  3. the leader's consumer marks its position and copies its state right behind the mark, on its stream, while the
     group runs (apus_consume_mark + a device-to-device copy; CUDA events around both)
  4. every replica stops; a fresh replica takes slot 4, is seeded at the mark and adjusted (the leader's kernel stands
     stopped from the stop to the relaunch: host clock, with the bytes the adjustment resent)
  5. relaunch: the time until the replacement's consumer has reached the leader's commit as it stood at the relaunch
  6. steady state with the replacement ("after"); at the end every replica has applied the same number of rows

Prints JSON lines, the first with the card's name and power limit read in the same run, and appends them to --out.

  python tools/rejoin_bench.py [--state-mib 64] [--window 2] [--out profiles/rejoin_bench.jsonl]
"""
import argparse
import ctypes
import json
import os
import sys
import threading
import time

# five replicas' launches and side streams plus a consumer stream each (DESIGN.md s2)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import apus_b200 as A  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consume_bench import card  # noqa: E402

REPLICAS, CTAS, PAYLOAD, BATCH, MAX_N = 5, 16, 64, 4096, 4096
ANY = E.F_DEVICE_APPLY | E.F_APPLY_ANY_ROLE
LOST = REPLICAS - 1


def runtime_stream():
    """a stream of the runtime's own, off torch's pool (whose streams share hardware queues with the launches)"""
    try:
        rt = ctypes.CDLL("libcudart.so.12")
    except OSError:
        import nvidia.cuda_runtime as ncr
        rt = ctypes.CDLL(os.path.join(list(ncr.__path__)[0], "lib", "libcudart.so.12"))
    s = ctypes.c_void_p()
    assert rt.cudaSetDevice(0) == 0 and rt.cudaStreamCreateWithFlags(ctypes.byref(s), 1) == 0
    return torch.cuda.ExternalStream(s.value, device=torch.device("cuda", 0))


class Applier:
    """one replica's consumer thread: consume_device (stride 64) and a count of the rows into the state's first word"""

    def __init__(self, rep, state_words, state=None):
        self.rep, self.stream = rep, runtime_stream()
        with torch.cuda.stream(self.stream):
            dev = torch.device("cuda", 0)
            self.out = (torch.empty(MAX_N, dtype=torch.int64, device=dev), torch.empty(MAX_N, dtype=torch.uint8, device=dev),
                        torch.empty(MAX_N, dtype=torch.int16, device=dev), torch.empty(MAX_N, dtype=torch.int64, device=dev),
                        torch.empty(MAX_N, dtype=torch.int16, device=dev),
                        torch.empty((MAX_N, PAYLOAD), dtype=torch.uint8, device=dev),
                        torch.empty(1, dtype=torch.int32, device=dev))
            self.state = torch.zeros(state_words, dtype=torch.int64, device=dev) if state is None else state.clone()
            self.mark = torch.zeros(2, dtype=torch.int64, device=dev)
        self.stream.synchronize()
        self.halt, self.want, self.snap, self.errs, self.th = threading.Event(), threading.Event(), None, [], None

    def step(self):
        self.rep.consume_device(MAX_N, PAYLOAD, out=self.out, stream=self.stream)
        with torch.cuda.stream(self.stream):
            self.state[:1].add_(self.out[6].to(torch.int64))
        if self.want.is_set():
            self.want.clear()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(self.stream)
            self.rep.consume_mark(out=self.mark, stream=self.stream)
            with torch.cuda.stream(self.stream):
                copy = self.state.clone()
            e1.record(self.stream)
            self.stream.synchronize()
            m = self.mark.cpu().numpy().astype(np.uint64)
            self.snap = (int(m[0]), int(m[1]), copy, e0.elapsed_time(e1))
        self.stream.synchronize()

    def start(self):
        def run():
            try:
                while not self.halt.is_set():
                    self.step()
            except Exception as e:        # noqa: BLE001 - reported by stop()
                self.errs.append(e)
        self.halt.clear()
        self.th = threading.Thread(target=run)
        self.th.start()

    def stop(self):
        self.halt.set()
        if self.th:
            self.th.join(120)
        self.th = None
        if self.errs:
            raise self.errs[0]


class Traffic:
    """a host thread submitting batches of 64 B SENDs; pause() holds it"""

    def __init__(self, lead):
        self.lead, self.rid, self.halt, self.go = lead, 1, threading.Event(), threading.Event()
        self.payload = np.frombuffer(bytes((k * 37 + 11) & 0xFF for k in range(PAYLOAD)) * BATCH, dtype=np.uint8)
        self.last, self.errs = 0, []
        self.go.set()
        self.th = threading.Thread(target=self.run)
        self.th.start()

    def run(self):
        try:
            while not self.halt.is_set():
                if not self.go.wait(0.01):
                    continue
                try:
                    self.last = self.lead.submit_uniform(BATCH, E.SEND, 1, self.rid, PAYLOAD, self.payload) + BATCH - 1
                    self.rid += BATCH
                except BlockingIOError:
                    time.sleep(0.0002)
        except Exception as e:            # noqa: BLE001 - reported by close()
            self.errs.append(e)

    def close(self):
        self.halt.set()
        self.th.join(60)
        if self.errs:
            raise self.errs[0]


def rate(lead, window):
    c0, t0 = lead.committed(), time.perf_counter()
    time.sleep(window)
    return (lead.committed() - c0) / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--state-mib", type=int, default=64)
    ap.add_argument("--window", type=float, default=2.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "rejoin_bench.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available() or A.lib().apus_device_count() < 1:
        raise SystemExit("rejoin_bench.py: no CUDA device; the engine has no CPU fallback")
    lib = A.lib()
    # every torch kernel the appliers use, loaded before the replica kernels are resident
    for dt in (torch.uint8, torch.int16, torch.int32, torch.int64):
        torch.zeros(16, dtype=dt, device="cuda:0").clone().add_(1)
    w = torch.zeros(16, dtype=torch.int64, device="cuda:0")
    w[:1].add_(torch.ones(1, dtype=torch.int32, device="cuda:0").to(torch.int64))
    torch.cuda.synchronize()
    words = (args.state_mib << 20) // 8
    head = {"card": card(), "torch": torch.__version__, "replicas": REPLICAS, "leader_ctas": CTAS,
            "log_size": A.LOG_SIZE, "payload": PAYLOAD, "batch": BATCH, "state_mib": args.state_mib,
            "window_s": args.window}
    lines = [head]
    print(json.dumps(head), flush=True)

    def replica(i):
        return E.Replica(0, i, REPLICAS, 0, 1, A.LOG_SIZE, E.RING_HOST_MAPPED, 1 << 16, 16 << 20,
                         E.F_DEVICE_STATS | ANY | (E.F_AUTOPRUNE if i == 0 else 0), CTAS)

    def launch(rs):
        for r in sorted(rs, key=lambda r: r.is_leader):
            E._ck(lib.apus_replicas_launch((ctypes.c_void_p * 1)(r.h), 1, E.UINT64_MAX), "apus_replicas_launch")

    def stop(rs):
        E._ck(lib.apus_replicas_stop((ctypes.c_void_p * len(rs))(*[r.h for r in rs]), len(rs)), "apus_replicas_stop")

    reps = [replica(i) for i in range(REPLICAS)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    apps = {i: Applier(r, words) for i, r in enumerate(reps)}
    lead = reps[0]
    live = list(reps)
    traffic = None
    try:
        launch(live)
        lead.wait_committed(lead.submit(E.CONFIG, 0, 0, E.cid_image(REPLICAS)))
        for a in apps.values():
            a.start()
        traffic = Traffic(lead)
        rate(lead, args.window / 2)                               # warm-up
        before = rate(lead, args.window)
        # follower LOST is gone for good
        traffic.go.clear()
        apps.pop(LOST).stop()
        stop(live)
        live = reps[:LOST]
        for r in live:
            E._ck(lib.apus_replica_disconnect(r.h, LOST), "apus_replica_disconnect")
        reps[LOST].close()
        launch(live)
        traffic.go.set()
        rate(lead, args.window / 2)
        # mark and copy the leader's state while the group runs
        apps[0].want.set()
        while apps[0].snap is None:
            time.sleep(0.001)
            if apps[0].errs:
                raise apps[0].errs[0]
        cur, nidx, snap, copy_ms = apps[0].snap
        # the replacement: stop, seed, adjust, relaunch
        traffic.go.clear()
        t0 = time.perf_counter()
        stop(live)
        t_stopped = time.perf_counter()
        r = replica(LOST)
        for p in live:
            r.connect(p.idx, p.export())
            p.connect(LOST, r.export())
        r.consume_seed(cur, nidx)
        got = ctypes.c_uint64()
        t_adj = time.perf_counter()
        rc = lib.apus_ctl_adjust_follower(lead.h, LOST, (1 << 9) | (1 << 8), ctypes.byref(got))
        adj_s = time.perf_counter() - t_adj
        E._ck(rc, "apus_ctl_adjust_follower")
        E._ck(lib.apus_replica_set_role(r.h, 0, 1), "apus_replica_set_role")
        target = lead.stats()["entries_published"] + 1               # the leader's commit as it stands (stopped)
        reps[LOST] = r
        live = list(reps)
        apps[LOST] = Applier(r, words, snap)
        launch(live)
        t_launched = time.perf_counter()
        stopped_s = t_launched - t0
        apps[LOST].start()
        traffic.go.set()
        while r.consume_status().next_idx < target:
            time.sleep(0.0002)
            assert time.perf_counter() - t_launched < 120, (r.consume_status(), target)
        catch_up_s = time.perf_counter() - t_launched
        rate(lead, args.window / 2)
        after = rate(lead, args.window)
        traffic.go.clear()
        time.sleep(0.05)
        lead.wait_committed(traffic.last, 60_000_000)
        # every replica applies the same rows: the counts agree once every consumer has caught up
        for a in apps.values():
            a.stop()
        commit = lead.offsets()["commit"]
        for a in apps.values():
            while a.rep.consume_status().cursor != commit or a.rep.offsets()["commit"] != commit:
                a.step()
        counts = {i: int(a.state[0].cpu()) for i, a in apps.items()}
        assert len(set(counts.values())) == 1, counts
        res = {"leg": "rejoin", "commits_per_s_before": before, "commits_per_s_after": after,
               "mark_and_copy_ms": copy_ms, "state_bytes": words * 8, "leader_stopped_ms": stopped_s * 1e3,
               "stop_ms": (t_stopped - t0) * 1e3, "adjust_ms": adj_s * 1e3, "bytes_resent": int(got.value),
               "seed": [cur, nidx], "catch_up_ms": catch_up_s * 1e3, "rows_applied": counts[0]}
        lines.append(res)
        print(json.dumps(res), flush=True)
    finally:
        if traffic:
            traffic.close()
        for a in apps.values():
            a.halt.set()
        for a in apps.values():
            if a.th:
                a.th.join(60)
        try:
            stop(live)
        finally:
            for x in live:
                x.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for x in lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
