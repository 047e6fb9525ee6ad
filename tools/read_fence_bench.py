"""Reads through the log against read fences (apus_read_fence), on one GPU: five replicas, 16 leader CTAs, a 64 MiB log
with device-side pruning, every replica applying on the device (APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE), and a
writer thread that submits 64 B SENDs at a steady rate (batches of 256 every 0.5 ms) for the whole run.

  log    what the reference does for a GET: submit a 64 B CSM read request on the leader, then consume on follower 1
         until the row carrying it has been applied (a consume_device loop on its own stream)
  fence  on each follower in turn: read_fence -> consume_device (everything committed up to F) -> a read kernel of
         --batch reads from the state, enqueued in that order on the follower's stream and synchronised once
  fence1 the same with one read behind each fence: per read, like for like with the log leg

Per leg: read latency p50 / p99 on the host clock, and on the device clock (CUDA events around the fence -> consume ->
read sequence, and around the fence kernel alone; not measured for the log leg, whose path starts on the host), reads
per second per replica, and the
writer's commit rate with and without the read load.  The legs alternate round by round.  Prints JSON lines: the card's
name and power limit, read in the same run, then one line per leg and the idle line; --out appends them to a file.

  python tools/read_fence_bench.py [--rounds 3] [--reads 1000] [--batch 64] [--out FILE] [--hang-s 300]
"""
import argparse
import faulthandler
import json
import os
import sys
import threading
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from apus_b200 import engine as E  # noqa: E402
from consume_bench import CTAS, REPLICAS, card  # noqa: E402
from consumers import new_stream  # noqa: E402

LOG = 64 << 20
PAYLOAD = 64
STRIDE = 128
MAX_N = 1 << 15
ANY = E.F_DEVICE_APPLY | E.F_APPLY_ANY_ROLE


def pct(xs, q):
    return float(np.percentile(np.asarray(xs, dtype=np.float64), q)) if xs else None


class Writer(threading.Thread):
    """64 B SENDs in batches of 256 every 0.5 ms on the leader, counting what commits"""

    def __init__(self, lead):
        super().__init__(daemon=True)
        self.lead, self.stop_ = lead, threading.Event()
        self.rid = 1
        self.mu = threading.Lock()       # submissions to one leader come from one thread at a time

    def run(self):
        pl = np.zeros(256 * PAYLOAD, dtype=np.uint8)
        while not self.stop_.is_set():
            try:
                with self.mu:
                    self.lead.submit_uniform(256, 5, 1, self.rid, PAYLOAD, pl)      # APUS_SEND
                self.rid += 256
            except BlockingIOError:
                pass
            time.sleep(0.0005)

    def rate(self, secs):
        c0, t0 = self.lead.committed(), time.perf_counter()
        time.sleep(secs)
        return (self.lead.committed() - c0) / (time.perf_counter() - t0)


class Reader:
    """one replica's consumer on its own stream, with a device state: the largest idx applied (the fold) and a table
    the read kernel gathers from"""

    def __init__(self, rep, batch):
        self.rep, self.batch = rep, batch
        self.stream = new_stream(rep.device)
        dev = torch.device("cuda", rep.device)
        with torch.cuda.stream(self.stream):
            self.out = (torch.zeros(MAX_N, dtype=torch.int64, device=dev), torch.empty(MAX_N, dtype=torch.uint8, device=dev),
                        torch.empty(MAX_N, dtype=torch.int16, device=dev), torch.empty(MAX_N, dtype=torch.int64, device=dev),
                        torch.empty(MAX_N, dtype=torch.int16, device=dev),
                        torch.empty((MAX_N, STRIDE), dtype=torch.uint8, device=dev),
                        torch.zeros(1, dtype=torch.int32, device=dev))
            self.applied = torch.zeros(1, dtype=torch.int64, device=dev)
            self.table = torch.arange(1 << 16, dtype=torch.int64, device=dev)
            # one key and answer tensor per read-batch size, each of its own allocation
            self.keys = {b: torch.randint(0, 1 << 16, (b,), dtype=torch.int64, device=dev) for b in (batch, 1)}
            self.answer = {b: torch.empty(b, dtype=torch.int64, device=dev) for b in (batch, 1)}
            self.index = torch.zeros(1, dtype=torch.int64, device=dev)
            self.outcome = torch.zeros(1, dtype=torch.int32, device=dev)
            # every torch kernel used below runs once before the replica kernels are resident: a kernel loaded lazily
            # while they run waits for them to end
            torch.maximum(self.applied, self.out[0].amax(0, keepdim=True), out=self.applied)
            for b in self.keys:
                torch.index_select(self.table, 0, self.keys[b], out=self.answer[b])
            self.applied.zero_()
        self.stream.synchronize()
        self.ev = tuple(torch.cuda.Event(enable_timing=True) for _ in range(3))

    def consume(self):
        """consume into the state: the largest idx applied"""
        self.rep.consume_device(MAX_N, STRIDE, out=self.out, stream=self.stream)
        with torch.cuda.stream(self.stream):
            torch.maximum(self.applied, self.out[0].amax(0, keepdim=True), out=self.applied)
            self.out[0].zero_()

    def warm(self):
        """the whole fenced read of either size once, before any replica kernel is resident (nothing is committed, so
        the fence times out): every torch kernel it launches is loaded by then -- a kernel loaded lazily while the
        replica kernels run waits for them to end"""
        for b in self.keys:
            self.fenced_read(b, timeout_us=100, check=False)

    def fenced_read(self, batch, timeout_us=1_000_000, check=True):
        """fence -> consume -> read kernel of `batch` reads; returns (host us, device us, device us of the fence
        alone), asserting READY and applied >= F"""
        t0 = time.perf_counter()
        self.ev[0].record(self.stream)
        self.rep.read_fence(timeout_us, index=self.index, outcome=self.outcome, stream=self.stream)
        self.ev[2].record(self.stream)
        self.consume()
        with torch.cuda.stream(self.stream):
            torch.index_select(self.table, 0, self.keys[batch], out=self.answer[batch])
        self.ev[1].record(self.stream)
        self.stream.synchronize()
        host = (time.perf_counter() - t0) * 1e6
        o, f, a = int(self.outcome.item()), int(self.index.item()), int(self.applied.item())
        assert not check or (o == E.WAIT_READY and (a >= f or f <= 1)), (self.rep.idx, o, f, a)
        return host, self.ev[0].elapsed_time(self.ev[1]) * 1e3, self.ev[0].elapsed_time(self.ev[2]) * 1e3


def log_read(w, rd, rid):
    """a CSM read request through the log, until follower 1's consumer has applied its row; host us"""
    t0 = time.perf_counter()
    with w.mu:
        w.lead.submit(1, 0x7777, rid, b"r" * PAYLOAD)   # APUS_CSM
    while True:
        rd.rep.consume_device(MAX_N, STRIDE, out=rd.out, stream=rd.stream)
        rd.stream.synchronize()
        k = int(rd.out[6].item())
        if k and rid in rd.out[3][:k].cpu().numpy():
            return (time.perf_counter() - t0) * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reads", type=int, default=1000, help="reads per leg and round (fence: per follower, in batches)")
    ap.add_argument("--batch", type=int, default=64, help="reads behind each fence")
    ap.add_argument("--out")
    ap.add_argument("--hang-s", type=float, default=300, help="dump every thread's stack and exit after this long")
    a = ap.parse_args()
    faulthandler.dump_traceback_later(a.hang_s, exit=True)
    lines = [card()]
    print(json.dumps(lines[0]), file=sys.stderr, flush=True)
    flags = E.F_DEVICE_STATS | E.F_AUTOPRUNE | ANY
    reps = [E.Replica(0, i, REPLICAS, 0, 1, LOG, E.RING_DEVICE if i == 0 else E.RING_HOST_MAPPED, 0, 0, flags, CTAS)
            for i in range(REPLICAS)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    lead = reps[0]
    readers = {i: Reader(reps[i], a.batch) for i in range(REPLICAS)}
    for rd in readers.values():
        rd.warm()
    drains = {}
    for i in list(range(1, REPLICAS)) + [0]:                          # followers first, one launch each
        arr = (E.C.c_void_p * 1)(reps[i].h)
        E._ck(E.lib().apus_replicas_launch(arr, 1, (1 << 64) - 1), "apus_replicas_launch")
    w = None
    try:
        lead.wait_committed(lead.submit(2, 0, 0, bytes(16)), 10_000_000)    # APUS_CONFIG
        w = Writer(lead)
        w.start()
        # every consumer keeps up in the background while the writer runs, so that the pruning rule moves on
        stop_drain = threading.Event()

        def drain(i):
            while not stop_drain.is_set():
                if not readers[i].busy.locked():
                    with readers[i].busy:
                        readers[i].consume()
                        readers[i].stream.synchronize()
                time.sleep(0.001)
        for i in range(REPLICAS):
            readers[i].busy = threading.Lock()
            drains[i] = threading.Thread(target=drain, args=(i,), daemon=True)
            drains[i].start()
        time.sleep(0.5)
        idle = []
        batches = {"log": 1, "fence": a.batch, "fence1": 1}
        legs = {name: {"host": [], "dev": [], "fdev": [], "rate": [], "rps": []} for name in batches}
        rid = 1 << 40
        for rnd in range(a.rounds + 1):
            print(f"round {rnd}", file=sys.stderr, flush=True)
            idle.append(w.rate(0.5))
            # log leg
            res = {}

            def log_leg():
                nonlocal rid
                lat = []
                with readers[1].busy:
                    for _ in range(a.reads):
                        rid += 1
                        lat.append(log_read(w, readers[1], rid))
                res["lat"] = lat
            th = threading.Thread(target=log_leg)
            t0 = time.perf_counter()
            th.start()
            rate = w.rate(0.3)
            th.join()
            el = time.perf_counter() - t0
            if rnd:
                legs["log"]["host"] += res["lat"]
                legs["log"]["rate"].append(rate)
                legs["log"]["rps"].append(a.reads / el)
            # fence legs (a batch of reads behind each fence, then one read per fence): each follower in turn
            for name in ("fence", "fence1"):
                b = batches[name]
                res = {}

                def fence_leg():
                    host, dev, fdev, rps = [], [], [], []
                    for i in range(1, REPLICAS):
                        with readers[i].busy:
                            t1 = time.perf_counter()
                            nf = max(1, a.reads // b)
                            for _ in range(nf):
                                h, d, f = readers[i].fenced_read(b)
                                host.append(h)
                                dev.append(d)
                                fdev.append(f)
                            rps.append(nf * b / (time.perf_counter() - t1))
                    res.update(host=host, dev=dev, fdev=fdev, rps=rps)
                th = threading.Thread(target=fence_leg)
                th.start()
                rate = w.rate(0.3)
                th.join()
                if rnd:
                    for k in ("host", "dev", "fdev", "rps"):
                        legs[name][k] += res[k]
                    legs[name]["rate"].append(rate)
        stop_drain.set()
        for i in range(REPLICAS):
            drains[i].join()
        for name, d in legs.items():
            lines.append({"leg": name, "reads": len(d["host"]) * batches[name],
                          "read_host_us_p50": pct(d["host"], 50), "read_host_us_p99": pct(d["host"], 99),
                          "read_dev_us_p50": pct(d["dev"], 50), "read_dev_us_p99": pct(d["dev"], 99),
                          "fence_kernel_dev_us_p50": pct(d["fdev"], 50), "fence_kernel_dev_us_p99": pct(d["fdev"], 99),
                          "reads_per_s_per_replica_min": min(d["rps"]), "reads_per_s_per_replica_max": max(d["rps"]),
                          "commit_rate_with_reads": [round(x) for x in d["rate"]],
                          "batch": batches[name]})
        lines.append({"leg": "no_reads", "commit_rate": [round(x) for x in idle[1:]]})
    finally:
        if w is not None:
            w.stop_.set()
            w.join()
        arr = (E.C.c_void_p * REPLICAS)(*[r.h for r in reps])
        E.lib().apus_replicas_stop(arr, REPLICAS)
        for r in reps:
            r.close()
    for ln in lines:
        print(json.dumps(ln), flush=True)
    if a.out:
        with open(a.out, "a") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
