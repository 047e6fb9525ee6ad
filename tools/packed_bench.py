"""Packed (values + offsets) against strided ([n, stride] + lens) device batches, on both ends: apus_submit_device_packed
against apus_submit_device on the leader, apus_consume_device_packed against apus_consume_device on every follower.
consume_bench.py's placement: five replicas on GPU 0, 16 leader CTAs, a 64 MiB log, the device submission ring,
device-side pruning; the kernels stay resident while the requests stream in.

Two request shapes, each run by both ways in alternating steps, each way on its own group and its own streams:
  u64    2^18 requests of 64 B per step, in batches of 4096; strided uses stride 64 on both ends
  heavy  2^16 requests per step in batches of 1024, seeded: 98% of 0..256 B, 2% of 1 KiB..64 KiB (65535 B included);
         strided needs stride 65535 on both ends, so its consumers take max_n 4096 (268 MB of rows each)

Each way's group is launched for its own steps only.  A step that makes no progress for --stall-s seconds prints the
leader's and the followers' progress words and exits; a host call that blocks is caught 10 s later by a watchdog that
prints every thread's stack and exits.

Prints JSON lines: per shape and way, committed ops/s (host clock from the first submit to the commit of the step's last
ticket), pack ms per batch (CUDA events around each submit call on the submitting stream, which waits for the packing),
consume entries/s and GB/s per follower (CUDA events around each consume call; bytes = 64 B header + cmd read, and the
row written), the tensor bytes allocated on each side, and the payload-ring bytes reserved per request from the
reservation formulas; the card's name and power limit read in the same run.

  python tools/packed_bench.py [--steps 3] [--warmup 1] [--shapes u64,heavy] [--out FILE]
"""
import argparse
import faulthandler
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
# A resident replica launch holds one of the process's hardware work queues for as long as it runs, and streams share
# those queues round robin (8 by default): consume or packing work whose stream lands on the launch's queue waits for
# the launch to end, which here it never does -- the followers' consumers stall and the leader cannot prune.  This tool
# creates about thirty streams (every replica's launch, copy and consume streams, torch's pool), so it asks for the
# maximum of 32 queues, creates torch's streams first and keeps only the group whose step runs resident.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import numpy as np  # noqa: E402
import torch  # noqa: E402

import apus_b200 as A  # noqa: E402
from apus_b200 import engine as E  # noqa: E402

REPLICAS = 5
# the largest payload ring a descriptor can address (24-bit offsets in 16 B units): one strided heavy batch of 1024
# requests reserves 1024 x 65552 B, so the ring holds one such batch at a time
RING_SLOTS, RING_BYTES = 1 << 21, 1 << 27
SHAPES = {"u64": dict(n=1 << 18, batch=4096, stride=64, max_n=1 << 16),
          "heavy": dict(n=1 << 16, batch=1024, stride=65535, max_n=4096)}
PACKED_MAX_N, PACKED_CAP = 1 << 16, 64 << 20
STALL_S = 60
CTAS = 16


T0 = time.perf_counter()


def note(msg):
    print(f"[{time.perf_counter() - T0:8.2f} s] {msg}", file=sys.stderr, flush=True)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def round16(x):
    return (x + 15) & ~15


def strided_reserve(n, stride):
    per = 2 + min(stride, 65535)
    return n * (round16(per) if per > 80 else 0)


def packed_reserve(n, values_bytes):
    return min(n * round16(2 + 65535), round16(values_bytes + 17 * n))


def lengths(shape, seed):
    sp = SHAPES[shape]
    if shape == "u64":
        return np.full(sp["n"], 64, dtype=np.int64)
    rng = np.random.default_rng(seed)
    ln = rng.integers(0, 257, sp["n"])
    tail = rng.random(sp["n"]) < 0.02
    ln[tail] = rng.integers(1024, 65536, int(tail.sum()))
    ln[np.flatnonzero(tail)[::4]] = 65535
    return ln.astype(np.int64)


class Batches:
    """one step's requests on the GPU, cut into batches, in both layouts"""

    def __init__(self, shape, seed):
        sp = SHAPES[shape]
        dev = torch.device("cuda", 0)
        self.lens = lengths(shape, seed)
        n, b = sp["n"], sp["batch"]
        g = torch.Generator(device=dev)
        g.manual_seed(seed)
        offs = np.concatenate([[0], np.cumsum(self.lens)])
        self.values = torch.randint(0, 256, (int(offs[-1]),), dtype=torch.uint8, device=dev, generator=g)
        self.types = torch.full((b,), E.SEND, dtype=torch.uint8, device=dev)
        self.conns = torch.zeros(b, dtype=torch.int16, device=dev)
        self.req_ids = torch.arange(b, dtype=torch.int64, device=dev)
        self.packed, self.strided = [], []
        stride = sp["stride"]
        for a in range(0, n, b):
            o = offs[a:a + b + 1]
            self.packed.append((torch.from_numpy(o - o[0]).to(dev), self.values[int(o[0]):int(o[-1])]))
            ln = torch.from_numpy(self.lens[a:a + b]).to(dev)
            rows = torch.zeros((b, stride), dtype=torch.uint8, device=dev)
            rows[torch.arange(stride, device=dev)[None, :] < ln[:, None]] = self.values[int(o[0]):int(o[-1])]
            self.strided.append((ln.to(torch.int32).to(torch.int16), rows))
        torch.cuda.synchronize()
        self.stride = stride
        self.packed_bytes = sum(o.numel() * 8 + v.numel() for o, v in self.packed) + b * 11
        self.strided_bytes = sum(l.numel() * 2 + r.numel() for l, r in self.strided) + b * 11
        self.reserve = {"packed": sum(packed_reserve(o.numel() - 1, v.numel()) for o, v in self.packed) / n,
                        "strided": strided_reserve(n, stride) / n}


def make_group():
    reps = [E.Replica(0, i, REPLICAS, 0, 1, A.LOG_SIZE, E.RING_DEVICE, RING_SLOTS, RING_BYTES,
                      E.F_DEVICE_STATS | (E.F_AUTOPRUNE if i == 0 else E.F_DEVICE_APPLY), CTAS) for i in range(REPLICAS)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    return reps


class Follower:
    """one follower's consumer thread state: reused output tensors, its own stream"""

    def __init__(self, r, way, shape, st):
        sp = SHAPES[shape]
        self.r, self.way = r, way
        self.st = st
        if way == "packed":
            self.max_n, self.cap = PACKED_MAX_N, PACKED_CAP
            self.out = r.consume_device_packed(self.max_n, self.cap, stream=self.st)
            self.bytes = self.max_n * 19 + (self.max_n + 1) * 8 + self.cap
        else:
            self.max_n, self.stride = sp["max_n"], sp["stride"]
            self.out = r.consume_device(self.max_n, self.stride, stream=self.st)
            self.bytes = self.max_n * (21 + self.stride)
        self.st.synchronize()

    def run(self, lens, log):
        # no torch kernel here: a module loaded lazily while the replica kernels are resident may wait for them
        got, cum = 0, np.concatenate([[0], np.cumsum(lens)])
        while got < len(lens):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(self.st)
            if self.way == "packed":
                self.r.consume_device_packed(self.max_n, self.cap, out=self.out, stream=self.st)
            else:
                self.r.consume_device(self.max_n, self.stride, out=self.out, stream=self.st)
            e1.record(self.st)
            self.st.synchronize()
            k = int(self.out[6].cpu()[0])
            assert self.r.consume_status().error == 0
            if k:
                if self.way == "packed":
                    cmd = int(self.out[4][k].cpu())
                    row = k * 19 + (k + 1) * 8 + cmd
                else:
                    cmd = int(cum[got + k] - cum[got])              # rows arrive in submission order
                    row = k * (21 + self.stride)
                log.append((k, 64 * k + cmd + row, e0.elapsed_time(e1)))
                got += k


def stall_check(deadline, way, what, lead, fols, logs):
    """no progress within STALL_S: print the leader's and the followers' progress words and stop"""
    if time.time() <= deadline:
        return
    note(f"{way}: {what} within {STALL_S} s")
    report = {"way": way, "what": what, "leader": lead.offsets(), "leader_stats": lead.stats(),
              "followers": [{"offsets": f.r.offsets(), "consume": f.r.consume_status()._asdict(),
                             "rows": sum(k for k, _, _ in logs[j])} for j, f in enumerate(fols)]}
    note("stalled: reading the progress words")
    print(json.dumps({"stall": report}), flush=True)
    print(f"packed_bench.py: {way}: {what} within {STALL_S} s", file=sys.stderr, flush=True)
    os._exit(1)                     # the consumer threads may be inside CUDA calls that do not return


def run_step(way, reps, fols, bt, sub):
    lead = reps[0]
    arr = (E.C.c_void_p * REPLICAS)(*[r.h for r in reps])
    E._ck(E.lib().apus_replicas_launch(arr, REPLICAS, E.UINT64_MAX), "apus_replicas_launch")
    n = len(bt.lens)
    logs = [[] for _ in fols]
    th = [threading.Thread(target=f.run, args=(bt.lens, logs[k]), daemon=True) for k, f in enumerate(fols)]
    for x in th:
        x.start()
    pack = []
    t0 = time.perf_counter()
    last = 0
    # a host call that blocks never reaches stall_check: after a further 10 s, print every thread's stack and exit
    faulthandler.dump_traceback_later(STALL_S + 10, exit=True)
    for q in range(len(bt.packed)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        rid = bt.req_ids
        deadline = time.time() + STALL_S
        while True:
            stall_check(deadline, way, f"batch {q} not accepted", lead, fols, logs)
            try:
                e0.record(sub)
                if way == "packed":
                    o, v = bt.packed[q]
                    last = lead.submit_device_packed(bt.types, bt.conns, rid, o, v, stream=sub) + bt.types.numel() - 1
                else:
                    ln, rows = bt.strided[q]
                    last = lead.submit_device(bt.types, bt.conns, rid, ln, rows, stream=sub) + bt.types.numel() - 1
                e1.record(sub)
                break
            except BlockingIOError:
                time.sleep(0.0002)
        pack.append((e0, e1))
        faulthandler.dump_traceback_later(STALL_S + 10, exit=True)
        if q % 16 == 15:
            note(f"{way}: {q + 1} batches accepted, {lead.committed()} tickets committed")
    deadline = time.time() + STALL_S
    while lead.committed() < last:
        stall_check(deadline, way, f"ticket {last} not committed", lead, fols, logs)
        time.sleep(0.0005)
    dt = time.perf_counter() - t0
    for x in th:
        x.join(300)
    sub.synchronize()
    faulthandler.cancel_dump_traceback_later()
    E._ck(E.lib().apus_replicas_stop(arr, REPLICAS), "apus_replicas_stop")
    return n / dt, [a.elapsed_time(b) for a, b in pack], logs


def main():
    global CTAS, STALL_S
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--ways", default="packed,strided", help="the order the two ways alternate in")
    ap.add_argument("--leader-ctas", type=int, default=CTAS)
    ap.add_argument("--stall-s", type=float, default=STALL_S)
    args = ap.parse_args()
    CTAS, STALL_S = args.leader_ctas, args.stall_s
    if not torch.cuda.is_available() or A.lib().apus_device_count() < 1:
        raise SystemExit("packed_bench.py: no CUDA device; the engine has no CPU fallback")
    lines = [json.dumps({"card": card(), "torch": torch.__version__, "replicas": REPLICAS, "leader_ctas": CTAS,
                         "log_size": A.LOG_SIZE, "ring_slots": RING_SLOTS, "ring_bytes": RING_BYTES,
                         "shapes": SHAPES, "packed_consume": {"max_n": PACKED_MAX_N, "values_cap": PACKED_CAP}})]
    print(lines[0], flush=True)
    ways = args.ways.split(",")
    for shape in args.shapes.split(","):
        streams = {w: [torch.cuda.Stream(device=0) for _ in range(REPLICAS)] for w in ways}   # before the engine's
        note(f"{shape}: building the batches")
        bt = Batches(shape, 0xBEE + len(shape))
        note(f"{shape}: creating the groups")
        groups = {w: make_group() for w in ways}
        fols = {w: [Follower(r, w, shape, st) for r, st in zip(reps[1:], streams[w])] for w, reps in groups.items()}
        torch.cuda.synchronize()
        note(f"{shape}: running")
        for w, reps in groups.items():
            reps[0].submit(E.CONFIG, 0, 0, E.cid_image(REPLICAS))
        res = {w: {"ops": [], "pack_ms": [], "calls": [[] for _ in range(REPLICAS - 1)]} for w in groups}
        for s in range(args.warmup + args.steps):
            for w in ways:                                                  # alternating
                ops, pk, logs = run_step(w, groups[w], fols[w], bt, streams[w][0])
                print(f"[{shape} {w}] step {s}: {ops:.0f} committed ops/s, pack {np.median(pk):.3f} ms per batch",
                      file=sys.stderr, flush=True)
                if s >= args.warmup:
                    res[w]["ops"].append(ops)
                    res[w]["pack_ms"] += pk
                    for k in range(REPLICAS - 1):
                        res[w]["calls"][k] += logs[k]
        for w in ways:
            r = res[w]
            per = []
            for k in range(REPLICAS - 1):
                n = sum(c for c, _, _ in r["calls"][k])
                by = sum(b for _, b, _ in r["calls"][k])
                ms = sum(m for _, _, m in r["calls"][k])
                per.append({"follower": k + 1, "entries": n, "calls": len(r["calls"][k]), "consume_ms": ms,
                            "entries_per_s": n / (ms / 1e3) if ms else None,
                            "gb_per_s": by / (ms / 1e3) / 1e9 if ms else None})
            out = {"shape": shape, "way": w, "steps": args.steps, "requests_per_step": len(bt.lens),
                   "mean_cmd_bytes": float(bt.lens.mean()), "max_cmd_bytes": int(bt.lens.max()),
                   "committed_ops_per_s": r["ops"], "committed_ops_per_s_median": float(np.median(r["ops"])),
                   "pack_ms_per_batch_median": float(np.median(r["pack_ms"])),
                   "pack_ms_per_batch_mean": float(np.mean(r["pack_ms"])),
                   "submit_tensor_bytes": bt.packed_bytes if w == "packed" else bt.strided_bytes,
                   "consume_tensor_bytes_per_follower": fols[w][0].bytes,
                   "payload_ring_bytes_reserved_per_request": bt.reserve[w], "per_follower": per}
            lines.append(json.dumps(out))
            print(lines[-1], flush=True)
        for reps in groups.values():
            for x in reps:
                x.close()
        del bt
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
