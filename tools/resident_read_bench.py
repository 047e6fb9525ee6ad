"""Resident read fences (apus_reader_attach, include/apus_reader.cuh) against stream fences (apus_read_fence), under the
load of tools/read_fence_bench.py: five replicas on one GPU, a 64 MiB log with device-side pruning, every replica
applying on the device (APUS_F_DEVICE_APPLY | APUS_F_APPLY_ANY_ROLE, stream consume calls that keep up in the
background), and a writer thread that submits 64 B SENDs in batches of 256 every 0.5 ms for the whole run.

  stream     on each follower in turn: read_fence -> consume -> one read, synchronised; the fence kernel alone is timed
             with CUDA events (device clock)
  resident   on each follower in turn: the test reader (tests/devicelogic/resident_reads.cu) runs --fences fences back to
             back in one slot; each is timed from its begin to READY on %globaltimer (device clock), and the fences per
             second are taken from the first begin to the last end
  commit     closed-loop commit latency on the leader (apus_closed_loop, host clock, 2000 requests of 64 B with the
             writer paused), with the test reader fencing in four slots on every follower, and with no reader

The legs alternate round by round.  Prints JSON lines: the card's name and power limit, read in the same run, then one
line per leg; --out appends them to a file.

  python tools/resident_read_bench.py [--rounds 3] [--fences 2000] [--out FILE] [--hang-s 300]
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

import reader as RD  # noqa: E402
from apus_b200 import engine as E  # noqa: E402
from consume_bench import CTAS, REPLICAS, card  # noqa: E402
from consumers import new_stream  # noqa: E402
from read_fence_bench import ANY, LOG, PAYLOAD, Reader, Writer, pct  # noqa: E402


def resident_leg(rep, stream, view, fences):
    """`fences` resident fences back to back in one slot; (begin-to-READY us of each, fences per second)"""
    r = RD.Reader(rep, stream, slots=1, target=fences, timeout_us=1_000_000, deadline_s=60, log_cap=fences).start(view)
    r.wait(90)
    _, fs = r.result()
    assert len(fs) == fences and all(f.outcome == E.WAIT_READY for f in fs), {f.outcome for f in fs}
    lat = [(f.t_end - f.t_begin) / 1e3 for f in fs]
    return lat, fences / ((fs[-1].t_end - fs[0].t_begin) / 1e9)


def commit_leg(w, lead, rid, readers_on):
    """closed-loop commit latencies (us) of 2000 requests, the writer paused; readers_on: {rep: (stream, view)} fence
    in four slots each meanwhile"""
    rs = [RD.Reader(rep, s, slots=4, timeout_us=1_000_000, deadline_s=1.5, log_cap=16).start(v)
          for rep, (s, v) in readers_on.items()]
    with w.mu:
        lat = lead.closed_loop(2000, PAYLOAD, 7, rid)
    for r in rs:
        r.wait(30)
        r.result()
    return [x / 1e3 for x in lat.tolist()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--fences", type=int, default=2000, help="fences per follower, leg and round")
    ap.add_argument("--out")
    ap.add_argument("--hang-s", type=float, default=300, help="dump every thread's stack and exit after this long")
    a = ap.parse_args()
    faulthandler.dump_traceback_later(a.hang_s, exit=True)
    lines = [card()]
    print(json.dumps(lines[0]), file=sys.stderr, flush=True)
    RD.lib()
    flags = E.F_DEVICE_STATS | E.F_AUTOPRUNE | ANY
    reps = [E.Replica(0, i, REPLICAS, 0, 1, LOG, E.RING_DEVICE if i == 0 else E.RING_HOST_MAPPED, 0, 0, flags, CTAS)
            for i in range(REPLICAS)]
    blobs = [r.export() for r in reps]
    for r in reps:
        for j, b in enumerate(blobs):
            if j != r.idx:
                r.connect(j, b)
    lead = reps[0]
    readers = {i: Reader(reps[i], 1) for i in range(REPLICAS)}
    for rd in readers.values():
        rd.warm()
    rstream = {i: new_stream(reps[i].device) for i in range(1, REPLICAS)}
    for i in list(range(1, REPLICAS)) + [0]:                          # followers first, one launch each
        arr = (E.C.c_void_p * 1)(reps[i].h)
        E._ck(E.lib().apus_replicas_launch(arr, 1, (1 << 64) - 1), "apus_replicas_launch")
    views = {}
    w = None
    stop_drain = threading.Event()
    drains = {}
    try:
        lead.wait_committed(lead.submit(2, 0, 0, bytes(16)), 10_000_000)    # APUS_CONFIG
        views = {i: reps[i].reader_attach(rstream[i]) for i in range(1, REPLICAS)}
        w = Writer(lead)
        w.start()

        def drain(i):
            while not stop_drain.is_set():
                with readers[i].busy:
                    readers[i].consume()
                    readers[i].stream.synchronize()
                time.sleep(0.001)
        for i in range(REPLICAS):
            readers[i].busy = threading.Lock()
            drains[i] = threading.Thread(target=drain, args=(i,), daemon=True)
            drains[i].start()
        time.sleep(0.5)
        legs = {k: {"lat": [], "rate": [], "fps": []} for k in ("stream", "resident", "commit_none", "commit_readers")}
        rid = 1 << 40

        def stream_leg():
            fdev, fps = [], []
            for i in range(1, REPLICAS):
                with readers[i].busy:
                    t1 = time.perf_counter()
                    for _ in range(a.fences // 4):
                        fdev.append(readers[i].fenced_read(1)[2])
                    fps.append(a.fences // 4 / (time.perf_counter() - t1))
            return fdev, fps

        def res_leg():
            lat, fps = [], []
            for i in range(1, REPLICAS):
                x, f = resident_leg(reps[i], rstream[i], views[i], a.fences)
                lat += x
                fps.append(f)
            return lat, fps

        for rnd in range(a.rounds + 1):
            print(f"round {rnd}", file=sys.stderr, flush=True)
            order = ["stream", "resident", "commit_none", "commit_readers"]
            if rnd % 2:
                order = order[::-1]
            for leg in order:
                res = {}
                if leg in ("stream", "resident"):
                    th = threading.Thread(target=lambda: res.update(r=(stream_leg if leg == "stream" else res_leg)()))
                    th.start()
                    rate = w.rate(0.3)
                    th.join()
                    lat, fps = res["r"]
                else:
                    rid += 10_000
                    lat = commit_leg(w, lead, rid, {reps[i]: (rstream[i], views[i]) for i in range(1, REPLICAS)}
                                     if leg == "commit_readers" else {})
                    fps, rate = [], None
                if rnd:
                    legs[leg]["lat"] += lat
                    legs[leg]["fps"] += fps
                    if rate is not None:
                        legs[leg]["rate"].append(rate)
        what = {"stream": "fence kernel alone, CUDA events (device clock)",
                "resident": "resident fence begin to READY, %globaltimer (device clock)",
                "commit_none": "closed-loop commit latency, host clock, no reader",
                "commit_readers": "closed-loop commit latency, host clock, four fencing slots on every follower"}
        for leg, d in legs.items():
            ln = {"leg": leg, "what": what[leg], "samples": len(d["lat"]), "us_p50": pct(d["lat"], 50),
                  "us_p99": pct(d["lat"], 99)}
            if d["fps"]:
                ln["fences_per_s_per_follower"] = float(np.median(d["fps"]))
            if d["rate"]:
                ln["writer_commits_per_s"] = float(np.median(d["rate"]))
            lines.append(ln)
    finally:
        stop_drain.set()
        for t in drains.values():
            t.join()
        if w is not None:
            w.stop_.set()
            w.join()
        for i in views:
            reps[i].reader_detach()
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
