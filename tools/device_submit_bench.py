"""Three ways of feeding the leader's HBM submission ring, compared on one GPU with resident kernels:

  synth   apus_submit_synth: the engine's fill kernel writes generated requests (inputs never leave the device)
  device  apus_submit_device: requests in torch tensors, written by a torch kernel on the caller's stream, packed
          into the ring in stream order (no host copy, no host synchronisation per batch)
  host    apus_submit_uniform: requests in host memory, slots written by host threads and copied over

Five replicas on GPU 0, 16 leader CTAs, 2^20 requests per step, 64 B and 1000 B payloads.  Each step's requests go in
as chunks with at most two chunks in flight (a chunk is submitted once the one before the previous has committed), so
the payload ring never needs more than three chunks.  Prints one JSON line per (payload, way) with committed ops/s, and
for `device` the packing time per chunk (CUDA events around apus_submit_device on the caller's stream, which waits for
the packing), plus the card's name and power limit read in the same run.

  python tools/device_submit_bench.py [--steps 3] [--warmup 1] [--payloads 64,1000] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import apus_b200 as A  # noqa: E402
from apus_b200 import engine as E  # noqa: E402

N_REQ = 1 << 20
REPLICAS, CTAS = 5, 16
SEND, CONNECT = E.SEND, E.CONNECT


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def chunk_of(payload):
    return N_REQ if 2 + payload <= 80 else 1 << 16


def run_leg(way, payload, steps, warmup):
    chunk = chunk_of(payload)
    need = 0 if 2 + payload <= 80 else (2 + payload + 15) // 16 * 16
    ring_bytes = max(1 << 20, 3 * chunk * need)                  # three chunks: exact tiling for apus_submit_synth
    g = A.Group(REPLICAS, devices=[0] * REPLICAS, log_size=A.LOG_SIZE, ring_mode=A.RING_DEVICE, ring_slots=1 << 21,
                ring_bytes=ring_bytes, flags=E.F_DEVICE_STATS | E.F_AUTOPRUNE, leader_ctas=CTAS)
    L = g.leader
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    rng = np.random.default_rng(payload)
    host_pl = rng.integers(0, 256, size=chunk * payload, dtype=np.uint8)
    if way == "device":
        base = torch.from_numpy(host_pl.reshape(chunk, payload)).to(dev)
        pl = torch.empty_like(base)
        types = torch.full((chunk,), SEND, dtype=torch.uint8, device=dev)
        conns = torch.zeros(chunk, dtype=torch.int16, device=dev)
        lens = torch.full((chunk,), payload, dtype=torch.int16, device=dev)
        req_ids = torch.empty(chunk, dtype=torch.int64, device=dev)
        ar = torch.arange(chunk, dtype=torch.int64, device=dev)
        # load torch's kernels before the replica kernels are resident (a lazy load may wait for running kernels)
        torch.add(ar, 0, out=req_ids)
        torch.bitwise_xor(base, 0, out=pl)
    torch.cuda.synchronize()
    g.launch(target=(1 << 64) - 1)
    g.leader.wait_committed(g.prologue(), 30_000_000)
    g.leader.wait_committed(g.submit(CONNECT, 0, 1, b""), 30_000_000)
    req = 2
    ends = []
    pack_ms = []
    t_start = None
    for s in range(warmup + steps):
        if s == warmup:
            t_start = time.perf_counter()
        for c in range(N_REQ // chunk):
            if len(ends) >= 2:
                L.wait_committed(ends[-2], 60_000_000)
            if way == "synth":
                t0 = L.submit_synth(chunk, SEND, 0, req, payload, 0xA5A50000 + payload)
            elif way == "host":
                t0 = L.submit_uniform(chunk, SEND, 0, req, payload, host_pl)
            else:
                with torch.cuda.stream(st):
                    torch.add(ar, req, out=req_ids)              # the producer: torch kernels on the caller's stream
                    torch.bitwise_xor(base, s & 0xFF, out=pl)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    t0 = L.submit_device(types, conns, req_ids, lens, pl, stream=st)
                    e1.record(st)
                if s >= warmup:
                    pack_ms.append((e0, e1))
            req += chunk
            ends.append(t0 + chunk - 1)
        print(f"[{way} {payload} B] step {s}: submitted up to ticket {ends[-1]}, committed {L.committed()}",
              file=sys.stderr, flush=True)
    L.wait_committed(ends[-1], 120_000_000)
    elapsed = time.perf_counter() - t_start
    st.synchronize()
    out = {"way": way, "payload": payload, "requests_per_step": N_REQ, "steps": steps, "chunk": chunk,
           "committed_ops_per_s": steps * N_REQ / elapsed}
    if pack_ms:
        ms = sorted(a.elapsed_time(b) for a, b in pack_ms)
        out["pack_ms_per_chunk_p50"] = ms[len(ms) // 2]
        out["pack_ms_per_chunk_max"] = ms[-1]
        # bytes the packing moves, from shapes: 128 B slot stores + external images, and the input reads
        out["pack_bytes_per_chunk"] = chunk * (128 + need + payload + 1 + 2 + 2 + 8)
    g.stop()
    g.close()
    return out


def main():
    import faulthandler
    faulthandler.dump_traceback_later(90, repeat=True)        # where a stalled leg waits, on stderr
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--payloads", default="64,1000")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available() or A.lib().apus_device_count() < 1:
        raise SystemExit("device_submit_bench.py: no CUDA device; the engine has no CPU fallback")
    info = {"card": card(), "torch": torch.__version__, "replicas": REPLICAS, "leader_ctas": CTAS}
    lines = [json.dumps(info)]
    print(lines[0], flush=True)
    for payload in [int(p) for p in args.payloads.split(",")]:
        for way in ("synth", "device", "host"):
            r = run_leg(way, payload, args.steps, args.warmup)
            lines.append(json.dumps(r))
            print(lines[-1], flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
