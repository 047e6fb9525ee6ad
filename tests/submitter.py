"""Resident submitters for the GPU tests and tools/resident_submitter_bench.py: tests/devicelogic/resident_submit.cu,
compiled with nvcc for sm_90a into a temporary directory against include/ alone, a host handle per launch that keeps
its request arrays and reads back the tickets it handed out, and the request streams and oracle orders the tests use.
Importing this module starts no CUDA context: torch is loaded where it is used."""
import ctypes as C

import numpy as np

import device_build as DB
import streams as S

WAIT, DROP_LAST = 1, 2                      # RS_WAIT, RS_DROP_LAST
OK, TIMED_OUT, STOPPED, NEVER_FITS = 0, 1, 2, 3
STEP_RESERVE, STEP_PUBLISH, STEP_WAIT = 1, 2, 3
ACCEPTED = (1, S.CONNECT, S.SEND, S.CLOSE)     # CSM, CONNECT, SEND, CLOSE
MAX_LEN = 0xFFFF                               # APUS_SUBMITTER_MAX_LEN: a longer cmd is rejected
NOOP = 0

vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


class Args(C.Structure):
    """rs_args of resident_submit.cu"""
    _fields_ = [("types", vp), ("conns", vp), ("req_ids", vp), ("offsets", vp), ("values", vp), ("n", u64),
                ("batch", u32), ("mode", u32), ("timeout_ns", u64), ("tickets", vp), ("lat_ns", vp), ("out", vp)]


_lib = None


def lib():
    """the compiled submitter, loaded (and its kernel loaded into the context) once per process"""
    global _lib
    if _lib is None:
        from apus_b200 import engine as E
        L = DB.load_kernel("resident_submit")
        L.rs_launch.argtypes = [vp, vp, C.c_uint, vp]
        L.rs_load.restype = C.c_int
        L.rs_args_size.restype = C.c_uint
        L.rs_view_size.restype = C.c_uint
        assert L.rs_args_size() == C.sizeof(Args)
        assert L.rs_view_size() == C.sizeof(E.SubmitterView)
        assert L.rs_load() == 0
        _lib = L
    return _lib


class Submitter:
    """one launch of resident_submit on `stream` for `requests` [(type, conn, req_id, payload)], `batch` requests per
    reservation, over `ctas` CTAs"""

    def __init__(self, view, stream, requests, batch=32, ctas=1, mode=0, timeout_s=20.0):
        import torch
        dev = stream.device
        n = len(requests)
        offs = np.zeros(n + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(p) for *_, p in requests])
        vals = np.frombuffer(b"".join(p for *_, p in requests) + b"\0", dtype=np.uint8)

        def t(a):
            return torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        self.view, self.stream, self.n, self.batch, self.ctas = view, stream, n, batch, ctas
        # on the submitter's own stream, which is then synchronised alone: a device-wide synchronise would wait for the
        # resident replica kernels
        with torch.cuda.stream(stream):
            self.types = t(np.array([r[0] for r in requests], dtype=np.uint8))
            self.conns = t(np.array([r[1] for r in requests], dtype=np.uint16).view(np.int16))
            self.req_ids = t(np.array([r[2] for r in requests], dtype=np.uint64).view(np.int64))
            self.offsets = t(offs)
            self.values = t(vals.copy())
            self.tickets = torch.zeros(max(n, 1), dtype=torch.int64, device=dev)
            self.lat = torch.zeros(max((n + batch - 1) // batch, 1), dtype=torch.int64, device=dev)
            self.out = torch.zeros(7, dtype=torch.int64, device=dev)
        stream.synchronize()
        self.a = Args(self.types.data_ptr(), self.conns.data_ptr(), self.req_ids.data_ptr(), self.offsets.data_ptr(),
                      self.values.data_ptr(), n, batch, mode, int(timeout_s * 1e9), self.tickets.data_ptr(),
                      self.lat.data_ptr(), self.out.data_ptr())

    def start(self):
        """launch; a handle may be started again once the previous launch has ended.  Construct it before the replica
        kernels are resident: its torch kernels must be loaded by then"""
        with torch_module().cuda.stream(self.stream):
            self.out.zero_()
        assert lib().rs_launch(C.byref(self.view), C.byref(self.a), self.ctas, self.stream.cuda_stream) == 0
        return self

    def result(self):
        """after the kernel has ended: (failure (step, outcome) or None, requests published, tickets [n])"""
        self.stream.synchronize()
        fail, pub = (int(x) for x in self.out[:2].cpu())
        return ((fail >> 8, fail & 0xFF) if fail else None), pub, self.tickets[:self.n].cpu().tolist()

    def phase_ns(self):
        """after the kernel has ended: thread 0's ns, summed over the CTAs, in the size sums, reserves, puts and
        publishes"""
        self.stream.synchronize()
        return dict(zip(("sum", "reserve", "put", "publish"), (int(x) for x in self.out[3:7].cpu())))

    def latencies_ns(self):
        self.stream.synchronize()
        return self.lat.cpu().tolist()


def torch_module():
    import torch
    return torch


def accepted(req):
    return req[0] in ACCEPTED and len(req[3]) <= MAX_LEN


def written(req):
    """what a request becomes in the log: itself, or the NOOP apus_submit(APUS_NOOP, conn, req_id) writes"""
    typ, conn, rid, payload = req
    return req if accepted(req) else (NOOP, conn, rid, b"")


def ticket_order(requests, tickets, upto=None):
    """the requests as the log holds them: sorted by ticket, rejected ones as NOOPs; only tickets <= upto"""
    pairs = sorted((t, written(r)) for t, r in zip(tickets, requests) if t and (upto is None or t <= upto))
    return [r for _, r in pairs], [t for t, _ in pairs]


def mixed_requests(n, seed, max_len=1500, big_every=0, reject_every=23, conns=4, first_req_id=1):
    """seeded requests of mixed types and sizes: ragged 0..max_len B, every big_every-th up to 64 KiB, every
    reject_every-th of a type the submitter rejects (NOOP, CONFIG, HEAD or 9)"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        typ = int(rng.choice([S.SEND] * 6 + [S.CONNECT, S.CLOSE, 1]))
        if reject_every and k % reject_every == reject_every - 1:
            typ = int(rng.choice([0, 2, 3, 9]))
        ln = int(rng.integers(0, max_len + 1))
        if big_every and k % big_every == big_every - 1:
            ln = int(rng.integers(1500, 65536))
        out.append((typ, int(rng.integers(0, conns)), first_req_id + k, rng.integers(0, 256, ln, dtype=np.uint8).tobytes()))
    return out
