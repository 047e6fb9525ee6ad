"""ctypes binding of include/apus_gpu.h (the C ABI is the product boundary).

`Group` mirrors how the reference deploys a Paxos group: `group_size` replicas,
`server_idx` 0..n-1 (env vars of benchmarks/run.sh:26), one of them the leader.
"""
import ctypes as C
import os
from collections import namedtuple

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libapus_gpu.so")

APUS_OK, APUS_ERROR, APUS_RETRY = 0, 1, -1
NOOP, CSM, CONFIG, HEAD, CONNECT, SEND, CLOSE = 0, 1, 2, 3, 4, 5, 6
RING_HOST_MAPPED, RING_DEVICE = 0, 1
LOG_SIZE = 16384 * 4096
MAX_SERVERS = 13
F_FENCED_ACK, F_DEVICE_STATS, F_AUTOPRUNE, F_FOLLOWER_WALK, F_EXPLICIT = 0x1, 0x2, 0x4, 0x8, 0x80000000
F_HOST_APPLY, F_NO_EXPRESS, F_PROFILE, F_FABRIC = 0x10, 0x20, 0x40, 0x100
F_DEVICE_APPLY = 0x200
F_APPLY_ANY_ROLE = 0x400   # with F_DEVICE_APPLY: the device consumers work on a leader too, and through a take-over
CONSUME_BAD_IDX = 1
WAIT_READY, WAIT_TIMED_OUT, WAIT_RELEASED = 0, 1, 2      # outcomes of Replica.consume_wait (APUS_WAIT_*)
WAIT_NOT_LEADER = 3        # ... and of Replica.read_fence: the leader it knew could not be confirmed
UINT64_MAX = (1 << 64) - 1

u64, u32, u16, u8, i64, i32 = C.c_uint64, C.c_uint32, C.c_uint16, C.c_uint8, C.c_int64, C.c_int32
vp, p64 = C.c_void_p, C.POINTER(C.c_uint64)


class ApusError(RuntimeError):
    pass


class Config(C.Structure):
    _fields_ = [("struct_size", u32), ("device", i32), ("server_idx", u8), ("group_size", u8),
                ("leader_idx", u8), ("ring_mode", u8), ("flags", u32), ("term", u64),
                ("log_size", u64), ("ring_slots", u32), ("ring_bytes", u32), ("leader_ctas", u32), ("reserved", u32),
                ("hb_period_us", u32), ("hb_timeout_us", u32)]


class PeerHandle(C.Structure):
    _fields_ = [("bytes", u8 * 128)]


class LogOffsets(C.Structure):
    _fields_ = [(k, u64) for k in ("head", "apply", "commit", "end", "tail", "old_end", "old_commit", "len")]


class Stats(C.Structure):
    _fields_ = [(k, u64) for k in ("tickets_submitted", "tickets_consumed", "tickets_committed",
                                   "entries_acked", "bytes_replicated", "batches", "kernel_launches",
                                   "lat_samples", "auto_heads", "entries_published")] + [("phase_ns", u64 * 8), ("turn_ns", u64 * 8)]


class ConsumerView(C.Structure):
    """apus_consumer_view_t: what a resident consumer kernel (include/apus_consumer.cuh) takes by value"""
    _fields_ = [("entries", vp), ("log_len", u64), ("index", vp), ("idx_mask", u32), ("pad", u32), ("rec", vp),
                ("cur", vp), ("error", vp), ("status", vp), ("stop", vp), ("stop_epoch", u64)]


# a dormant submitter's apus_submitter_state_t (its replica has not led since attach): the host holds its lock word,
# and lead_term names no term
SUBMITTER_HOST_HELD, SUBMITTER_DORMANT = 2, (1 << 64) - 1


class SubmitterView(C.Structure):
    """apus_submitter_view_t: what a resident submitter kernel (include/apus_submitter.cuh) takes by value.  `state`
    points at apus_submitter_state_t: lock, submitted, pay_head, wrap_next, consumed, rejected, first_rejected and
    lead_term (the term the submitter holds the ring in, SUBMITTER_DORMANT until then), eight 64-bit words"""
    _fields_ = [("slots", vp), ("pay", vp), ("doorbell", vp), ("ring_slots", u32), ("ring_bytes", u32), ("state", vp),
                ("pay_end", vp), ("consumed", vp), ("committed", vp), ("stop", vp), ("stop_epoch", u64)]


class ReaderView(C.Structure):
    """apus_reader_view_t: what a resident reader kernel (include/apus_reader.cuh) takes by value"""
    _fields_ = [("entries", vp), ("log_len", u64), ("index", vp), ("idx_mask", u32), ("pad", u32), ("rec", vp),
                ("role", vp), ("busy", vp), ("member", vp), ("n", u32), ("own", u32), ("on_off", u32), ("rec_off", u32),
                ("sid_off", u32), ("pad2", u32), ("release", vp), ("stop", vp), ("stop_epoch", u64)]


ConsumeStatus = namedtuple("ConsumeStatus", "cursor next_idx need_stride error")
WaitStatus = namedtuple("WaitStatus", "outcome available")
FenceStatus = namedtuple("FenceStatus", "outcome index")

_lib = None

# Every function include/apus_gpu.h declares, in its order: name -> (restype, argtypes).  load_library applies them all,
# so that no caller depends on ctypes' default of a 32-bit int; tests/test_abi.py checks each against the header.
SIGNATURES = {
    "apus_abi_version": (C.c_int, []),
    "apus_last_error": (C.c_char_p, []),
    "apus_device_count": (C.c_int, []),
    "apus_device_numa_node": (C.c_int, [C.c_int]),
    "apus_replica_create": (C.c_int, [C.POINTER(Config), C.POINTER(vp)]),
    "apus_replica_destroy": (None, [vp]),
    "apus_replica_export": (C.c_int, [vp, C.POINTER(PeerHandle)]),
    "apus_replica_connect": (C.c_int, [vp, u8, C.POINTER(PeerHandle)]),
    "apus_group_multicast": (C.c_int, [C.POINTER(vp), C.c_int]),
    "apus_replicas_launch": (C.c_int, [C.POINTER(vp), C.c_int, u64]),
    "apus_replica_wait": (C.c_int, [vp, i64]),
    "apus_replica_last_launch_ms": (C.c_int, [vp, C.POINTER(C.c_float)]),
    "apus_replicas_stop": (C.c_int, [C.POINTER(vp), C.c_int]),
    "apus_submit": (C.c_int, [vp, u8, u16, u64, vp, u16, p64]),
    "apus_submit_batch": (C.c_int, [vp, u32, vp, vp, vp, vp, vp, C.c_size_t, p64]),
    "apus_submit_uniform": (C.c_int, [vp, u32, u8, u16, u64, u16, vp, C.c_size_t, p64]),
    "apus_submit_synth": (C.c_int, [vp, u32, u8, u16, u64, u16, u32, p64]),
    "apus_synth_byte": (u8, [u32, u64, u32]),
    "apus_submit_device": (C.c_int, [vp, u32, vp, vp, vp, vp, vp, C.c_size_t, vp, p64]),
    "apus_submit_device_packed": (C.c_int, [vp, u32, vp, vp, vp, vp, vp, u64, vp, p64]),
    "apus_device_submit_status": (C.c_int, [vp, p64, p64]),
    "apus_submit_defer": (C.c_int, [vp, C.c_int]),
    "apus_submit_flush": (C.c_int, [vp]),
    "apus_submit_release": (C.c_int, [vp, u64]),
    "apus_committed_tickets": (u64, [vp]),
    "apus_progress": (C.c_int, [vp, p64, p64]),
    "apus_wait_committed": (C.c_int, [vp, u64, i64]),
    "apus_stream_wait_committed": (C.c_int, [vp, u64, vp]),
    "apus_committed_word": (vp, [vp]),
    "apus_closed_loop": (C.c_int, [vp, u32, u16, u16, u64, vp]),
    "apus_log_offsets": (C.c_int, [vp, C.POINTER(LogOffsets)]),
    "apus_log_read": (C.c_int, [vp, u64, u64, vp]),
    "apus_get_stats": (C.c_int, [vp, C.POINTER(Stats)]),
    "apus_latency_samples": (C.c_int, [vp, vp, u32, C.POINTER(u32)]),
    "apus_set_applied": (C.c_int, [vp, u64]),
    "apus_log_read_range": (C.c_int, [vp, u64, u64, vp, u64, p64]),
    "apus_consume_device": (C.c_int, [vp, u32, vp, vp, vp, vp, vp, vp, C.c_size_t, vp, vp]),
    "apus_consume_device_packed": (C.c_int, [vp, u32, vp, vp, vp, vp, vp, vp, u64, vp, vp]),
    "apus_consume_status": (C.c_int, [vp, p64, p64, p64, p64]),
    "apus_consume_wait": (C.c_int, [vp, u32, u32, vp, vp]),
    "apus_consume_wait_release": (C.c_int, [vp]),
    "apus_consume_wait_status": (C.c_int, [vp, p64, p64]),
    "apus_consume_mark": (C.c_int, [vp, vp, vp]),
    "apus_consume_seed": (C.c_int, [vp, u64, u64]),
    "apus_read_fence": (C.c_int, [vp, u32, vp, vp, vp]),
    "apus_read_fence_status": (C.c_int, [vp, p64, p64]),
    "apus_consumer_attach": (C.c_int, [vp, vp, C.POINTER(ConsumerView)]),
    "apus_consumer_detach": (C.c_int, [vp]),
    "apus_submitter_attach": (C.c_int, [vp, vp, C.POINTER(SubmitterView)]),
    "apus_submitter_detach": (C.c_int, [vp]),
    "apus_reader_attach": (C.c_int, [vp, vp, C.POINTER(ReaderView)]),
    "apus_reader_detach": (C.c_int, [vp]),
    "apus_leader_suspect": (u64, [vp]),
    "apus_last_commit_ns": (u64, [vp]),
    "apus_ctl_read": (C.c_int, [vp, vp]),
    "apus_ctl_set_sid": (C.c_int, [vp, u64]),
    "apus_ctl_reset_votes": (C.c_int, [vp]),
    "apus_ctl_clear_vote_request": (C.c_int, [vp, u8]),
    "apus_ctl_send_vote_request": (C.c_int, [vp, u8, u64, u64, u64, vp]),
    "apus_ctl_send_vote_ack": (C.c_int, [vp, u8, u64]),
    "apus_ctl_heartbeat": (C.c_int, [vp, p64]),
    "apus_ctl_last_entry": (C.c_int, [vp, p64, p64, p64, p64]),
    "apus_ctl_adjust_follower": (C.c_int, [vp, u8, u64, p64]),
    "apus_replica_set_role": (C.c_int, [vp, u8, u64]),
    "apus_follower_beats": (C.c_int, [vp, p64]),
    "apus_replica_disconnect": (C.c_int, [vp, u8]),
    "apus_set_head": (C.c_int, [vp, u64]),
    "apus_remote_apply_offsets": (C.c_int, [vp, p64]),
}
EXPORTS = list(SIGNATURES)


def load_library(path=LIB_PATH):
    """Load libapus_gpu.so and give every ABI function its signature; raises (no fallback) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise ApusError(f"{path} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(make -C apus_b200/csrc). There is no CPU fallback.")
    L = C.CDLL(path)
    for name, (restype, argtypes) in SIGNATURES.items():
        try:
            fn = getattr(L, name)
        except AttributeError:
            raise ApusError(f"{path} does not export {name}: rebuild it (make -C apus_b200/csrc)") from None
        fn.restype, fn.argtypes = restype, argtypes
    _lib = L
    return L


def lib():
    return load_library()


def _ck(rc, what):
    if rc == APUS_OK:
        return
    msg = lib().apus_last_error().decode(errors="replace")
    if rc == APUS_RETRY:
        raise BlockingIOError(f"{what}: {msg}")
    raise ApusError(f"{what}: {msg}")


def _check_tensors(what, dev, spec):
    """Raise ApusError for the first (name, tensor, dtypes, shape) of `spec` whose tensor is not a contiguous torch tensor
    on `dev` with one of `dtypes` and that shape (None: any 1-D shape): the device calls hand raw pointers to kernels."""
    import torch
    for name, t, dtypes, shape in spec:
        if not isinstance(t, torch.Tensor):
            raise ApusError(f"{what}: {name} must be a torch tensor")
        if t.device != dev:
            raise ApusError(f"{what}: {name} is on {t.device}, the replica is on {dev}")
        if t.dtype not in dtypes:
            raise ApusError(f"{what}: {name} has dtype {t.dtype}, expected one of {dtypes}")
        if (tuple(t.shape) != shape) if shape is not None else t.dim() != 1:
            raise ApusError(f"{what}: {name} has shape {tuple(t.shape)}, expected {'1-D' if shape is None else shape}")
        if not t.is_contiguous():
            raise ApusError(f"{what}: {name} is not contiguous")


class Replica:
    def __init__(self, device, server_idx, group_size, leader_idx=0, term=1, log_size=0,
                 ring_mode=RING_HOST_MAPPED, ring_slots=0, ring_bytes=0, flags=None, leader_ctas=0,
                 hb_period_us=0, hb_timeout_us=0):
        cfg = Config()
        cfg.leader_ctas = leader_ctas
        cfg.hb_period_us, cfg.hb_timeout_us = hb_period_us, hb_timeout_us
        cfg.struct_size = C.sizeof(Config)
        cfg.device, cfg.server_idx, cfg.group_size, cfg.leader_idx = device, server_idx, group_size, leader_idx
        cfg.ring_mode, cfg.term, cfg.log_size = ring_mode, term, log_size
        cfg.ring_slots, cfg.ring_bytes = ring_slots, ring_bytes
        cfg.flags = 0 if flags is None else (flags | F_EXPLICIT)
        self.h = C.c_void_p()
        _ck(lib().apus_replica_create(C.byref(cfg), C.byref(self.h)), "apus_replica_create")
        self.cfg = cfg
        self.device, self.idx, self.n, self.leader = device, server_idx, group_size, leader_idx
        self.log_len = log_size or LOG_SIZE

    @property
    def is_leader(self):
        return self.idx == self.leader

    def close(self):
        if self.h:
            lib().apus_replica_destroy(self.h)
            self.h = C.c_void_p()

    def export(self) -> bytes:
        ph = PeerHandle()
        _ck(lib().apus_replica_export(self.h, C.byref(ph)), "apus_replica_export")
        return bytes(ph.bytes)

    def connect(self, peer_idx, blob: bytes):
        ph = PeerHandle()
        C.memmove(ph.bytes, blob, 128)
        _ck(lib().apus_replica_connect(self.h, peer_idx, C.byref(ph)), "apus_replica_connect")

    def wait(self, timeout_ms=-1):
        _ck(lib().apus_replica_wait(self.h, timeout_ms), "apus_replica_wait")

    def last_launch_ms(self):
        ms = C.c_float()
        _ck(lib().apus_replica_last_launch_ms(self.h, C.byref(ms)), "apus_replica_last_launch_ms")
        return float(ms.value)

    def submit(self, typ, conn, req_id, payload=b""):
        t = u64()
        buf = (u8 * max(len(payload), 1)).from_buffer_copy(bytes(payload) or b"\0")
        _ck(lib().apus_submit(self.h, typ, conn, req_id, C.cast(buf, C.c_void_p), len(payload), C.byref(t)),
            "apus_submit")
        return int(t.value)

    def submit_batch(self, types, conns, req_ids, lens, payloads, stride):
        """numpy arrays: types u8[n], conns u16[n], req_ids u64[n], lens u16[n], payloads u8[n*stride]."""
        n = len(types)
        types = np.ascontiguousarray(types, dtype=np.uint8)
        conns = np.ascontiguousarray(conns, dtype=np.uint16)
        req_ids = np.ascontiguousarray(req_ids, dtype=np.uint64)
        lens = np.ascontiguousarray(lens, dtype=np.uint16)
        pp = None
        if payloads is not None:
            payloads = np.ascontiguousarray(payloads, dtype=np.uint8)
            pp = payloads.ctypes.data
        t = u64()
        _ck(lib().apus_submit_batch(self.h, n, types.ctypes.data, conns.ctypes.data, req_ids.ctypes.data,
                                    lens.ctypes.data, pp, stride, C.byref(t)), "apus_submit_batch")
        return int(t.value)

    def submit_uniform(self, n, typ, conn, first_req_id, length, payloads, stride=None):
        """n requests of one shape, filled by the engine's host threads (apus_submit_uniform)."""
        pp = None
        if payloads is not None and length:
            payloads = np.ascontiguousarray(payloads, dtype=np.uint8)
            pp = payloads.ctypes.data
        t = u64()
        _ck(lib().apus_submit_uniform(self.h, n, typ, conn, first_req_id, length, pp, length if stride is None else stride,
                                      C.byref(t)), "apus_submit_uniform")
        return int(t.value)

    def submit_synth(self, n, typ, conn, first_req_id, length, seed):
        """n device-generated requests written straight into the HBM submission ring."""
        t = u64()
        _ck(lib().apus_submit_synth(self.h, n, typ, conn, first_req_id, length, seed, C.byref(t)), "apus_submit_synth")
        return int(t.value)

    def _stream(self, stream):
        import torch
        if stream is None:
            return torch.cuda.current_stream(self.device)
        if stream.device != torch.device("cuda", self.device):
            raise ApusError(f"stream on {stream.device}, the leader is on cuda:{self.device}")
        return stream

    def submit_device(self, types, conns, req_ids, lens, payloads, stream=None):
        """n requests whose fields are CUDA tensors on the leader's device, packed into the HBM submission ring in
        `stream` order (apus_submit_device): types uint8 [n], conns int16/uint16 [n], req_ids int64 [n] (as uint64),
        lens int16/uint16/int32 [n], payloads uint8 [n, stride].  All contiguous.  Returns the first ticket; the
        tensors may be overwritten or freed in stream order as soon as this returns.  Invalid requests (a type that
        is not CSM/CONNECT/SEND/CLOSE, len > stride) become NOOP entries, see device_submit_status()."""
        import torch
        dev = torch.device("cuda", self.device)
        if payloads is None or not isinstance(payloads, torch.Tensor) or payloads.dim() != 2:
            raise ApusError("submit_device: payloads must be a 2-D uint8 CUDA tensor [n, stride]")
        n, stride = payloads.shape
        _check_tensors("submit_device", dev, (
            ("types", types, (torch.uint8,), (n,)), ("conns", conns, (torch.int16, torch.uint16), (n,)),
            ("req_ids", req_ids, (torch.int64,), (n,)), ("lens", lens, (torch.int16, torch.uint16, torch.int32), (n,)),
            ("payloads", payloads, (torch.uint8,), (n, stride))))
        s = self._stream(stream)
        if lens.dtype == torch.int32:
            # the ABI takes uint16 lengths: a length outside [0, stride] must stay > stride after the narrowing
            if stride >= 0xFFFF:
                raise ApusError("submit_device: int32 lengths need stride < 65535 (use uint16 lengths)")
            with torch.cuda.stream(s):
                lens = torch.where((lens >= 0) & (lens <= stride), lens, 0xFFFF).to(torch.int16)
        t = u64()
        _ck(lib().apus_submit_device(self.h, n, types.data_ptr(), conns.data_ptr(), req_ids.data_ptr(), lens.data_ptr(),
                                     payloads.data_ptr() if stride else None, stride, s.cuda_stream, C.byref(t)),
            "apus_submit_device")
        return int(t.value)

    def submit_device_packed(self, types, conns, req_ids, offsets, values, stream=None):
        """n requests in the packed (jagged) layout, packed into the HBM submission ring in `stream` order
        (apus_submit_device_packed): request k's cmd is values[offsets[k]:offsets[k+1]].  types uint8 [n], conns
        int16/uint16 [n], req_ids int64 [n] (as uint64), offsets int64 [n+1] (offsets[0] may be > 0), values a 1-D uint8
        tensor; all contiguous CUDA tensors on the leader's device.  The payload-ring reservation is bounded by
        values.numel() (min(n * 65552, round16(values.numel() + 17 n)) bytes), so pass only the slice of values the batch
        uses.  Returns the first ticket.  A type that is not CSM/CONNECT/SEND/CLOSE or a cmd above 65535 B becomes a
        NOOP entry; offsets that decrease or end past values.numel() turn the whole batch into NOOPs (see
        device_submit_status())."""
        import torch
        dev = torch.device("cuda", self.device)
        if not isinstance(types, torch.Tensor) or types.dim() != 1:
            raise ApusError("submit_device_packed: types must be a 1-D uint8 CUDA tensor [n]")
        n = types.shape[0]
        _check_tensors("submit_device_packed", dev, (
            ("types", types, (torch.uint8,), (n,)), ("conns", conns, (torch.int16, torch.uint16), (n,)),
            ("req_ids", req_ids, (torch.int64,), (n,)), ("offsets", offsets, (torch.int64,), (n + 1,)),
            ("values", values, (torch.uint8,), None)))
        s = self._stream(stream)
        nv = values.numel()
        t = u64()
        _ck(lib().apus_submit_device_packed(self.h, n, types.data_ptr(), conns.data_ptr(), req_ids.data_ptr(),
                                            offsets.data_ptr(), values.data_ptr() if nv else None, nv, s.cuda_stream,
                                            C.byref(t)), "apus_submit_device_packed")
        return int(t.value)

    def device_submit_status(self):
        """(requests of device batches written as NOOPs, ticket of the first of them or 0)"""
        rej, first = u64(), u64()
        _ck(lib().apus_device_submit_status(self.h, C.byref(rej), C.byref(first)), "apus_device_submit_status")
        return int(rej.value), int(first.value)

    def consume_device(self, max_n, stride, out=None, stream=None):
        """Follower created with F_DEVICE_APPLY, or any replica created with F_DEVICE_APPLY | F_APPLY_ANY_ROLE: the next
        committed entries, at most max_n of them, into CUDA tensors on this replica's device, in `stream` order
        (apus_consume_device).  On a leader they are every committed entry of its log, its own tickets and the entries
        of earlier terms alike: every replica applies the same rows in the same order.  Returns (idx int64 [max_n], types uint8
        [max_n], conns int16 [max_n], req_ids int64 [max_n], lens int16 [max_n], payloads uint8 [max_n, stride],
        count int32 [1]): rows 0 .. count-1 are the CSM-like entries examined; NOOP / CONFIG / HEAD entries are
        skipped, idx shows them.  Read count after synchronising with `stream`.  `out`: those seven tensors to
        fill (allocated when None); int16 or uint16 for conns and lens, int32 or uint32 for count."""
        import torch
        dev = torch.device("cuda", self.device)
        s = self._stream(stream)
        if out is None:
            with torch.cuda.stream(s):
                out = (torch.empty(max_n, dtype=torch.int64, device=dev), torch.empty(max_n, dtype=torch.uint8, device=dev),
                       torch.empty(max_n, dtype=torch.int16, device=dev), torch.empty(max_n, dtype=torch.int64, device=dev),
                       torch.empty(max_n, dtype=torch.int16, device=dev),
                       torch.empty((max_n, stride), dtype=torch.uint8, device=dev),
                       torch.empty(1, dtype=torch.int32, device=dev))
        if len(out) != 7:
            raise ApusError("consume_device: out must be (idx, types, conns, req_ids, lens, payloads, count)")
        idx, types, conns, req_ids, lens, payloads, count = out
        _check_tensors("consume_device", dev, (
            ("idx", idx, (torch.int64,), (max_n,)), ("types", types, (torch.uint8,), (max_n,)),
            ("conns", conns, (torch.int16, torch.uint16), (max_n,)), ("req_ids", req_ids, (torch.int64,), (max_n,)),
            ("lens", lens, (torch.int16, torch.uint16), (max_n,)),
            ("payloads", payloads, (torch.uint8,), (max_n, stride)), ("count", count, (torch.int32, torch.uint32), (1,))))
        _ck(lib().apus_consume_device(self.h, max_n, idx.data_ptr(), types.data_ptr(), conns.data_ptr(),
                                      req_ids.data_ptr(), lens.data_ptr(), payloads.data_ptr() if stride else None,
                                      stride, count.data_ptr(), s.cuda_stream), "apus_consume_device")
        return out

    def consume_device_packed(self, max_n, values_cap, out=None, stream=None):
        """consume_device with packed output (apus_consume_device_packed), in the same roles.  Returns (idx int64 [max_n], types uint8
        [max_n], conns int16 [max_n], req_ids int64 [max_n], offsets int64 [max_n+1], values uint8 [values_cap], count
        int32 [1]): row r's cmd is values[offsets[r]:offsets[r+1]], offsets[0] = 0, for the count rows written.  The
        call stops before the first cmd that would end past values_cap; when that is the first row, consume_status()
        .need_stride is the capacity it needs.  `out`: those seven tensors to fill (allocated when None); int16 or
        uint16 for conns, int32 or uint32 for count."""
        import torch
        dev = torch.device("cuda", self.device)
        s = self._stream(stream)
        if out is None:
            with torch.cuda.stream(s):
                out = (torch.empty(max_n, dtype=torch.int64, device=dev), torch.empty(max_n, dtype=torch.uint8, device=dev),
                       torch.empty(max_n, dtype=torch.int16, device=dev), torch.empty(max_n, dtype=torch.int64, device=dev),
                       torch.empty(max_n + 1, dtype=torch.int64, device=dev),
                       torch.empty(values_cap, dtype=torch.uint8, device=dev),
                       torch.empty(1, dtype=torch.int32, device=dev))
        if len(out) != 7:
            raise ApusError("consume_device_packed: out must be (idx, types, conns, req_ids, offsets, values, count)")
        idx, types, conns, req_ids, offsets, values, count = out
        _check_tensors("consume_device_packed", dev, (
            ("idx", idx, (torch.int64,), (max_n,)), ("types", types, (torch.uint8,), (max_n,)),
            ("conns", conns, (torch.int16, torch.uint16), (max_n,)), ("req_ids", req_ids, (torch.int64,), (max_n,)),
            ("offsets", offsets, (torch.int64,), (max_n + 1,)), ("values", values, (torch.uint8,), (values_cap,)),
            ("count", count, (torch.int32, torch.uint32), (1,))))
        _ck(lib().apus_consume_device_packed(self.h, max_n, idx.data_ptr(), types.data_ptr(), conns.data_ptr(),
                                             req_ids.data_ptr(), offsets.data_ptr(),
                                             values.data_ptr() if values_cap else None, values_cap, count.data_ptr(),
                                             s.cuda_stream), "apus_consume_device_packed")
        return out

    def consume_status(self):
        """(cursor offset, idx of the next entry, stride the entry that stopped the latest call needs or 0,
        CONSUME_* error or 0), as the latest consume call that ran left them"""
        cur, nidx, need, err = u64(), u64(), u64(), u64()
        _ck(lib().apus_consume_status(self.h, C.byref(cur), C.byref(nidx), C.byref(need), C.byref(err)),
            "apus_consume_status")
        return ConsumeStatus(int(cur.value), int(nidx.value), int(need.value), int(err.value))

    def consume_wait(self, min_entries, timeout_us, outcome=None, stream=None):
        """Make the consumers wait in `stream` order, without the host, until at least min_entries committed entries
        (NOOP / CONFIG / HEAD included) lie past the cursor, or a release, or timeout_us from when the wait starts to
        run (apus_consume_wait), in the roles consume_device accepts.  A consume call made after it sees at least the
        entries it waited for.  `outcome`: an int32 or uint32 CUDA tensor [1] on this replica's device that receives
        WAIT_READY, WAIT_TIMED_OUT or WAIT_RELEASED, for device code downstream; returned (None when not given)."""
        import torch
        dev = torch.device("cuda", self.device)
        s = self._stream(stream)
        if outcome is not None:
            _check_tensors("consume_wait", dev, (("outcome", outcome, (torch.int32, torch.uint32), (1,)),))
        _ck(lib().apus_consume_wait(self.h, min_entries, timeout_us, None if outcome is None else outcome.data_ptr(),
                                    s.cuda_stream), "apus_consume_wait")
        return outcome

    def consume_wait_release(self):
        """end every consume wait enqueued so far (they report WAIT_RELEASED); later waits are not affected"""
        _ck(lib().apus_consume_wait_release(self.h), "apus_consume_wait_release")

    def consume_wait_status(self):
        """(WAIT_* outcome of the latest consume wait that ran, or UINT64_MAX before any; committed entries past the
        cursor when it ended)"""
        o, a = u64(), u64()
        _ck(lib().apus_consume_wait_status(self.h, C.byref(o), C.byref(a)), "apus_consume_wait_status")
        return WaitStatus(int(o.value), int(a.value))

    def consume_mark(self, out=None, stream=None):
        """Write the consumers' position {cursor offset, idx of the next entry}, as the consume calls before it left it,
        into a 2-word device tensor in `stream` order (apus_consume_mark), in the roles consume_device accepts.  A copy
        of the application's state enqueued on `stream` right behind it is the state at that position: seed a
        replacement replica with consume_seed(*mark) and give it the copy.  Next idx 0 marks a consumer stopped by
        CONSUME_BAD_IDX.  `out`: an int64 or uint64 CUDA tensor [2] on this replica's device, 16 B aligned (allocated when
        None); returned."""
        import torch
        dev = torch.device("cuda", self.device)
        s = self._stream(stream)
        if out is None:
            with torch.cuda.stream(s):
                out = torch.empty(2, dtype=torch.int64, device=dev)
        _check_tensors("consume_mark", dev, (("out", out, (torch.int64, torch.uint64), (2,)),))
        _ck(lib().apus_consume_mark(self.h, out.data_ptr(), s.cuda_stream), "apus_consume_mark")
        return out

    def consume_seed(self, cursor, next_idx):
        """Start the consumers of a fresh follower (F_DEVICE_APPLY | F_APPLY_ANY_ROLE, stopped, empty log, no consume call
        yet) at a mark another replica's consume_mark wrote (apus_consume_seed); the leader's adjustment then accepts
        it from there"""
        _ck(lib().apus_consume_seed(self.h, int(cursor), int(next_idx)), "apus_consume_seed")

    def read_fence(self, timeout_us, index=None, outcome=None, stream=None):
        """Enqueue a read fence in `stream` order (apus_read_fence; F_DEVICE_APPLY | F_APPLY_ANY_ROLE): it ends
        WAIT_READY once this replica holds every entry committed anywhere in the group before it began to run, and then
        writes the read index F -- a state that has applied through idx F answers a linearizable read.  WAIT_NOT_LEADER:
        the leader this replica knew could not be confirmed; WAIT_TIMED_OUT / WAIT_RELEASED as consume_wait.  `index`:
        an int64 or uint64 CUDA tensor [1] on this replica's device (written on READY only); `outcome`: an int32 or
        uint32 one; each allocated when None.  Returns (index, outcome)."""
        import torch
        dev = torch.device("cuda", self.device)
        s = self._stream(stream)
        with torch.cuda.stream(s):
            if index is None:
                index = torch.zeros(1, dtype=torch.int64, device=dev)
            if outcome is None:
                outcome = torch.full((1,), -1, dtype=torch.int32, device=dev)
        _check_tensors("read_fence", dev, (("index", index, (torch.int64, torch.uint64), (1,)),
                                           ("outcome", outcome, (torch.int32, torch.uint32), (1,))))
        _ck(lib().apus_read_fence(self.h, timeout_us, index.data_ptr(), outcome.data_ptr(), s.cuda_stream),
            "apus_read_fence")
        return index, outcome

    def read_fence_status(self):
        """(outcome of the latest read fence that ran, or UINT64_MAX before any; its read index, 0 unless READY)"""
        o, i = u64(), u64()
        _ck(lib().apus_read_fence_status(self.h, C.byref(o), C.byref(i)), "apus_read_fence_status")
        return FenceStatus(int(o.value), int(i.value))

    def consumer_attach(self, stream=None):
        """Attach a resident consumer (apus_consumer_attach), in the roles consume_device accepts: consume work enqueued
        before has run when this returns.  `stream`: the stream its kernel will be launched on (default: the current
        stream of this replica's device).  Returns the ConsumerView to pass to that kernel by value.  Until
        consumer_detach(), consume_device*, consume_wait and consume_mark are refused."""
        s = self._stream(stream)
        v = ConsumerView()
        _ck(lib().apus_consumer_attach(self.h, s.cuda_stream, C.byref(v)), "apus_consumer_attach")
        return v

    def consumer_detach(self):
        """Ask the resident consumer to end and wait for the stream it was attached with (apus_consumer_detach); the
        stream-ordered calls then continue from the cursor it left"""
        _ck(lib().apus_consumer_detach(self.h), "apus_consumer_detach")

    def submitter_attach(self, stream=None):
        """Attach a resident submitter to this replica (apus_submitter_attach; APUS_RING_DEVICE only).  On a leader it
        is active at once: everything the host submitted has reached the ring when this returns, and until
        submitter_detach() every call that writes the ring, and set_role, is refused.  On a follower it is dormant: its
        reserves end NOT_LEADER and the host calls behave as without it, until the first launch that runs this replica
        as leader hands the ring over.  `stream`: the stream its kernel will be launched on (default: the current
        stream of this replica's device).  Returns the SubmitterView to pass to that kernel by value."""
        s = self._stream(stream)
        v = SubmitterView()
        _ck(lib().apus_submitter_attach(self.h, s.cuda_stream, C.byref(v)), "apus_submitter_attach")
        return v

    def submitter_detach(self):
        """Ask the resident submitter to end, wait for its stream and, if it was active, hand the ring back to the host
        (apus_submitter_detach): the next host ticket follows the last one it published"""
        _ck(lib().apus_submitter_detach(self.h), "apus_submitter_detach")

    def reader_attach(self, stream=None):
        """Attach a resident reader (apus_reader_attach; F_DEVICE_APPLY | F_APPLY_ANY_ROLE, no peer mapped through CUDA
        IPC).  `stream`: the stream its kernel will be launched on (default: the current stream of this replica's
        device).  Returns the ReaderView to pass to that kernel by value.  Until reader_detach(), connecting a peer
        through CUDA IPC is refused; everything else stays accepted."""
        s = self._stream(stream)
        v = ReaderView()
        _ck(lib().apus_reader_attach(self.h, s.cuda_stream, C.byref(v)), "apus_reader_attach")
        return v

    def reader_detach(self):
        """Ask the resident reader to end and wait for the stream it was attached with (apus_reader_detach)"""
        _ck(lib().apus_reader_detach(self.h), "apus_reader_detach")

    def wait_committed_on_stream(self, ticket, stream=None):
        """make `stream` (default: the current stream of the leader's device) wait until `ticket` is committed"""
        s = self._stream(stream)
        _ck(lib().apus_stream_wait_committed(self.h, ticket, s.cuda_stream), "apus_stream_wait_committed")

    def committed_word(self):
        """device-visible address of the committed-tickets word (pinned, mapped)"""
        return int(lib().apus_committed_word(self.h) or 0)

    def release(self, ticket):
        _ck(lib().apus_submit_release(self.h, ticket), "apus_submit_release")

    def set_applied(self, offset):
        _ck(lib().apus_set_applied(self.h, offset), "apus_set_applied")

    def read_range(self, start, stop, cap=1 << 20):
        out = np.empty(cap, dtype=np.uint8)
        got = u64()
        _ck(lib().apus_log_read_range(self.h, start, stop, out.ctypes.data, cap, C.byref(got)), "apus_log_read_range")
        return out[: got.value].copy()

    def leader_suspect(self):
        return int(lib().apus_leader_suspect(self.h))

    def last_commit_ns(self):
        return int(lib().apus_last_commit_ns(self.h))

    def defer(self, on=True):
        _ck(lib().apus_submit_defer(self.h, 1 if on else 0), "apus_submit_defer")

    def flush(self):
        _ck(lib().apus_submit_flush(self.h), "apus_submit_flush")

    def committed(self):
        return int(lib().apus_committed_tickets(self.h))

    def progress(self):
        off, cnt = u64(), u64()
        _ck(lib().apus_progress(self.h, C.byref(off), C.byref(cnt)), "apus_progress")
        return int(off.value), int(cnt.value)

    def wait_committed(self, ticket, timeout_us=10_000_000):
        _ck(lib().apus_wait_committed(self.h, ticket, timeout_us), "apus_wait_committed")

    def closed_loop(self, n, payload_len, conn, first_req_id):
        """n requests, one in flight; returns host-clock latencies in ns (uint32 array)."""
        out = np.empty(n, dtype=np.uint32)
        _ck(lib().apus_closed_loop(self.h, n, payload_len, conn, first_req_id, out.ctypes.data), "apus_closed_loop")
        return out

    def offsets(self):
        o = LogOffsets()
        _ck(lib().apus_log_offsets(self.h, C.byref(o)), "apus_log_offsets")
        return {k: int(getattr(o, k)) for k, _ in LogOffsets._fields_}

    def image(self, start=0, stop=None):
        stop = self.log_len if stop is None else stop
        out = np.empty(stop - start, dtype=np.uint8)
        if stop > start:
            _ck(lib().apus_log_read(self.h, start, stop - start, out.ctypes.data), "apus_log_read")
        return out

    def stats(self):
        s = Stats()
        _ck(lib().apus_get_stats(self.h, C.byref(s)), "apus_get_stats")
        d = {k: int(getattr(s, k)) for k, _ in Stats._fields_ if k not in ("phase_ns", "turn_ns")}
        d["phase_ns"] = [int(x) for x in s.phase_ns]
        d["turn_ns"] = [int(x) for x in s.turn_ns]
        return d

    def latency_ns(self, max_samples=65536):
        out = np.empty(max_samples, dtype=np.uint32)
        n = u32()
        _ck(lib().apus_latency_samples(self.h, out.ctypes.data, max_samples, C.byref(n)), "apus_latency_samples")
        return out[: n.value].copy()

    def set_head(self, head):
        _ck(lib().apus_set_head(self.h, head), "apus_set_head")

    def remote_apply_offsets(self):
        arr = (u64 * MAX_SERVERS)()
        _ck(lib().apus_remote_apply_offsets(self.h, arr), "apus_remote_apply_offsets")
        return [int(x) for x in arr]


def synth_payload(seed: int, req_id: int, length: int) -> bytes:
    """Payload of the device-generated request `req_id` (apus_submit_synth), computed on the host with numpy --
    the same integer mix the fill kernel runs (apus_slot.h: synth_word)."""
    if length == 0:
        return b""
    w = np.arange((length + 3) // 4, dtype=np.uint64)
    x = (np.uint64(seed) ^ np.uint64((req_id * 0x9E3779B1) & 0xFFFFFFFF) ^ np.uint64(((req_id >> 32) * 0x7F4A7C15) & 0xFFFFFFFF)
         ^ ((w * np.uint64(0x85EBCA77)) & np.uint64(0xFFFFFFFF)))
    M = np.uint64(0xFFFFFFFF)
    x ^= x >> np.uint64(16); x = (x * np.uint64(0x7FEB352D)) & M
    x ^= x >> np.uint64(15); x = (x * np.uint64(0x846CA68B)) & M
    x ^= x >> np.uint64(16)
    return x.astype(np.uint32).view(np.uint8)[:length].tobytes()


def pin_to_device_node(device: int):
    """Run this process on the CPUs of the NUMA node next to `device` (its pinned rings are then allocated there too).
    Returns the node, or None when the topology is not exposed."""
    try:
        node = int(lib().apus_device_numa_node(device))
        if node < 0:
            return None
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        cpus &= os.sched_getaffinity(0)
        if cpus:
            os.sched_setaffinity(0, cpus)
            return node
    except Exception:                                        # noqa: BLE001 - best effort
        pass
    return None


def cid_image(n: int) -> bytes:
    """dare_cid_t of a fresh stable group (dare_server.c:285-291)."""
    return (0).to_bytes(8, "little") + bytes([n, 0, 0, 0]) + ((1 << n) - 1).to_bytes(4, "little")


class Group:
    """All replicas of one Paxos group inside this process (tests, 1..8 GPUs)."""

    def __init__(self, n, devices=None, leader=0, term=1, log_size=0, ring_mode=RING_HOST_MAPPED,
                 ring_slots=0, ring_bytes=0, flags=None, leader_ctas=0, hb_period_us=0, hb_timeout_us=0):
        ndev = lib().apus_device_count()
        if ndev <= 0:
            raise ApusError("no CUDA device visible: the engine has no CPU fallback")
        if devices is None:
            devices = [i % ndev for i in range(n)]
        self.n, self.leader_idx, self.devices = n, leader, list(devices)
        self.replicas = [Replica(devices[i], i, n, leader, term, log_size, ring_mode, ring_slots, ring_bytes, flags,
                                 leader_ctas, hb_period_us, hb_timeout_us) for i in range(n)]
        blobs = [r.export() for r in self.replicas]
        for r in self.replicas:
            for j, b in enumerate(blobs):
                if j != r.idx:
                    r.connect(j, b)
        self.tickets = 0

    @property
    def leader(self) -> Replica:
        return self.replicas[self.leader_idx]

    def close(self):
        for r in self.replicas:
            r.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        try:
            self.stop()
        except Exception:
            pass
        self.close()

    def launch(self, target=None):
        """One fused launch per device; `target` = cumulative tickets (None -> all submitted)."""
        target = self.tickets if target is None else target
        by_dev = {}
        for r in self.replicas:
            by_dev.setdefault(r.device, []).append(r)
        # followers first, so a leader never waits for a CTA that is not scheduled yet
        for dev, rs in sorted(by_dev.items(), key=lambda kv: any(r.is_leader for r in kv[1])):
            arr = (C.c_void_p * len(rs))(*[r.h for r in rs])
            _ck(lib().apus_replicas_launch(arr, len(rs), target), "apus_replicas_launch")

    def wait(self, timeout_ms=60_000):
        for r in self.replicas:
            r.wait(timeout_ms)

    def stop(self):
        arr = (C.c_void_p * self.n)(*[r.h for r in self.replicas])
        _ck(lib().apus_replicas_stop(arr, self.n), "apus_replicas_stop")

    def multicast(self):
        """Bind the replicas' regions (created with F_FABRIC, one GPU each) to an NVSwitch multicast object."""
        arr = (C.c_void_p * self.n)(*[r.h for r in self.replicas])
        _ck(lib().apus_group_multicast(arr, self.n), "apus_group_multicast")

    def prologue(self):
        """Blank CONFIG entry the election winner appends (dare_server.c:1412-1421);
        none when the group has a single member (dare_server.c:416-424)."""
        if self.n == 1:
            return 0
        self.tickets = self.leader.submit(CONFIG, 0, 0, cid_image(self.n))
        return self.tickets

    def submit(self, typ, conn, req_id, payload=b""):
        self.tickets = self.leader.submit(typ, conn, req_id, payload)
        return self.tickets

    def submit_stream(self, stream):
        """stream: iterable of (type, connection_id, req_id, payload) -- tailq_entry_t fields."""
        self.leader.defer(True)
        try:
            for typ, conn, rid, payload in stream:
                self.tickets = self.leader.submit(typ, conn, rid, payload)
        finally:
            self.leader.flush()
            self.leader.defer(False)
        return self.tickets

    def submit_uniform(self, n_req, length, conn, first_req_id, payloads=None, typ=SEND):
        """n_req requests of `length` bytes on one connection (batch ABI call)."""
        types = np.full(n_req, typ, dtype=np.uint8)
        conns = np.full(n_req, conn, dtype=np.uint16)
        req_ids = np.arange(first_req_id, first_req_id + n_req, dtype=np.uint64)
        lens = np.full(n_req, length, dtype=np.uint16)
        t0 = self.leader.submit_batch(types, conns, req_ids, lens, payloads, length)
        self.tickets = t0 + n_req - 1
        return self.tickets

    def submit_device(self, types, conns, req_ids, lens, payloads, stream=None):
        """Replica.submit_device on the leader; keeps `tickets` up to date so that run() covers the batch."""
        n = payloads.shape[0]
        t0 = self.leader.submit_device(types, conns, req_ids, lens, payloads, stream)
        if n:
            self.tickets = t0 + n - 1
        return t0

    def submit_device_packed(self, types, conns, req_ids, offsets, values, stream=None):
        """Replica.submit_device_packed on the leader; keeps `tickets` up to date so that run() covers the batch."""
        n = types.shape[0]
        t0 = self.leader.submit_device_packed(types, conns, req_ids, offsets, values, stream)
        if n:
            self.tickets = t0 + n - 1
        return t0

    def run(self, timeout_ms=60_000):
        """Launch for everything submitted so far and wait until it is committed everywhere."""
        self.launch()
        self.wait(timeout_ms)
