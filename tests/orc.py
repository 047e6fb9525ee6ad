"""ctypes bindings for the CPU oracle (TEST INFRASTRUCTURE ONLY).

Two libraries share one flat API (see oracle/oracle_port.c, oracle/ref_harness.c):
  prefix "orc": oracle/liboracle_port.so  -- the restatement of dare_log.h
  prefix "ref": oracle/_ref/libapus_ref.so -- the reference's own dare_log.h, compiled
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
PORT_SO = os.path.join(ORACLE_DIR, "liboracle_port.so")
REF_SO = os.path.join(ORACLE_DIR, "_ref", "libapus_ref.so")

NOOP, CSM, CONFIG, HEAD, CONNECT, SEND, CLOSE = 0, 1, 2, 3, 4, 5, 6
RULES_REFERENCE, RULES_ENGINE = 0, 1
LOG_SIZE = 16384 * 4096
HDR = 64

u64, u32, u16, u8 = C.c_uint64, C.c_uint32, C.c_uint16, C.c_uint8
vp = C.c_void_p


def build_oracle():
    """(Re)build the oracle libraries; the ref target is a no-op without /root/reference."""
    subprocess.run(["make", "-s", "-C", ORACLE_DIR, "port", "ref"], check=True,
                   stdout=subprocess.DEVNULL)


def have_ref():
    return os.path.exists(REF_SO)


def cmd_image(payload: bytes) -> bytes:
    """sm_cmd_t image {u16 len; u8 cmd[len]} (dare_sm.h:23-27)."""
    return len(payload).to_bytes(2, "little") + bytes(payload)


def cid_image(n: int) -> bytes:
    """dare_cid_t as init_server_data builds it (dare_server.c:285-291)."""
    return (0).to_bytes(8, "little") + bytes([n, 0, 0, 0]) + ((1 << n) - 1).to_bytes(4, "little")


def fnv1a(buf) -> int:
    h = 0xCBF29CE484222325
    for b in bytes(buf):
        h ^= b
        h = (h * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


class Oracle:
    """One of the two oracle libraries, addressed through its symbol prefix."""

    def __init__(self, prefix="orc"):
        self.prefix = prefix
        path = PORT_SO if prefix == "orc" else REF_SO
        if not os.path.exists(path):
            build_oracle()
        self.lib = C.CDLL(path)
        L = self.lib
        f = self._f
        f("log_create", vp, [u64])
        f("log_destroy", None, [vp])
        f("log_append", u64, [vp, u64, u64, u16, u8, vp])
        f("log_offsets", None, [vp, C.POINTER(u64)])
        f("log_set_offsets", None, [vp, C.POINTER(u64)])
        f("log_entries", C.POINTER(u8), [vp])
        f("log_end_distance", u64, [vp, u64])
        f("log_is_offset_larger", C.c_int, [vp, u64, u64])
        f("log_get_tail", u64, [vp])
        f("sizeof_entry", u32, [])
        f("cluster_new", vp, [C.c_int, C.c_int, u64, u64])
        f("cluster_free", None, [vp])
        f("submit", u64, [vp, u8, u16, u64, vp])
        f("prologue", u64, [vp])
        f("leader_persist", None, [vp])
        f("replicate", None, [vp, C.c_int])
        f("follower_persist", None, [vp, C.c_int])
        f("commit_scan", C.c_int, [vp])
        f("push_commit", None, [vp, C.c_int])
        f("apply", None, [vp, C.c_int])
        f("poll_head", None, [vp, C.c_int, C.POINTER(u64)])
        f("prune", u64, [vp])
        # newer than the rest of the API: a library built by an older recipe (a prebuilt oracle/_ref kept where the
        # reference tree is absent) lacks it, and everything else in it still works
        f("prune_to", u64, [vp, u64], optional=True)
        f("round", None, [vp])
        f("cluster_offsets", None, [vp, C.c_int, C.POINTER(u64)])
        f("cluster_entries", C.POINTER(u8), [vp, C.c_int])
        f("applied_count", u64, [vp, C.c_int])
        f("applied_get", None, [vp, C.c_int, u64, C.POINTER(u64)])
        f("store_cmd_calls", u64, [vp, C.c_int])
        f("update_state_calls", u64, [vp])
        f("bytes_replicated", u64, [vp])
        f("remote_end", u64, [vp, C.c_int])
        f("bench_run", C.c_double, [C.c_int, C.c_int, u64, C.c_int, C.POINTER(C.c_double)])
        if prefix == "orc":
            L.orc_set_rules.argtypes = [C.c_int]
            L.orc_set_rules.restype = None

    def _f(self, name, restype, argtypes, optional=False):
        sym = f"{self.prefix}_{name}"
        if optional and not hasattr(self.lib, sym):
            def missing(*_):
                raise AttributeError(f"{self.lib._name} has no {sym}: it was built from an older oracle/cluster_sim.inc "
                                     "(make -C oracle port ref)")
            setattr(self, name, missing)
            return
        fn = getattr(self.lib, sym)
        fn.restype = restype
        fn.argtypes = argtypes
        setattr(self, name, fn)

    def set_rules(self, rules):
        if self.prefix != "orc":
            assert rules == RULES_REFERENCE, "the compiled reference has only its own rules"
            return
        self.lib.orc_set_rules(rules)


class Log:
    """A single log (restates / wraps dare_log_t)."""

    def __init__(self, oracle: Oracle, length=LOG_SIZE):
        self.o = oracle
        self.h = oracle.log_create(length)
        self.len = length

    def close(self):
        if self.h:
            self.o.log_destroy(self.h)
            self.h = None

    def append(self, term, req_id, clt_id, typ, data=b""):
        buf = C.create_string_buffer(bytes(data) + b"\0" * 16)
        return self.o.log_append(self.h, term, req_id, clt_id, typ, C.cast(buf, vp))

    def offsets(self):
        out = (u64 * 8)()
        self.o.log_offsets(self.h, out)
        k = ["head", "apply", "commit", "end", "tail", "old_end", "old_commit", "len"]
        return dict(zip(k, [int(x) for x in out]))

    def set_offsets(self, **kw):
        cur = self.offsets()
        cur.update(kw)
        arr = (u64 * 8)(*[cur[k] for k in
                          ["head", "apply", "commit", "end", "tail", "old_end", "old_commit", "len"]])
        self.o.log_set_offsets(self.h, arr)

    def image(self, start=0, stop=None):
        stop = self.len if stop is None else stop
        p = self.o.log_entries(self.h)
        return np.ctypeslib.as_array(p, shape=(self.len,))[start:stop].copy()

    def poke(self, off, data: bytes):
        p = self.o.log_entries(self.h)
        arr = np.ctypeslib.as_array(p, shape=(self.len,))
        arr[off:off + len(data)] = np.frombuffer(data, dtype=np.uint8)


class Cluster:
    """N logs + the restated replicate / ack / commit / apply steps."""

    def __init__(self, oracle: Oracle, n, leader=0, term=1, length=LOG_SIZE):
        self.o, self.n, self.leader, self.len = oracle, n, leader, length
        self.h = oracle.cluster_new(n, leader, term, length)
        assert self.h

    def close(self):
        if self.h:
            self.o.cluster_free(self.h)
            self.h = None

    def submit(self, typ, clt_id, req_id, data=b"\0\0"):
        buf = C.create_string_buffer(bytes(data) + b"\0" * 16)
        return self.o.submit(self.h, typ, clt_id, req_id, C.cast(buf, vp))

    def prologue(self):
        return self.o.prologue(self.h)

    def prune_to(self, head):
        """SIM(prune_to): head := `head` and append <HEAD, head>, without the pruning rule's checks (the replay of a
        run whose HEAD entries the engine decided, tests/autoprune_replay.py).  Returns the HEAD idx, 0 when full."""
        return self.o.prune_to(self.h, head)

    def round(self, live=None):
        """One round of SIM(round) (oracle/cluster_sim.inc).  With `live` (follower indices), only those followers
        are up: they receive, ack, get the commit offset pushed and apply; the others keep their state.  The steps run
        in SIM(round)'s order, the commit scan once."""
        if live is None:
            self.o.round(self.h)
            return
        up = [i for i in range(self.n) if i == self.leader or i in set(live)]
        self.leader_persist()
        for i in up:
            self.replicate(i)
        for i in up:
            self.follower_persist(i)
        self.commit_scan()
        for i in up:
            self.push_commit(i)
        for i in up:
            self.apply(i)

    def offsets(self, i):
        out = (u64 * 8)()
        self.o.cluster_offsets(self.h, i, out)
        k = ["head", "apply", "commit", "end", "tail", "old_end", "old_commit", "len"]
        return dict(zip(k, [int(x) for x in out]))

    def image(self, i, start=0, stop=None):
        stop = self.len if stop is None else stop
        p = self.o.cluster_entries(self.h, i)
        return np.ctypeslib.as_array(p, shape=(self.len,))[start:stop].copy()

    def applied(self, i):
        n = self.o.applied_count(self.h, i)
        out = (u64 * 5)()
        res = []
        for k in range(n):
            self.o.applied_get(self.h, i, k, out)
            res.append(tuple(int(x) for x in out))
        return res

    def __getattr__(self, name):
        # leader_persist, replicate, follower_persist, commit_scan, push_commit, apply, prune ...
        fn = getattr(self.o, name)
        return lambda *a: fn(self.h, *a)


def walk_entries(img: np.ndarray, start: int, end: int, length: int):
    """Walk entry boundaries [start,end) the way every reference loop does
    (log_get_entry + log_fit_entry + log_entry_len).  Returns [(offset, stride)].
    `end` may be < start (wrapped).  Ghost headers are skipped like the reference."""
    out = []
    off = start
    guard = 0
    while off != end:
        guard += 1
        assert guard < 10_000_000
        if length - off < HDR:
            off = 0
            if off == end:
                break
        typ = int(img[off + 26])
        stride = HDR if typ in (NOOP, CONFIG, HEAD) else HDR + int(img[off + 48]) + 256 * int(img[off + 49])
        if length - off < stride:
            off = 0
            continue
        out.append((off, stride))
        off += stride
        if off == length and end == 0:
            break
    return out


def mask_replies(img: np.ndarray, entries):
    """Zero reply[0..12] of every entry (the H5 mask of SURVEY.md s8c)."""
    img = img.copy()
    for off, _ in entries:
        img[off + 28: off + 41] = 0
    return img
