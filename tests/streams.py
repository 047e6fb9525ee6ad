"""Deterministic synthetic request streams shared by the oracle tests, the golden
generator and the GPU parity tests (SURVEY.md s8d "Synthetic inputs").

A request is (type, connection_id, req_id, payload) -- exactly the fields of the
reference's tailq_entry_t (src/include/dare/message.h:11-17); numbering follows
proxy.c:114-156: connection_id = (leader_idx << 8) | c, req_id counts per
connection from 1 (the CONNECT itself is req_id 1).
"""
import numpy as np

CONNECT, SEND, CLOSE = 4, 5, 6
MASK = (1 << 64) - 1


def xorshift64s_bytes(seed: int, n: int) -> np.ndarray:
    """n pseudo-random bytes from xorshift64* (vectorised over independent lanes
    would change the sequence, so this is the scalar generator, run on 8-byte words)."""
    words = (n + 7) // 8
    out = np.empty(words, dtype=np.uint64)
    x = seed & MASK or 0x9E3779B97F4A7C15
    for i in range(words):
        x ^= x >> 12
        x ^= (x << 25) & MASK
        x ^= x >> 27
        out[i] = (x * 0x2545F4914F6CDD1D) & MASK
    return out.view(np.uint8)[:n]


def payload_kat(i: int, length: int) -> bytes:
    """payload byte k of request i = (i*31 + k) & 0xFF (the vector quoted in SURVEY.md s8c)."""
    return bytes(((i * 31 + k) & 0xFF) for k in range(length))


def uniform_stream(n_req: int, length: int, conns: int = 1, leader: int = 0, seed=None):
    """One CONNECT per connection, then n_req SENDs of `length` bytes round-robin."""
    seed = (0xA5A50000 + length) if seed is None else seed
    rng = np.random.default_rng(seed)
    req_id = [0] * conns
    out = []
    for c in range(conns):
        req_id[c] += 1
        out.append((CONNECT, (leader << 8) | c, req_id[c], b""))
    blob = rng.integers(0, 256, size=n_req * length, dtype=np.uint8).tobytes() if length else b""
    for i in range(n_req):
        c = i % conns
        req_id[c] += 1
        out.append((SEND, (leader << 8) | c, req_id[c], blob[i * length:(i + 1) * length]))
    return out


def ragged_stream(n_req: int, max_len: int, conns: int = 3, leader: int = 0, seed: int = 1234,
                  close_every: int = 0):
    """SENDs with lengths drawn from [0, max_len] (0-length and odd lengths included),
    optional CLOSE + re-CONNECT churn."""
    rng = np.random.default_rng(seed)
    req_id = {}
    out = []
    live = []
    next_conn = 0

    def connect():
        nonlocal next_conn
        cid = (leader << 8) | (next_conn & 0xFF)
        next_conn += 1
        req_id[cid] = 1
        out.append((CONNECT, cid, 1, b""))
        live.append(cid)

    for _ in range(conns):
        connect()
    for i in range(n_req):
        cid = live[int(rng.integers(0, len(live)))]
        ln = int(rng.integers(0, max_len + 1))
        if rng.random() < 0.1:
            ln = int(rng.choice([0, 1, 13, 14, 15, 16, 17, 63, 64, 65, max_len]))
            ln = min(ln, max_len)
        req_id[cid] += 1
        out.append((SEND, cid, req_id[cid], rng.integers(0, 256, size=ln, dtype=np.uint8).tobytes()))
        if close_every and (i + 1) % close_every == 0 and len(live) > 1:
            victim = live.pop(0)
            req_id[victim] += 1
            out.append((CLOSE, victim, req_id[victim], b""))
            connect()
    return out


def stream_bytes(stream):
    """Log bytes the stream occupies (64 + len per request), ignoring wrap waste."""
    return sum(64 + len(p) for _, _, _, p in stream)


def sized_stream(n_req: int, lo: int, hi: int, conn: int = 0, seed: int = 1234):
    """One CONNECT, then n_req SENDs with lengths drawn from [lo, hi]."""
    rng = np.random.default_rng(seed)
    out = [(CONNECT, conn, 1, b"")]
    for i in range(n_req):
        ln = int(rng.integers(lo, hi + 1))
        out.append((SEND, conn, 2 + i, rng.integers(0, 256, size=ln, dtype=np.uint8).tobytes()))
    return out
