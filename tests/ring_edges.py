"""Plans that bring the leader's end to an exact byte of its ring, and the edge cases run there (TEST INFRASTRUCTURE
ONLY).  Used by tests/test_ring_edges_plan.py on the oracle alone and by tests/test_gpu_ring_edges.py on the engine.

The decisions at the ring's end are byte-exact comparisons: whether the next entry fits before `len` (and ends exactly
there, rule E1), whether its header fits (a ghost header stays behind) or not (the stretch is skipped), whether rule E2
lets it wrap, and whether the pruning rule is due.  A random stream meets each of them only by chance.  Here a filler
request of stride 64 + len (len 0..65535) moves the end by any amount from 64 to 65599 bytes, one or two of them reach
any offset, and the edge request is placed exactly where its case says.

Two kinds of plan:
  Tour      -- lockstep with the oracle, no device-side pruning: the host prunes at quiescent points (SIM(prune), a
               HEAD entry submitted with the head), every edge preceded by a lap so its stretch holds stale bytes.
               The plan is a list of steps the GPU test replays on the engine and on a fresh oracle.
  scenario  -- APUS_F_AUTOPRUNE: the leader prunes on its own, by the apply offsets the followers report.  One request
               per claim, so the rule is evaluated before every entry, as in the reference.  The script reads the state
               back from its driver: `AutoModel` (the oracle plus the engine's rule, here) or the GPU test's driver (the
               engine, replayed into the oracle by autoprune_replay.Replay).
"""
from dataclasses import dataclass, field

import numpy as np

import autoprune_replay as AR
import orc as O
import streams as S

HDR = O.HDR
MAXLEN = 65535
MAX_STRIDE = HDR + MAXLEN


def u64(img, off):
    return int.from_bytes(img[off:off + 8].tobytes(), "little")


def landing(L, end, stride, has_cmd):
    """where log_append_entry puts an entry of `stride` bytes appended at `end`, by the engine's rules: (offset, ghost)"""
    pos0 = 0 if end == L else end
    left = L - pos0
    if stride <= left:
        return pos0, False
    return 0, left >= HDR and has_cmd


def klass(L, end, stride, has_cmd):
    """the edge an append meets: "at0" (the end is 0 after an exact fit), "fit", "e1" (ends exactly at len), "ghost"
    (wraps, header left behind) or "skip" (wraps, not even the header fits)"""
    if end == 0:
        return "at0"
    at, ghost = landing(L, end, stride, has_cmd)
    if at == end:
        return "e1" if at + stride == L else "fit"
    return "ghost" if ghost else "skip"


def fill_to(d, target, step, between=None):
    """Append fillers through `d` (`d.end()`, `d.send(stride)`) until the end is exactly `target` (0 < target <= L; L:
    the last filler ends exactly at len, so the end is 0).  At most `step` bytes per piece; `between()` is called
    between pieces (the tour prunes there).  Goes round the ring when the target is behind the end or less than one
    header ahead of it."""
    L = d.L
    goal = target % L
    for _ in range(64):
        e = d.end()
        if e == goal and (goal != 0 or d.last_ended_at_len()):
            return
        to = target if target > e else L                      # behind the end: first to the ring's end
        rem = to - e
        if rem < HDR:
            if to == L:                                       # the header does not fit: the filler goes to 0
                d.send(HDR)
            else:                                             # too close ahead: go round
                fill_to(d, L, step, between)
            if between:
                between()
            continue
        chunk = min(rem, step)
        if 0 < rem - chunk < HDR:
            chunk = rem - HDR if rem - HDR >= HDR else rem
        while chunk:
            s = min(chunk, MAX_STRIDE)
            if 0 < chunk - s < HDR:
                s = chunk - HDR
            d.send(s)
            chunk -= s
        if d.end() != goal and between:
            between()
    raise AssertionError(f"fill_to({target}) did not converge, end {d.end()}")


# ---- A: wrap geometry, lockstep with the oracle, the host prunes ---------------------------------------------------
@dataclass
class Edge:
    """one edge request at `left` bytes before len (0: the entry before ended exactly at len, rule E1) and what it is
    expected to meet (`expect`, see klass).  The rest is what the oracle computed."""
    kind: str           # empty | send | max | connect | head
    left: int
    pos: str            # first | middle | last: the edge entry's place in its launch
    expect: str
    stride: int = 0
    end_before: int = -1
    at: int = -1
    ghost: bool = False
    end: int = -1
    idx: int = 0
    refusal: str = None     # autoprune_replay.placement_refusal: why the leader would not block (None: it blocks)
    stale: int = 0          # non-zero stale bytes in the skipped stretch (or the ghost's) before the append


SEND_LEN = 777              # the stride of the 'send' edge entry is 841


def edge_stride(kind):
    return {"empty": HDR, "connect": HDR, "head": HDR, "send": HDR + SEND_LEN, "max": MAX_STRIDE}[kind]


def _expect(kind, left):
    s = edge_stride(kind)
    if left == 0:
        return "at0"
    if s < left:
        return "fit"
    if s == left:
        return "e1"
    return "ghost" if left >= HDR and kind not in ("head",) else "skip"


def tour_edges(big=False):
    """the edges of one tour: `big` the maximal cmd on a ring that holds it, else the rest"""
    if big:
        cases = [("max", lf) for lf in (0, 1, 63, 64, 65, MAX_STRIDE - 1, MAX_STRIDE, MAX_STRIDE + 1)]
    else:
        cases = [(k, lf) for k in ("empty", "send", "connect", "head") for lf in (0, 1, 15, 16, 17, 63, 64, 65)]
        cases += [("send", edge_stride("send") + dl) for dl in (-1, 0, 1)]
    out = []
    for i, (k, lf) in enumerate(cases):
        pos = "first" if k == "head" else ("first", "middle", "last")[i % 3]
        out.append(Edge(k, lf, pos, _expect(k, lf)))
    return out


# the tours the tests run: (replicas, ring bytes, seed, the maximal cmd tour)
TOURS = {"small": (3, 1 << 14, 0xE0, False), "small-n5": (5, 1 << 14, 0xE2, False), "max": (3, 1 << 18, 0xE1, True)}


def make_tour(orc, name):
    n, L, seed, big = TOURS[name]
    return Tour(orc, n, L, seed, tour_edges(big))


class Tour:
    """The lockstep plan of one ring: `steps` to replay on the engine and a fresh oracle, ("req", request), ("run",)
    (a launch, then two oracle rounds), ("prune",) (SIM(prune) and the same HEAD submitted to the engine) and
    ("check", k) (compare every replica with the oracle, and edge k's geometry)."""

    def __init__(self, orc, n, L, seed, edges):
        orc.set_rules(O.RULES_ENGINE)
        self.n, self.L = n, L
        self.c = O.Cluster(orc, n, leader=0, term=1, length=L)
        self.c.prologue()
        self.rng = np.random.default_rng(seed)
        self.rid = 1
        self.steps = [("config",)]
        self.edges = []
        self.step = L // 4
        self.req((S.CONNECT, 0, 1, b""))
        # a lap and a half of ragged requests first: every stretch an edge meets holds an earlier lap's bytes
        n_lap = 0
        while n_lap < 1.5 * L:
            ln = int(self.rng.integers(0, 400))
            self.send(HDR + ln)
            n_lap += HDR + ln
            if n_lap % self.step < HDR + 400:
                self.prune()
        for e in edges:
            self.edge(e)
        self.run()

    def close(self):
        self.c.close()

    def end(self):
        return self.c.offsets(0)["end"]

    def last_ended_at_len(self):
        o = self.c.offsets(0)
        return o["end"] == 0

    def req(self, r):
        typ, clt, rid, payload = r
        idx = self.c.submit(typ, clt, rid, O.cmd_image(payload))
        assert idx, f"the oracle refused {r[:3]} at end {self.end()} (ring full)"
        self.steps.append(("req", r))
        return idx

    def send(self, stride):
        self.rid += 1
        payload = self.rng.integers(1, 256, stride - HDR, dtype=np.uint8).tobytes()
        return self.req((S.SEND, 0, self.rid, payload))

    def run(self):
        if self.steps[-1] != ("run",):
            self.c.round(); self.c.round()
            self.steps.append(("run",))

    def prune(self):
        self.run()
        if self.c.prune():
            self.steps.append(("prune",))
            self.run()

    def edge(self, e):
        L = self.L
        e.stride = edge_stride(e.kind)
        self.prune()
        fill_to(self, L - e.left, self.step, self.prune)
        if e.pos == "first":
            self.run()
        o = self.c.offsets(0)
        e.end_before = o["end"]
        img = self.c.image(0)
        if e.end_before:
            e.stale = int(np.count_nonzero(img[e.end_before:]))
        e.refusal = AR.placement_refusal(L, o["head"], o["end"], e.stride)
        if e.kind == "head":
            e.idx = self.c.prune()
            assert e.idx, "SIM(prune) did not prune before the edge"
            self.steps.append(("prune",))
        elif e.kind == "connect":
            self.rid += 1
            e.idx = self.req((S.CONNECT, 0x40 + len(self.edges), 1, b""))
        else:
            self.rid += 1
            e.idx = self.req((S.SEND, 0, self.rid, self.rng.integers(1, 256, e.stride - HDR, dtype=np.uint8).tobytes()))
        o = self.c.offsets(0)
        e.at, e.end = o["tail"], o["end"]
        img = self.c.image(0)
        e.ghost = e.at != e.end_before and L - e.end_before >= 8 and u64(img, e.end_before) == e.idx
        if e.pos in ("first", "middle"):
            self.send(HDR + 33)
        self.run()
        self.steps.append(("check", len(self.edges)))
        self.edges.append(e)


# ---- C: the pruning rule at the ring's end (APUS_F_AUTOPRUNE) --------------------------------------------------------
def auto_head(L, head, end, tail, prev_head, applies):
    """the pruning rule as leader_place evaluates it before an entry appended at `end` (never between a wrap's gap and
    its entry): the head a HEAD entry placed there carries, or None"""
    if end == L or prev_head or L - end < HDR:
        return None
    used = AR.dist(head, end, L)
    if used < L // 4:
        return None
    d = max(min(AR.dist(a, end, L), used) for a in applies)
    if d == 0:
        d = AR.dist(tail, end, L)
    if d <= used and used - d >= L // 8:
        return (end - d) % L
    return None


INLINE_BYTES = 80            # APUS_SLOT_INLINE: a cmd image (2 + len bytes) up to this size travels in its slot


def express_takes(L, head, end, req):
    """whether the leader's express path (one request in flight, resident kernels) places `req` at `end` itself: an
    inline cmd that fits before len and before the head (rule E2 with the HEAD reserve), while the ring is under half
    used.  It never evaluates the pruning rule; from half used on it hands every request to the tile machine."""
    pos0 = 0 if end == L else end
    used = 0 if end == L else AR.dist(head, end, L)
    stride = AR.request_stride(req)
    return (req[0] not in (O.NOOP, O.CONFIG, O.HEAD) and 2 + len(req[3]) <= INLINE_BYTES and used < L // 2 and
            pos0 + stride <= L and used + stride + HDR < L)


class AutoModel:
    """The CPU stand-in for a leader that prunes on the device, with host-applying followers that report `pin` as
    applied: the oracle, plus auto_head before every request (one request per claim).  With `express`, a request the
    leader's express path takes (express_takes) is placed without the rule, as the express path does."""

    def __init__(self, orc, n, L, seed, express=False):
        orc.set_rules(O.RULES_ENGINE)
        self.n, self.L = n, L
        self.express = express
        self.c = O.Cluster(orc, n, leader=0, term=1, length=L)
        self.c.prologue()
        self.c.round(); self.c.round()
        self.rng = np.random.default_rng(seed)
        self.rid = 1
        self.pinned = 0
        self.prev_head = False
        self.heads = []                  # (offset, value) of every HEAD entry appended
        self.info = {}
        self.cid = [0] * n
        self.put((S.CONNECT, 0, 1, b""))

    def close(self):
        self.c.close()

    def offsets(self):
        return self.c.offsets(0)

    def end(self):
        return self.c.offsets(0)["end"]

    def last_ended_at_len(self):
        return self.end() == 0

    def image(self):
        return self.c.image(0)

    def pin(self, v):
        self.pinned = v

    def put(self, r):
        c, L = self.c, self.L
        o = c.offsets(0)
        stride = AR.request_stride(r)
        v = auto_head(L, o["head"], o["end"], o["tail"], self.prev_head, [o["end"]] + [self.pinned] * (self.n - 1))
        if self.express and express_takes(L, o["head"], o["end"], r):
            v = None
        if v is not None:
            assert c.prune_to(v)
            self.heads.append((c.offsets(0)["tail"], v))
            self.prev_head = True
            c.round(); c.round()
            AR.poll_heads(c, self.cid)
            o = c.offsets(0)
        assert AR.placement_refusal(L, o["head"], o["end"], stride), f"the placement of {stride} B at {o['end']} blocks"
        typ, clt, rid, payload = r
        assert c.submit(typ, clt, rid, O.cmd_image(payload))
        self.prev_head = False
        c.round(); c.round()
        AR.poll_heads(c, self.cid)

    def send(self, stride):
        self.rid += 1
        self.put((S.SEND, 0, self.rid, self.rng.integers(1, 256, stride - HDR, dtype=np.uint8).tobytes()))

    def put_held(self, r, release):
        """`r` must not be placeable (rule E2) until the followers report `release` as applied; then it is"""
        o = self.c.offsets(0)
        why = AR.placement_refusal(self.L, o["head"], o["end"], AR.request_stride(r))
        assert why is None, f"the placement was expected to hold: {why}"
        self.pin(release)
        self.put(r)

    def request(self, stride):
        self.rid += 1
        return (S.SEND, 0, self.rid, self.rng.integers(1, 256, stride - HDR, dtype=np.uint8).tobytes())


@dataclass
class AutoCase:
    """At `end` = L - `left`, `used` bytes in use, the followers having applied up to `adv` bytes past the head: append
    an entry of `stride` bytes, then one more.  `expect`: the layout the rule and the wrap rules give, as
    (HEAD at the end, what the entry meets (klass, after that HEAD), HEAD right behind the entry)."""
    name: str
    left: int
    used: int
    adv: int
    stride: int
    expect: tuple
    got: tuple = None
    info: dict = field(default_factory=dict)


def auto_cases(L):
    q, e = L // 4, L // 8
    return [
        # C1: not due at the end; due at 0 if the skipped stretch counted.  Ghost, then the entry at 0, no HEAD
        # between them; the HEAD comes behind the entry, where the rule is evaluated next
        AutoCase("c1-ghost", 1000, q - 16, e + 512, 1500, (False, "ghost", True)),
        AutoCase("c1-skip", 40, q - 16, e + 512, 1500, (False, "skip", True)),
        # C2: due at the end, with exactly one header left: the HEAD ends at len (E1), the entry goes to 0, no gap
        AutoCase("c2-head-e1", 64, q + 256, e + 512, 1500, (True, "at0", False)),
        # C3: due at the end, then the entry wraps behind the HEAD: HEAD, ghost (or skip), entry at 0
        AutoCase("c3-head-ghost", 300, q + 256, e + 512, 1500, (True, "ghost", False)),
        AutoCase("c3-head-skip", 100, q + 256, e + 512, 1500, (True, "skip", False)),
        # C4: the thresholds, away from the ring's end
        AutoCase("c4-used-below", L // 3, q - 1, e + 512, 200, (False, "fit", True)),
        AutoCase("c4-used-at", L // 3, q, e + 512, 200, (True, "fit", False)),
        AutoCase("c4-adv-below", L // 3, q + 256, e - 1, 200, (False, "fit", False)),
        AutoCase("c4-adv-at", L // 3, q + 256, e, 200, (True, "fit", False)),
    ]


TRIGGER = HDR + 100         # the request behind which a HEAD is expected: its image is external, the express path never
                            # takes it


def _lap(d, nbytes):
    """fillers of 64 B to a sixteenth of the ring, the followers reporting the end before each as applied (the head
    follows them): the ring's every stretch ends up holding non-zero bytes"""
    done = 0
    while done < nbytes:
        d.pin(d.end())
        s = HDR + int(d.rng.integers(0, d.L // 16))
        d.send(s)
        done += s


def _hop(d, jitter):
    """move the head by one HEAD entry: hold the followers' reports at the head, append an eighth of the ring and
    `jitter` bytes past it, mark that boundary, append past a quarter, then report the mark as applied"""
    L = d.L
    h = d.offsets()["head"]
    d.pin(h)
    while AR.dist(h, d.end(), L) < L // 8 + jitter:
        d.send(HDR + min(L // 16, L // 8 + jitter - AR.dist(h, d.end(), L)))
    x = d.end()
    d.send(2 * HDR)                                            # the end past the mark: the HEAD carries it, not the tail
    while AR.dist(h, d.end(), L) < L // 4:
        d.send(L // 16)
    d.pin(x)
    d.send(TRIGGER)
    assert d.offsets()["head"] == x, (d.offsets(), x)
    d.pin(x)


def prepare(d, E, used, adv):
    """After a lapped ring: the head at H = E - `used`, a boundary at P = H + `adv`, the end at E, the followers
    reporting H (so nothing is due).  Returns P."""
    L = d.L
    H = (E - used) % L
    _lap(d, int(2.3 * L))
    d.pin(d.end())
    fill_to(d, L, L // 8)                                      # a filler's data up to the slack before len
    # hop the head until H is about a quarter to half a ring ahead of it, with the end still before H
    for _ in range(40):
        o = d.offsets()
        h, e = o["head"], o["end"]
        ah, ae = AR.dist(h, H, L), AR.dist(h, e, L)
        if L // 4 - 1024 <= ah <= L // 2 and ae + HDR <= ah:
            break
        _hop(d, int(d.rng.integers(0, L // 8)))
    else:
        raise AssertionError(f"the head never reached a place to move to {H} from: {d.offsets()}")
    d.pin(d.offsets()["head"])                                 # nothing due while filling
    fill_to(d, H, L // 8)
    d.send(2 * HDR)                                            # the end past H: a HEAD there carries H, not the tail
    while AR.dist(d.offsets()["head"], d.end(), L) < L // 4:
        d.send(L // 32 + HDR)
    assert AR.dist(H, d.end(), L) + HDR + TRIGGER + HDR <= adv, (d.offsets(), H, adv)
    d.pin(H)
    d.send(TRIGGER)                                            # HEAD(H), then this filler
    assert d.offsets()["head"] == H, (d.offsets(), H)
    d.pin(H)
    P = (H + adv) % L
    fill_to(d, P, L // 8)
    fill_to(d, E, L // 8)
    o = d.offsets()
    assert o["end"] == E % L and AR.dist(o["head"], o["end"], L) == used, (o, E, used)
    img = d.image()
    d.info.update(stale=int(np.count_nonzero(img[E:])) if E % L else 0, end_before=E % L)
    return P


def scenario(d, case):
    """run `case` through the driver `d`; sets case.got and case.info"""
    L = d.L
    E = L - case.left
    P = prepare(d, E, case.used, case.adv)
    d.pin(P)
    n_heads = len(d.heads)
    d.send(case.stride)
    o = d.offsets()
    head_at_end = len(d.heads) > n_heads and d.heads[-1][0] == E
    at = o["tail"]
    img = d.image()
    e_at = E + HDR if head_at_end else E
    if head_at_end and e_at == L:
        k = "at0"
    else:
        k = "fit" if at == e_at else ("ghost" if u64(img, e_at) == u64(img, at) and L - e_at >= 8 else "skip")
    n_heads = len(d.heads)
    d.info.update(at=at, idx=u64(img, at))
    d.send(TRIGGER)
    after = len(d.heads) > n_heads and d.heads[-1][0] == (at + case.stride) % L
    case.got = (head_at_end, k, after)
    case.info = d.info


# ---- B: rule E2 to the byte, with the HEAD reserve of device-side pruning --------------------------------------------
@dataclass
class E2Case:
    """An entry of `stride` bytes at `left` bytes before len, with the ring used so that used + stride + 64 (in place)
    or used + left + stride + 64 (wrapped) is L - 1 + `extra`: 0 places, 1 holds until the followers report more."""
    name: str
    left: int
    stride: int
    extra: int
    held: bool = None
    info: dict = field(default_factory=dict)


def e2_cases(L):
    return [E2Case("in-place", L // 3, 1000, 0), E2Case("in-place+1", L // 3, 1000, 1),
            E2Case("wrapped", 500, 1000, 0), E2Case("wrapped+1", 500, 1000, 1)]


def e2_scenario(d, case):
    """the placement and (extra 1) the hold and its release by a HEAD entry at the end; sets case.held, case.info"""
    L = d.L
    E = L - case.left
    wrap = case.stride > case.left
    used = L - 1 - HDR - case.stride - (case.left if wrap else 0) + case.extra
    P = prepare(d, E, used, L // 8 + 512)
    r = d.request(case.stride)
    n_heads = len(d.heads)
    case.held = case.extra > 0
    if case.held:
        d.put_held(r, P)                                       # HEAD(P) at E, then the entry
        assert d.heads[n_heads:] == [(E, P)], (d.heads[n_heads:], E, P)
    else:
        d.put(r)
        assert len(d.heads) == n_heads, d.heads[n_heads:]
    case.info = dict(d.info, at=d.offsets()["tail"], end=d.end())


# ---- C5 and the express path's hand-over -----------------------------------------------------------------------------
def c5_scenario(d):
    """right after a wrap every replica has applied up to the end (d == 0): the next HEAD carries the tail, the wrapped
    entry at 0.  Returns (the HEAD's offset, the head it carries, the wrapped entry's offset)."""
    L = d.L
    prepare(d, L - 1000, L // 4 - 16, L // 8 + 512)
    d.send(1500)                                               # ghost at L - 1000, the entry at 0
    at = d.offsets()["tail"]
    d.pin(d.end())
    n_heads = len(d.heads)
    d.send(TRIGGER)
    assert len(d.heads) == n_heads + 1, d.heads[n_heads:]
    off, v = d.heads[-1]
    return off, v, at


def express_scenario(d, used):
    """the rule due (a quarter used, the followers an eighth past the head) with the ring `used` bytes full: an inline
    request the express path takes below half used goes in without a HEAD; at half used it is handed to the tile
    machine, which puts the HEAD first.  Returns whether a HEAD was put before it."""
    L = d.L
    P = prepare(d, L // 2 + 2048, used, L // 8 + 512)
    d.pin(P)
    n_heads = len(d.heads)
    d.send(HDR + 40)
    return len(d.heads) > n_heads
