"""Replay of device-side log pruning (APUS_F_AUTOPRUNE) into the CPU oracle (TEST INFRASTRUCTURE ONLY).

Where the leader puts an auto HEAD entry, and which head it carries, depends on how far the followers had applied when
the place turn was taken, so the oracle cannot predict it.  The layout depends only on the sequence of appends,
though: the wrap, ghost and E1 rules look at `end` and `len`, not at `head`, and rule E2 only decides whether the
leader blocks.  So the engine's own sequence is read back after every launch that stays under one lap, and the oracle
appends the same sequence: the submitted requests in order, and <HEAD, v> (SIM(prune_to)) wherever the engine put a
HEAD entry carrying v.  Every replayed HEAD is first checked against the engine's pruning rule (`head_violation`),
so the replay cannot launder an arbitrary head.  At the end every byte of every replica is compared with the oracle.

Inside one launch that laps the ring many times the leader overwrites its entries long before the launch ends.
Followers whose host applies the log (APUS_F_HOST_APPLY) see all of them, though: a `Recorder` reads every committed
range before it reports it as applied, and the leader may not overwrite what a follower has not reported.
`replay_recordings` cuts the recorded sequence at every offset any follower read up to, replays the pieces, and
compares every recorded read with the oracle as it was at that point.  Positions in a recording are absolute: ring
bytes appended since the start, counting the stretch skipped at a wrap, like `Replay.written`.
"""
import ctypes as C
import threading
import time
from collections import defaultdict
from dataclasses import dataclass, field

import numpy as np

import orc as O


@dataclass
class Entry:
    """one entry as the leader wrote it: ring offset, stride and the header fields the replay checks"""
    off: int
    stride: int
    typ: int
    idx: int
    req_id: int
    clt_id: int
    value: int          # HEAD: the head it carries (bytes 48..55); else the data length (bytes 48..49)


def _u(img, off, n):
    return int.from_bytes(img[off:off + n].tobytes(), "little")


def parse_entries(img, start, end, L):
    """the entries of [start, end) of a full ring image `img`, in append order (ghost headers skipped)"""
    if start == end:
        return []
    out = []
    for off, stride in O.walk_entries(img, start, end, L):
        typ = int(img[off + 26])
        value = _u(img, off + 48, 8) if typ == O.HEAD else (0 if typ in (O.NOOP, O.CONFIG) else _u(img, off + 48, 2))
        out.append(Entry(off, stride, typ, _u(img, off, 8), _u(img, off + 16, 8), _u(img, off + 24, 2), value))
    return out


@dataclass
class Launch:
    """what one launch appended: the leader's bytes of [start, end) (`buf`, wrapped at the ring's end) and the
    entries parsed from them"""
    start: int
    end: int
    buf: np.ndarray
    entries: list


def launch_from_image(img, start, end, L):
    """the Launch of [start, end) on the leader's full ring image `img` (under one lap)"""
    buf = img[(start + np.arange((end - start) % L)) % L]
    return Launch(start, end, buf, parse_entries(img, start, end, L))


def read_launch(rep, start, end, L):
    """the Launch of [start, end) on the replica `rep`, through apus_log_read_range (safe while the kernels are
    resident); the range must be under one lap"""
    if start == end:
        return Launch(start, end, np.zeros(0, dtype=np.uint8), [])
    buf = rep.read_range(start, end, cap=L)
    assert len(buf) == (end - start) % L, (start, end, len(buf))
    img = np.zeros(L, dtype=np.uint8)
    img[(start + np.arange(len(buf))) % L] = buf
    return Launch(start, end, buf, parse_entries(img, start, end, L))


def dist(a, b, L):
    """bytes from offset a forward to offset b on a ring of L bytes"""
    return (b - a) % L


def request_stride(req):
    """ring bytes the entry of request `req` = (type, clt_id, req_id, payload) takes"""
    return O.HDR if req[0] in (O.NOOP, O.CONFIG, O.HEAD) else O.HDR + len(req[3])


def oracle_view(c, i):
    """replica i's ring of the oracle cluster `c`, without a copy (valid until the next step of the cluster)"""
    return np.ctypeslib.as_array(c.cluster_entries(i), shape=(c.len,))


def placement_refusal(L, head, end, stride):
    """Why the leader would not block placing an entry of `stride` bytes at `end` while the head is `head`, by its own
    arithmetic (leader_place without a HEAD in the sub-tile): it fits before the ring's end and strictly before the
    head with room kept for one HEAD entry (rule E2), or it does not fit before the ring's end but does after a wrap.
    None when the placement blocks.  (The tile's image and staging caps exceed any one entry, so they never decide.)"""
    pos0 = 0 if end == L else end
    used = 0 if end == L else dist(head, end, L)
    left = L - pos0
    if stride <= left and used + stride + 1 + O.HDR <= L:
        return f"the next entry (stride {stride}) would have fit at {pos0} (head {head}, {used} bytes used)"
    if stride > left and used + left + stride + O.HDR < L:
        return f"the next entry (stride {stride}) would have wrapped to 0 (head {head}, {used} bytes used, {left} left)"
    return None


def head_violation(L, head_old, end, v, boundaries, prev_was_head, next_stride=None, at=None):
    """The engine's pruning rule (leader_place) as a predicate over one HEAD entry appended at `end` while the head was
    `head_old`: None when a HEAD carrying `v` is legal there, else the reason.  `boundaries`: the starts and ends of
    the entries of [head_old, end).  `prev_was_head`: the entry just before is a HEAD.  The leader appends a second
    HEAD right behind one only when its placement blocked on space there: `next_stride`, the stride of the next
    non-HEAD entry of the sequence (None: there is none), must then not be placeable at the head and end the first
    HEAD left, which are `head_old` and `end`.  `at`: where the engine wrote the HEAD.  A HEAD is never placed
    anywhere but at `end`: the rule is not evaluated between a wrapping entry's ghost (or skipped stretch) and the
    entry, which the reference appends as one, nor where less than a header is left before len."""
    pos0 = 0 if end == L else end
    if at is not None and at != pos0:
        return (f"HEAD between a wrapping entry's ghost/skip and the entry: HEAD at {at}, the end was {end} "
                f"({L - pos0} bytes skipped)")
    if L - pos0 < O.HDR:
        return f"the HEAD's header does not fit at {end}: {L - pos0} bytes before len (the rule is not evaluated there)"
    used = 0 if end == L else dist(head_old, end, L)
    if used < L // 4:
        return f"ring used {used} < L/4 = {L // 4}"
    adv = dist(head_old, v, L)
    if adv > used:
        return f"head {v} is past the HEAD entry's own position {end} (head was {head_old})"
    if adv < L // 8:
        return f"head advances by {adv} < L/8 = {L // 8} ({head_old} -> {v})"
    if v not in boundaries:
        return f"head {v} is not an entry boundary of [{head_old}, {end})"
    if prev_was_head:
        if next_stride is None:
            return "two HEAD entries in a row with no entry behind them"
        why = placement_refusal(L, head_old, end, next_stride)
        if why is not None:
            return f"two HEAD entries in a row, but the placement was not blocked: {why}"
    return None


def live_boundaries(img, head, end, L):
    """entry starts and ends of [head, end) on the ring image `img` (E1: an end at L is offset 0)"""
    out = set()
    if head == end:
        return out
    for off, stride in O.walk_entries(img, head, end, L):
        out.add(off)
        out.add((off + stride) % L)
    return out


@dataclass
class ReplayedHead:
    off: int
    idx: int
    value: int
    lap_pos: int        # ring bytes appended before it, counting the stretches skipped at wraps


class Replay:
    """An oracle cluster fed with the engine's own append sequence, one launch at a time."""

    def __init__(self, orc, n, L, term=1):
        orc.set_rules(O.RULES_ENGINE)
        self.c = O.Cluster(orc, n, leader=0, term=term, length=L)
        self.n, self.L = n, L
        self.heads = []                     # ReplayedHead, in append order
        self.prev_head = False
        self.pairs = 0                      # HEAD entries appended right behind another one (blocked placements)
        self.written = 0                    # ring bytes appended so far (laps = written / L)
        self.last_start = 0                 # ring bytes appended before the last entry started (its absolute start)
        self.cid = [0] * n                  # poll_head's scan position per replica
        self.pos = 0                        # requests consumed

    def close(self):
        self.c.close()

    def end(self):
        return self.c.offsets(self.c.leader)["end"]

    def launch(self, lc, requests, replica=None, on_head=None, live=None):
        """Append what one launch appended (`lc`, read back from replica `replica`; `requests` the submitted stream, a
        CONFIG request standing for the prologue), run two quiescent rounds and poll_head on every follower, then
        compare the oracle's bytes of that replica in the launch's range with the ones read back: every entry the
        launch wrote, before a later lap overwrites it.  A follower's reply bytes are masked: nothing orders its own
        reply-byte stores before a host read of a committed range.  `on_head(entry, abs_start, prev_abs_start)`, called
        for every HEAD entry once appended, returns None or why that HEAD could not have been taken when it was.
        `replica` defaults to the leader; `live` (follower indices, default all) are the followers that ran: only they
        receive, ack and poll heads in the oracle's rounds."""
        c, L = self.c, self.L
        lead = c.leader
        replica = lead if replica is None else replica
        src = "" if replica == c.leader else f"follower {replica}'s read: "
        for e in lc.entries:
            before = c.offsets(lead)
            if e.typ == O.HEAD:
                b = live_boundaries(oracle_view(c, lead), before["head"], before["end"], L)
                nxt = request_stride(requests[self.pos]) if self.pos < len(requests) else None
                why = head_violation(L, before["head"], before["end"], e.value, b, self.prev_head, nxt, at=e.off)
                assert why is None, f"{src}HEAD idx {e.idx} at {e.off}: {why}"
                idx = c.prune_to(e.value)
                self.pairs += self.prev_head
                self.prev_head = True
            else:
                assert self.pos < len(requests), f"entry idx {e.idx} at {e.off} beyond the submitted stream"
                typ, clt, rid, payload = requests[self.pos]
                self.pos += 1
                got = (e.typ, e.clt_id, e.req_id, 0 if e.typ == O.CONFIG else e.value)
                want = (typ, clt, rid, 0 if typ == O.CONFIG else len(payload))
                assert got == want, f"entry idx {e.idx} at {e.off}: engine {got}, request {self.pos - 1} is {want}"
                idx = c.prologue() if typ == O.CONFIG else c.submit(typ, clt, rid, O.cmd_image(payload))
                self.prev_head = False
            after = c.offsets(lead)
            assert idx == e.idx, f"engine idx {e.idx} at {e.off}, oracle appended idx {idx}"
            assert after["tail"] == e.off, f"idx {e.idx}: engine wrote it at {e.off}, the oracle at {after['tail']}"
            start = 0 if before["end"] == L else before["end"]
            prev_start = self.last_start
            self.written += dist(start, after["end"], L)
            self.last_start = self.written - e.stride
            if e.typ == O.HEAD:
                self.heads.append(ReplayedHead(e.off, idx, e.value, self.last_start))
                if on_head is not None:
                    why = on_head(e, self.last_start, prev_start)
                    assert why is None, f"{src}HEAD idx {e.idx} at {e.off}: {why}"
                # commit it and let the followers poll it now: poll_head keeps the head closer to `end`, and a follower
                # head left stale while the launch laps most of the ring would look closer than the new one
                c.round(live=live)
                c.round(live=live)
                poll_heads(c, self.cid, live)
        assert c.offsets(lead)["end"] == lc.end, f"engine end {lc.end}, oracle end {c.offsets(lead)['end']}"
        c.round(live=live)
        c.round(live=live)
        poll_heads(c, self.cid, live)
        if len(lc.buf):
            pos = (lc.start + np.arange(len(lc.buf))) % L
            mine, want = lc.buf, oracle_view(c, replica)[pos]
            if replica != c.leader:
                ents = [((e.off - lc.start) % L, e.stride) for e in lc.entries]
                mine, want = O.mask_replies(mine, ents), O.mask_replies(want, ents)
            d = np.nonzero(want != mine)[0]
            if len(d):
                at = int(pos[d[0]])
                ent = next((e for e in lc.entries if e.off <= at < e.off + e.stride), None)
                what = (f"byte {at - ent.off} of the {'HEAD' if ent.typ == O.HEAD else 'type ' + str(ent.typ)} entry "
                        f"idx {ent.idx} at {ent.off}") if ent else "outside every entry"
                who = "leader" if replica == c.leader else f"follower {replica}"
                raise AssertionError(f"{who}: {len(d)} bytes of the launch [{lc.start}, {lc.end}) differ, first at "
                                     f"{at}, {what} (engine {mine[d[0]]} oracle {want[d[0]]})")

    def last_committed_head(self):
        """the head carried by the last HEAD entry replayed (what every follower holds once it is committed)"""
        return self.heads[-1].value if self.heads else 0


def poll_heads(c, cid, live=None):
    """SIM(poll_head) on every follower of the oracle cluster `c` (on those in `live`, when given); `cid`: each replica's
    scan position, carried over"""
    for i in range(c.n):
        if i != c.leader and (live is None or i in live):
            cur = C.c_uint64(cid[i])
            c.poll_head(i, C.byref(cur))
            cid[i] = int(cur.value)


def hole_bytes_of_head(img, off):
    """bytes 41..47 and 56..63 of the HEAD entry at `off`: no append writes them, the ring's old bytes stay"""
    return np.concatenate([img[off + 41:off + 48], img[off + 56:off + 64]])


def assert_heads_have_teeth(rp, img):
    """At least one replayed HEAD that is still in the final image lies in a range an earlier lap wrote, and its holes
    are not all zero there: a prefill that stored zeros in place of the HEAD's holes, or loaded the wrong chunks, then
    shows in the byte comparison.  Returns how many HEADs qualify."""
    L = rp.L
    cands = [h for h in rp.heads if h.lap_pos >= L and _u(img, h.off, 8) == h.idx and img[h.off + 26] == O.HEAD]
    teeth = [h for h in cands if np.count_nonzero(hole_bytes_of_head(img, h.off))]
    assert teeth, (f"no replayed HEAD over bytes of an earlier lap with non-zero holes: {len(rp.heads)} HEADs, "
                   f"{len(cands)} still in the ring past the first lap")
    return len(teeth)


# ---- recordings of followers whose host applies the log (APUS_F_HOST_APPLY) ---------------------------------------
@dataclass
class Recording:
    """What one follower's host read and reported, in absolute positions.  `segs`: (start, bytes, t) per read of a
    committed range, t the time the read returned; `reports`: (offset, t) per apply offset reported, t the time just
    before the report."""
    follower: int
    segs: list = field(default_factory=list)
    reports: list = field(default_factory=list)


def boundary_within(buf, start, L, step):
    """the largest entry end at most `step` bytes into `buf`, the ring bytes read from ring offset `start` (at least
    the first entry's end, so a lagging host always moves on)"""
    img = np.zeros(L, dtype=np.uint8)
    img[(start + np.arange(len(buf))) % L] = buf
    best = None
    for off, stride in O.walk_entries(img, start, (start + len(buf)) % L, L):
        k = dist(start, (off + stride) % L, L) or L
        if k > step and best is not None:
            break
        best = k
    return best


class Recorder:
    """A follower's host that applies the log the way libapus_dare.so's follower_pump does: read the committed range
    [apply, commit), keep the bytes, report the new apply offset.  Prompt (`step` None) it reports all it read at
    once; lagging it sleeps `lag_s` after each read and reports at most `step` bytes, ending on an entry boundary.
    It stops once its commit offset is the leader's final end (`finish`) and it has reported it."""

    def __init__(self, r, follower, L, step=None, lag_s=0.0):
        self.r, self.L, self.step, self.lag_s = r, L, step, lag_s
        self.rec = Recording(follower)
        self.final = None
        self.error = None
        self.stop = threading.Event()
        self.th = threading.Thread(target=self._run, daemon=True)

    def start(self):
        self.th.start()
        return self

    def finish(self, final_end, timeout=60.0):
        """the leader's end once everything is committed: wait until this follower has read and reported it"""
        self.final = final_end
        self.th.join(timeout)
        if self.th.is_alive():
            self.stop.set()
            self.th.join(5.0)
            raise AssertionError(f"follower {self.rec.follower}: its host did not reach the final end {final_end}")
        self.check()

    def check(self):
        if self.error:
            raise AssertionError(f"follower {self.rec.follower}'s host: {self.error}")

    def _run(self):
        try:
            self._loop()
        except Exception as ex:                                  # noqa: BLE001 - raised by check()
            self.error = f"{type(ex).__name__}: {ex}"
            self.stop.set()

    def _loop(self):
        r, L, rec = self.r, self.L, self.rec
        apply, at = 0, 0                                         # ring offset reported, and its absolute position
        while not self.stop.is_set():
            off, _ = r.progress()
            if off == apply:
                if self.final is not None and off == self.final:
                    return
                time.sleep(0.0002)
                continue
            buf = r.read_range(apply, off, cap=L)
            t = time.perf_counter()
            assert len(buf) == dist(apply, off, L), (apply, off, len(buf))
            rec.segs.append((at, buf, t))
            if self.step is None:
                adv = len(buf)
            else:
                time.sleep(self.lag_s)
                adv = boundary_within(buf, apply, L, self.step)
            apply, at = (apply + adv) % L, at + adv
            t = time.perf_counter()
            r.set_applied(apply)
            rec.reports.append((at, t))


def coverage_gap(rec, final):
    """the first stretch of [0, final) that no read of `rec` covers, or None"""
    covered = 0
    for s, b, _ in sorted(rec.segs, key=lambda x: x[0]):
        if s > covered:
            return covered, s
        covered = max(covered, s + len(b))
    return None if covered >= final else (covered, final)


def _entry_at(pieces, at, L):
    """(absolute start, Entry) of the entry of the replayed sequence whose bytes hold the absolute position `at`"""
    for c0, lc in pieces:
        for e in lc.entries:
            a = c0 + dist(lc.start, e.off, L)
            if a <= at < a + e.stride:
                return a, e
    return None, None


def _kind(typ):
    return "HEAD" if typ == O.HEAD else f"type {typ}"


def compare_read(rp, j, s, buf, flat):
    """follower j's read of [s, s + len(buf)) against replica j of the oracle right after the piece ending at its end,
    reply bytes masked.  `flat`: the recorded sequence by absolute position, to tell a read that a later lap had
    overwritten from any other difference."""
    c, L = rp.c, rp.L
    view = oracle_view(c, j)
    e = s + len(buf)
    pos = (s + np.arange(len(buf))) % L
    ents = O.walk_entries(view, s % L, e % L, L)
    rel = [((off - s) % L, stride) for off, stride in ents]
    mine, want = O.mask_replies(buf, rel), O.mask_replies(view[pos], rel)
    d = np.nonzero(mine != want)[0]
    if not len(d):
        return
    at = int(pos[d[0]])
    ent = next(((off, stride) for off, stride in ents if off <= at < off + stride), None)
    if ent is None:
        raise AssertionError(f"follower {j}: {len(d)} bytes of the read of [{s}, {e}) differ from the oracle, first at "
                             f"{at}, outside every entry (recorded {mine[d[0]]} oracle {want[d[0]]})")
    off, stride = ent
    idx, typ = _u(view, off, 8), int(view[off + 26])
    k0 = (off - s) % L
    for lap in range(1, (len(flat) - s) // L + 1):               # the bytes a later lap left there?
        later = s + k0 + lap * L
        span = d[(d >= k0) & (d < k0 + stride)]
        if later + stride <= len(flat) and len(span) and np.mean(flat[s + span + lap * L] == buf[span]) > 0.9:
            raise AssertionError(f"follower {j}: entry idx {idx} at {off} was overwritten by lap +{lap} before the read "
                                 f"of [{s}, {e}) returned: byte {at - off} is {mine[d[0]]}, the oracle {want[d[0]]}")
    raise AssertionError(f"follower {j}: {len(d)} bytes of the read of [{s}, {e}) differ from the oracle, first at "
                         f"{at}: byte {at - off} of the {_kind(typ)} entry idx {idx} at {off} "
                         f"(recorded {mine[d[0]]} oracle {want[d[0]]})")


def recording_pieces(recs, L):
    """The recorded sequence cut at every offset any follower read up to (each a commit offset, so an entry boundary
    of the one append sequence), parsed from the gap-free recording of the most prompt host.  Returns (pieces, flat,
    source follower, gaps): pieces as (absolute start, Launch), flat the recorded bytes by absolute position."""
    final = max(s + len(b) for rec in recs for s, b, _ in rec.segs)
    gaps = {rec.follower: coverage_gap(rec, final) for rec in recs}
    whole = [rec for rec in recs if gaps[rec.follower] is None]
    assert whole, f"every recording has a gap: {gaps}"
    # the most prompt host: the least read and left unreported, summed over its reads
    src = min(whole, key=lambda rec: sum(s + len(b) - a for (s, b, _), (a, _) in zip(rec.segs, rec.reports)))
    flat = np.zeros(final, dtype=np.uint8)
    for s, b, _ in src.segs:
        flat[s:s + len(b)] = b
    ring = np.zeros(L, dtype=np.uint8)
    pieces, prev = [], 0
    for cut in sorted({s + len(b) for rec in recs for s, b, _ in rec.segs}):
        assert cut - prev < L, f"the piece [{prev}, {cut}) between two reads is a lap or more"
        ring[(prev + np.arange(cut - prev)) % L] = flat[prev:cut]
        pieces.append((prev, Launch(prev % L, cut % L, flat[prev:cut], parse_entries(ring, prev % L, cut % L, L))))
        prev = cut
    return pieces, flat, src.follower, gaps


def replay_recordings(rp, recs, requests, pieces=None):
    """Replay what the followers' hosts recorded over one or more launches (`recs`, one Recording per follower) into
    the fresh Replay `rp`, piece by piece.  After each piece every read that ended there is compared with the oracle,
    and every HEAD entry is checked against the apply offsets the followers had reported before it was first read:
    its head may be past none of them, and is one of them, or the tail when every follower had reported the HEAD's
    own position (the leader leaves one entry then).  `pieces`: recording_pieces' pieces, to replay in their place
    (a test of the harness alters them).  Returns the pieces."""
    L = rp.L
    cut, flat, src, gaps = recording_pieces(recs, L)
    pieces = cut if pieces is None else pieces
    for j, gap in sorted(gaps.items()):
        if gap is not None:
            a, e = _entry_at(pieces, gap[0], L)
            what = f"byte {gap[0] - a} of the {_kind(e.typ)} entry idx {e.idx} at {e.off}" if e else "past every entry"
            raise AssertionError(f"follower {j}: the recording has a gap [{gap[0]}, {gap[1]}): {what} was never read")
    ends = defaultdict(list)
    for rec in recs:
        for s, b, _ in rec.segs:
            ends[s + len(b)].append((rec.follower, s, b))
    starts = np.array([s for rec in recs for s, _, _ in rec.segs], dtype=np.int64)
    stops = np.array([s + len(b) for rec in recs for s, b, _ in rec.segs], dtype=np.int64)
    times = np.array([t for rec in recs for _, _, t in rec.segs], dtype=np.float64)
    reports = {rec.follower: [(0, float("-inf"))] + sorted(rec.reports, key=lambda x: x[1]) for rec in recs}

    def on_head(e, at, prev_at):
        seen = (starts <= at) & (stops >= at + e.stride)
        if not seen.any():
            return "no follower's host read it"
        t = times[seen].min()
        v = at - dist(e.value, e.off, L)                         # the head it carries, as an absolute position
        legal = set()
        last = {}
        for j, rs in reports.items():
            before = [a for a, tr in rs if tr < t]
            last[j] = max(before)
            legal.update(before)
            if v > last[j]:
                return (f"head {e.value} (absolute {v}) is past follower {j}'s last report {last[j]} before the HEAD "
                        f"was first read (byte 48 of the HEAD entry at absolute {at})")
        if v in legal or (v == prev_at and all(x == at for x in last.values())):
            return None
        return (f"head {e.value} (absolute {v}) is no follower's report before the HEAD was first read, nor the tail "
                f"with every follower caught up (byte 48 of the HEAD entry; last reports {last})")

    for c0, lc in pieces:
        rp.launch(lc, requests, replica=src, on_head=on_head)
        for j, s, b in ends[c0 + len(lc.buf)]:
            compare_read(rp, j, s, b, flat)
    return pieces
