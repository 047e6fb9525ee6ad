"""Replay of device-side log pruning (APUS_F_AUTOPRUNE) into the CPU oracle (TEST INFRASTRUCTURE ONLY).

Where the leader puts an auto HEAD entry, and which head it carries, depends on how far the followers had applied when
the place turn was taken, so the oracle cannot predict it.  The layout depends only on the sequence of appends,
though: the wrap, ghost and E1 rules look at `end` and `len`, not at `head`, and rule E2 only decides whether the
leader blocks.  So the engine's own sequence is read back after every launch that stays under one lap, and the oracle
appends the same sequence: the submitted requests in order, and <HEAD, v> (SIM(prune_to)) wherever the engine put a
HEAD entry carrying v.  Every replayed HEAD is first checked against the engine's pruning rule (`head_violation`),
so the replay cannot launder an arbitrary head.  At the end every byte of every replica is compared with the oracle.
"""
import ctypes as C
from dataclasses import dataclass

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


def head_violation(L, head_old, end, v, boundaries, prev_was_head, allow_two=False):
    """The engine's pruning rule (leader_place) as a predicate over one HEAD entry appended at `end` while the head was
    `head_old`: None when a HEAD carrying `v` is legal there, else the reason.  `boundaries`: the starts and ends of
    the entries of [head_old, end).  `prev_was_head`: the entry just before is a HEAD; `allow_two` accepts that, which
    the leader does only when its placement was blocked on space behind the first one."""
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
    if prev_was_head and not allow_two:
        return "two HEAD entries in a row"
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
        self.written = 0                    # ring bytes appended so far (laps = written / L)
        self.cid = [0] * n                  # poll_head's scan position per replica
        self.pos = 0                        # requests consumed

    def close(self):
        self.c.close()

    def end(self):
        return self.c.offsets(0)["end"]

    def launch(self, lc, requests, allow_two=False):
        """Append what one launch appended (`lc`, read back from the leader; `requests` the submitted stream, a
        CONFIG request standing for the prologue), run two quiescent rounds and poll_head on every follower, then
        compare the oracle leader's bytes of the launch's range with the leader's: every entry the launch wrote,
        before a later lap overwrites it."""
        c, L = self.c, self.L
        for e in lc.entries:
            before = c.offsets(0)
            if e.typ == O.HEAD:
                b = live_boundaries(c.image(0), before["head"], before["end"], L)
                why = head_violation(L, before["head"], before["end"], e.value, b, self.prev_head, allow_two)
                assert why is None, f"HEAD idx {e.idx} at {e.off}: {why}"
                idx = c.prune_to(e.value)
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
            after = c.offsets(0)
            assert idx == e.idx, f"engine idx {e.idx} at {e.off}, oracle appended idx {idx}"
            assert after["tail"] == e.off, f"idx {e.idx}: engine wrote it at {e.off}, the oracle at {after['tail']}"
            start = 0 if before["end"] == L else before["end"]
            self.written += dist(start, after["end"], L)
            if e.typ == O.HEAD:
                self.heads.append(ReplayedHead(e.off, idx, e.value, self.written - e.stride))
                # commit it and let the followers poll it now: poll_head keeps the head closer to `end`, and a follower
                # head left stale while the launch laps most of the ring would look closer than the new one
                c.round()
                c.round()
                poll_heads(c, self.cid)
        assert c.offsets(0)["end"] == lc.end, f"engine end {lc.end}, oracle end {c.offsets(0)['end']}"
        c.round()
        c.round()
        poll_heads(c, self.cid)
        if len(lc.buf):
            pos = (lc.start + np.arange(len(lc.buf))) % L
            d = np.nonzero(c.image(0)[pos] != lc.buf)[0]
            if len(d):
                at = int(pos[d[0]])
                ent = next((e for e in lc.entries if e.off <= at < e.off + e.stride), None)
                what = (f"byte {at - ent.off} of the {'HEAD' if ent.typ == O.HEAD else 'type ' + str(ent.typ)} entry "
                        f"idx {ent.idx} at {ent.off}") if ent else "outside every entry"
                raise AssertionError(f"leader: {len(d)} bytes of the launch [{lc.start}, {lc.end}) differ, first at "
                                     f"{at}, {what} (engine {lc.buf[d[0]]} oracle {c.image(0)[at]})")

    def last_committed_head(self):
        """the head carried by the last HEAD entry replayed (what every follower holds once it is committed)"""
        return self.heads[-1].value if self.heads else 0


def poll_heads(c, cid):
    """SIM(poll_head) on every follower of the oracle cluster `c`; `cid`: each replica's scan position, carried over"""
    for i in range(c.n):
        if i != c.leader:
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
