"""The public device headers (include/apus_consumer.cuh, include/apus_submitter.cuh) primitive by primitive: the probe
kernels of tests/devicelogic/header_probe.cu call each primitive on views whose words all lie in plain device buffers
that the test fills, so every case is set up exactly and nothing depends on timing.  The references share no code with
the headers: numpy slices of seeded random bytes for the copy and the loads, the oracle's own log images walked with
orc.walk_entries for the consumer, and header_probe.Placement with the gcc-built slot writer (tests/hostlogic/
slot_writer.c) for the submitter.  One end-to-end leg runs a replica group with a payload ring whose size is not a power
of two.  Marked gpu."""
import ctypes as C

import numpy as np
import pytest

import autoprune_replay as AR
import engine_util as EU
import header_probe as HP
import orc as O
import submitter as SB
from apus_b200 import engine as E
from engine_util import MODES, devices_for, eng, submit_host, torch_module  # noqa: F401
from shadow import check_heads

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

RINGS = [1 << 17, 33 * 4096]
SECOND = 1_000_000_000
SHORT = 2_000_000          # 2 ms: a wait that must end TIMED_OUT


@pytest.fixture(scope="module")
def probe():
    import torch
    torch.cuda.init()
    return HP.lib()


def cuda(a):
    import torch
    return torch.from_numpy(np.array(a, copy=True)).cuda()


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------
# copy and loads
# ---------------------------------------------------------------------------------
COPY_LENS = list(range(41)) + [47, 48, 49, 63, 64, 65, 79, 80, 81, 127, 128, 129, 1500, 4095]
COPY_DT = np.dtype([("src", "<u8"), ("dst", "<u8"), ("len", "<u4"), ("nthr", "<u4"), ("groups", "<u4"),
                    ("via", "<u4")])
SRC_END = 1 << 20          # the source pattern; the 4 KiB after it hold other bytes
GUARD = 32


def copy_cases(rng):
    """(src, len, nthr, groups, via, dst alignment) of every case"""
    out = []
    for sa in range(16):
        for da in range(16):
            for ln in COPY_LENS:
                for nthr in (1, 3, 8, 32, 128):
                    out.append((sa, ln, nthr, 1, len(out) & 1, da))
                for nthr, groups in ((8, 2), (8, 4), (3, 4), (32, 4), (128, 4)):
                    if nthr != 8 and ln % 3:
                        continue
                    out.append((sa, ln, nthr, groups, len(out) & 1, da))
    for sa, da in ((0, 0), (0, 1), (1, 0), (7, 9), (15, 15), (15, 1), (8, 8)):
        for nthr in (1, 8, 128):
            out.append((sa, 65535, nthr, 1, nthr & 1, da))
    cases = []
    for sa, ln, nthr, groups, via, da in out:
        tot = ln * groups
        src = 16 * int(rng.integers(1, (SRC_END - tot - 64) // 16)) + sa
        cases.append((src, tot, ln, nthr, groups, via, da))
    # sources whose range ends exactly at the 16 B-aligned end of the pattern
    for ln in COPY_LENS + [65535]:
        for da in range(16):
            for nthr in (1, 8, 32):
                cases.append((SRC_END - ln, ln, ln, nthr, 1, da & 1, da))
    return cases


def test_copy_every_alignment_and_split(probe):
    """apus_copy_cmd and apus_consumer_copy_cmd: every src % 16 and dst % 16 pair, lengths 0..40 and around every
    16 B step up to 4095 (and 65535 on a few pairs), groups of 1, 3, 8, 32 and 128 threads, two or four groups side by
    side copying to adjacent destinations, and sources that end exactly at the pattern's end.  Every destination byte
    equals the source byte, and the 32 guard bytes on each side of every destination are untouched"""
    rng = np.random.default_rng(20261018)
    src = rng.integers(0, 256, SRC_END + 4096, dtype=np.uint8)
    cases = copy_cases(rng)
    arr = np.zeros(len(cases), dtype=COPY_DT)
    at = 0
    for q, (s, tot, ln, nthr, groups, via, da) in enumerate(cases):
        d = at + GUARD + da
        arr[q] = (s, d, ln, nthr, groups, via)
        at = (d + tot + GUARD + 15) & ~15
    guard = rng.integers(0, 256, at + GUARD, dtype=np.uint8)
    want = guard.copy()
    for (s, d, ln, nthr, groups, via), (_, tot, *_) in zip(arr, cases):
        want[d:d + tot] = src[s:s + tot]
    assert not np.array_equal(want, guard)
    d_src, d_dst, d_cases = cuda(src), cuda(guard), cuda(arr.view(np.uint8))
    assert probe.hp_copy(d_src.data_ptr(), d_dst.data_ptr(), d_cases.data_ptr(), len(arr), stream()) == 0
    got = d_dst.cpu().numpy()
    if not np.array_equal(got, want):
        for (s, d, ln, nthr, groups, via), (_, tot, *_) in zip(arr, cases):
            lo, hi = int(d) - GUARD, int(d) + tot + GUARD
            if not np.array_equal(got[lo:hi], want[lo:hi]):
                bad = np.nonzero(got[lo:hi] != want[lo:hi])[0] - GUARD
                pytest.fail(f"src {s} (% 16 = {s % 16}) dst % 16 = {d % 16} len {ln} nthr {nthr} groups {groups} "
                            f"via {via}: bytes {bad[:8].tolist()} differ")
    print(f"copy cases: {len(arr)}")


def test_loads_at_every_offset(probe):
    """apus_ld_u8_any, apus_ld_u16_any and apus_ld_u64_any at every offset 0..63 are the little-endian values there"""
    buf = np.random.default_rng(7).integers(0, 256, 128, dtype=np.uint8)
    d = cuda(buf)
    import torch
    o8 = torch.zeros(64, dtype=torch.int32, device="cuda")
    o16 = torch.zeros(64, dtype=torch.int32, device="cuda")
    o64 = torch.zeros(64, dtype=torch.int64, device="cuda")
    assert probe.hp_loads(d.data_ptr(), o8.data_ptr(), o16.data_ptr(), o64.data_ptr(), stream()) == 0
    g8, g16 = o8.cpu().numpy().view(np.uint32), o16.cpu().numpy().view(np.uint32)
    g64 = o64.cpu().numpy().view(np.uint64)
    for a in range(64):
        assert g8[a] == buf[a], a
        assert g16[a] == buf[a:a + 2].view("<u2")[0], a
        assert g64[a] == buf[a:a + 8].view("<u8")[0], a


# ---------------------------------------------------------------------------------
# consumer
# ---------------------------------------------------------------------------------
LOG = 1 << 16


def u16(img, at):
    return int(img[at]) | int(img[at + 1]) << 8


def u64(img, at):
    return int(img[at:at + 8].view("<u8")[0])


class Snapshot:
    """the leader's log image and the history of appended entries [(idx, off, type)] at one point of the build"""

    def __init__(self, c, hist, name):
        self.img, self.hist, self.name = c.image(0), list(hist), name
        o = c.offsets(0)
        self.head, self.end = o["head"], o["end"]
        self.live = O.walk_entries(self.img, self.head, self.end, LOG)
        for off, _ in self.live:                        # the walk and the history agree on the live entries
            i = u64(self.img, off)
            assert self.hist[i - 1][:2] == (i, off), (name, i, off)

    def index(self, mask, upto=None):
        """the offset index as the leader writes it, entry after entry (words of pruned entries stay stale); only the
        entries through idx `upto` when given"""
        ix = np.zeros(mask + 1, dtype=np.uint32)
        for i, off, typ in self.hist:
            if upto is None or i <= upto:
                ix[i & mask] = off | (HP.HEAD_BIT if typ == O.HEAD else 0)
        return ix

    def idx(self, k):
        return u64(self.img, self.live[k][0])

    def stop(self, k):
        """the consumer position where live entry k ends: its end, L mapped to 0"""
        off, st = self.live[k]
        return (off + st) % LOG


def build_log():
    """An oracle log of LOG bytes over several laps, with HEAD entries from prune_to and snapshots where an entry ends
    exactly at L ("exact"), where one is placed at 0 behind a gap ("ghost"), and at the end ("final")"""
    orc = O.Oracle("orc")
    orc.set_rules(O.RULES_ENGINE)
    c = O.Cluster(orc, 3, length=LOG)
    rng = np.random.default_rng(99)
    hist, snaps, pending = [], {}, {}

    def appended(typ):
        i = len(hist) + 1
        hist.append((i, c.offsets(0)["tail"], typ))

    assert c.prologue() == 1
    appended(O.CONFIG)
    exact_done = False
    while len(hist) < 1500:
        o = c.offsets(0)
        live = (o["end"] - o["head"]) % LOG
        if live > LOG // 2 and hist[-1][2] != O.HEAD:
            assert c.prune_to(hist[-60][1]) == len(hist) + 1
            appended(O.HEAD)
            continue
        room = LOG - o["end"]
        typ = int(rng.choice([O.CSM, O.SEND, O.CONNECT, O.CLOSE, O.NOOP]))
        ln = int(rng.integers(0, 300)) if rng.random() > 0.05 else int(rng.integers(1000, 3000))
        if not exact_done and len(hist) > 200 and 2 * HP.HDR <= room <= 2 * HP.HDR + 400:
            typ, ln = O.SEND, room - HP.HDR            # this entry ends exactly at L
            exact_done = True
        if typ == O.NOOP:
            idx = c.submit(O.NOOP, 0, 10_000 + len(hist), b"")
        else:
            idx = c.submit(typ, int(rng.integers(0, 9)), 10_000 + len(hist), O.cmd_image(rng.bytes(ln)))
        assert idx == len(hist) + 1
        appended(typ)
        t = hist[-1][1]
        if typ != O.NOOP and t + HP.HDR + ln == LOG and "exact" not in pending:
            pending["exact"] = len(hist) + 30
        if t == 0 and len(hist) > 2 and hist[-2][1] > 0 and "ghost" not in pending:
            prev_off = hist[-2][1]
            prev_img = c.image(0)
            prev_end = prev_off + stride_at(prev_img, prev_off)
            if prev_end < LOG:
                pending["ghost"] = len(hist) + 30
        for name, at in list(pending.items()):
            if at == len(hist) and name not in snaps:
                snaps[name] = Snapshot(c, hist, name)
    snaps["final"] = Snapshot(c, hist, "final")
    c.close()
    assert set(snaps) == {"exact", "ghost", "final"}, set(snaps)
    return snaps


def stride_at(img, off):
    typ = int(img[off + 26])
    return HP.HDR if typ in (O.NOOP, O.CONFIG, O.HEAD) else HP.HDR + u16(img, off + 48)


@pytest.fixture(scope="module")
def logs():
    O.build_oracle()
    return build_log()


def expect_entry(img, off, idx):
    typ = int(img[off + 26])
    has = typ not in (O.NOOP, O.CONFIG, O.HEAD)
    ln = u16(img, off + 48) if has else 0
    return dict(idx=idx, off=off, type=typ, len=ln, cmd_off=off + 50, clt_id=u16(img, off + 24) if has else 0,
                req_id=u64(img, off + 16) if has else 0, status=HP.CONS_OK)


def run_consumer(probe, img, index, cursor, next_idx, committed, held, threads, error=0, cap=2048, stride=4096):
    """one pass of hp_consumer; returns (out words, entries, rows, error, status, cur)"""
    import torch
    d_img, d_ix = cuda(img), cuda(index.view(np.int32))
    words = torch.tensor([committed, held, cursor, next_idx, error, 0, 0, 0, 0, 7], dtype=torch.int64, device="cuda")
    ents = torch.zeros(cap * C.sizeof(HP.Entry), dtype=torch.uint8, device="cuda")
    rows = torch.zeros(cap * stride, dtype=torch.uint8, device="cuda")
    out = torch.zeros(8, dtype=torch.int64, device="cuda")
    p = words.data_ptr()
    v = E.ConsumerView(d_img.data_ptr(), LOG, d_ix.data_ptr(), len(index) - 1, 0, p, p + 16, p + 32, p + 40, p + 72, 7)
    assert probe.hp_consumer(C.byref(v), ents.data_ptr(), cap, rows.data_ptr(), stride, out.data_ptr(), threads,
                             stream()) == 0
    o = [int(x) for x in out.cpu()]
    w = [int(x) for x in words.cpu()]
    eb = ents.cpu().numpy().tobytes()
    es = [HP.Entry.from_buffer_copy(eb, k * C.sizeof(HP.Entry)) for k in range(min(o[2], cap))]
    return o, es, rows.cpu().numpy().reshape(cap, stride), w[4], w[5:9], w[2:4]


def check_ok(e, want, rows, k, img):
    got = dict(idx=e.idx, off=e.off, type=e.type, len=e.len, cmd_off=e.cmd_off, clt_id=e.clt_id, req_id=e.req_id,
               status=e.status)
    assert got == want, (k, got, want)
    if want["type"] not in (O.NOOP, O.CONFIG, O.HEAD):
        assert np.array_equal(rows[k, :want["len"]], img[want["cmd_off"]:want["cmd_off"] + want["len"]]), k


def consume_case(probe, s, k0, k1, threads, held=None, committed=None, index=None, mask=4095):
    """the consumer pass from live entry k0 with entries k0 .. k1 - 1 committed (the record's offset at entry k1's start,
    or `committed`); `held` overrides the entries the record holds"""
    cursor = s.live[k0][0] if k0 == 0 or s.stop(k0 - 1) == s.live[k0][0] else s.stop(k0 - 1)
    nxt = s.idx(k0)
    if committed is None:
        committed = s.live[k1][0] if k1 < len(s.live) else s.end
    if held is None:
        held = s.idx(k1 - 1) if k1 > k0 else nxt - 1
    ix = s.index(mask) if index is None else index
    return cursor, nxt, run_consumer(probe, s.img, ix, cursor, nxt, committed, held, threads)


@pytest.mark.parametrize("threads", [1, 32, 100, 256])
@pytest.mark.parametrize("snap", ["final", "ghost", "exact"])
def test_consumer_plain_run(probe, logs, snap, threads):
    """the live range of a lapped log, HEAD entries included, with and without a wrap: every entry between cursor and
    commit, in walk order, with its fields and cmd bytes; the cursor moves to the commit and nothing more is
    available"""
    s = logs[snap]
    k0, k1 = 3, len(s.live)
    cursor, nxt, (o, es, rows, err, status, cur) = consume_case(probe, s, k0, k1, threads)
    walk = O.walk_entries(s.img, cursor, s.end, LOG)
    assert walk == s.live[k0:]
    assert o[:5] == [cursor, nxt, len(walk), s.end, len(walk)]
    for k, (off, _) in enumerate(walk):
        check_ok(es[k], expect_entry(s.img, off, nxt + k), rows, k, s.img)
    assert any(es[k].type == O.HEAD for k in range(len(walk)))
    assert any(off < cursor for off, _ in walk) == (snap != "final")
    assert o[5:] == [s.end, nxt + len(walk), 0]
    assert cur == [s.end, nxt + len(walk)] and err == 0 and status == [s.end, nxt + len(walk), 0, 0]


@pytest.mark.parametrize("threads", [1, 64])
def test_consumer_entry_ending_at_L(probe, logs, threads):
    """the examined range ends with an entry that ends exactly at L: the new cursor is 0, the entry at 0 is next"""
    s = logs["exact"]
    j = next(k for k, (off, st) in enumerate(s.live) if off + st == LOG)
    assert s.live[j + 1][0] == 0
    cursor, nxt, (o, es, rows, err, status, cur) = consume_case(probe, s, j - 4, j + 1, threads, committed=0)
    assert o[2] == 5 and o[4] == 5
    for k in range(5):
        check_ok(es[k], expect_entry(s.img, s.live[j - 4 + k][0], nxt + k), rows, k, s.img)
    assert o[5:7] == [0, s.idx(j + 1)] and cur == [0, s.idx(j + 1)] and err == 0
    # from there on: the entry at 0 and the ones after it
    cursor, nxt, (o, es, *_r) = consume_case(probe, s, j + 1, j + 4, threads)
    assert cursor == 0 and o[4] == 3 and es[0].off == 0 and o[5] == s.stop(j + 3)


@pytest.mark.parametrize("threads", [1, 32])
def test_consumer_cursor_in_the_ghost_gap(probe, logs, threads):
    """a cursor in the gap an entry left at the ring's end: the next entry is the one at 0"""
    s = logs["ghost"]
    g = next(k for k, (off, _) in enumerate(s.live) if off == 0 and k and s.stop(k - 1) != 0)
    cursor, nxt, (o, es, rows, err, status, cur) = consume_case(probe, s, g, g + 3, threads)
    assert cursor == s.stop(g - 1) and 0 < cursor < LOG
    assert o[4] == 3 and [e.off for e in es] == [s.live[g + q][0] for q in range(3)]
    for k in range(3):
        check_ok(es[k], expect_entry(s.img, s.live[g + k][0], nxt + k), rows, k, s.img)
    assert o[5] == s.stop(g + 2) and err == 0


def test_consumer_head_entry(probe, logs):
    """a HEAD entry's index word carries APUS_INDEX_HEAD_BIT; the entry is found at the offset without it"""
    s = logs["final"]
    h = next(k for k, (off, _) in enumerate(s.live) if k > 2 and s.img[off + 26] == O.HEAD)
    ix = s.index(4095)
    assert ix[s.idx(h) & 4095] & HP.HEAD_BIT
    _, nxt, (o, es, rows, err, *_r) = consume_case(probe, s, h, h + 2, 32)
    assert o[4] == 2 and es[0].type == O.HEAD and es[0].off == s.live[h][0] and es[0].len == 0 and err == 0
    check_ok(es[0], expect_entry(s.img, s.live[h][0], nxt), rows, 0, s.img)


def test_consumer_nothing_committed_past_the_cursor(probe, logs):
    """committed == cursor: nothing is available; a record whose entry count runs ahead of its offset still gives
    LATER for every entry, and the cursor stays"""
    s = logs["final"]
    cursor, nxt, (o, es, _, err, status, cur) = consume_case(probe, s, 10, 10, 32)
    assert o[2] == 0 and o[4] == 0 and o[5:7] == [cursor, nxt] and cur == [cursor, nxt] and err == 0
    cursor, nxt, (o, es, _, err, status, cur) = consume_case(probe, s, 10, 10, 32, held=s.idx(13), committed=cursor)
    assert o[2] == 4 and o[4] == 0 and [e.status for e in es] == [HP.CONS_LATER] * 4
    assert [e.off for e in es] == [s.live[10 + q][0] for q in range(4)]
    assert o[5:7] == [cursor, nxt] and err == 0 and o[7] == 4


@pytest.mark.parametrize("threads", [1, 7, 128])
def test_consumer_commit_at_an_entry_start(probe, logs, threads):
    """committed exactly at an entry's start: that entry is LATER and the examination stops just before it"""
    s = logs["final"]
    cursor, nxt, (o, es, rows, err, status, cur) = consume_case(probe, s, 20, 30, threads, held=s.idx(30))
    assert o[2] == 11 and o[4] == 10
    for k in range(10):
        check_ok(es[k], expect_entry(s.img, s.live[20 + k][0], nxt + k), rows, k, s.img)
    assert es[10].status == HP.CONS_LATER and es[10].off == s.live[30][0] and es[10].idx == nxt + 10
    assert o[5:7] == [s.live[30][0], nxt + 10] and err == 0 and o[7] == 1


@pytest.mark.parametrize("threads", [1, 16, 64])
def test_consumer_small_index_and_a_stale_word(probe, logs, threads):
    """idx_mask 15: the index wraps and the first 16 entries are found; the word of the 17th still names an entry of
    another idx (the leader has not written it), which is BAD: the sticky error and status[3] are set, the cursor
    stops after the 16th, and the next available reports nothing"""
    s = logs["final"]
    k0 = next(k for k in range(5, 40) if s.idx(k) & 15 == 9)          # the 16 words wrap around the index
    ix = s.index(15, upto=s.idx(k0 + 15))
    cursor, nxt, (o, es, rows, err, status, cur) = consume_case(probe, s, k0, k0 + 18, threads, index=ix, mask=15)
    assert o[2] == 18 and o[4] == 16
    for k in range(16):
        check_ok(es[k], expect_entry(s.img, s.live[k0 + k][0], nxt + k), rows, k, s.img)
    assert es[16].status == HP.CONS_BAD and es[16].off == s.live[k0][0]
    assert err == 1
    assert o[5:] == [s.stop(k0 + 15), nxt + 16, 0] and status == [s.stop(k0 + 15), nxt + 16, 0, 1]


def test_consumer_index_word_past_L_and_stride_past_L(probe, logs):
    """an index word with o + 64 > L, and an entry whose poked cmd length makes its stride pass L: both are BAD"""
    s = logs["ghost"]
    g = next(k for k, (off, _) in enumerate(s.live) if off == 0 and k and s.stop(k - 1) != 0)
    k0 = g - 6
    ix = s.index(4095)
    ix[s.idx(k0 + 2) & 4095] = LOG - 32
    _, nxt, (o, es, _, err, status, _) = consume_case(probe, s, k0, g + 2, 32, index=ix)
    assert o[4] == 2 and es[2].status == HP.CONS_BAD and es[2].off == LOG - 32 and err == 1 and status[3] == 1
    assert o[5:] == [s.stop(k0 + 1), nxt + 2, 0]
    c = max(k for k in range(k0, g) if s.img[s.live[k][0] + 26] not in (O.NOOP, O.CONFIG, O.HEAD))
    off = s.live[c][0]
    img = s.img.copy()
    s2 = Snapshot.__new__(Snapshot)
    s2.__dict__.update(s.__dict__)
    s2.img = img
    bad_len = LOG - off - HP.HDR + 1
    img[off + 48:off + 50] = np.array([bad_len & 0xFF, bad_len >> 8], dtype=np.uint8)
    _, nxt, (o, es, _, err, status, _) = consume_case(probe, s2, k0, g + 2, 32)
    assert o[4] == c - k0 and es[c - k0].status == HP.CONS_BAD and err == 1 and status[3] == 1


# ---------------------------------------------------------------------------------
# submitter
# ---------------------------------------------------------------------------------
EPOCH = 7


class Ring:
    """a submitter view over test buffers: S slots, R payload bytes, guard-filled, and the words the leader shares"""

    def __init__(self, S, R, seed=5):
        import torch
        self.S, self.R = S, R
        rng = np.random.default_rng(seed)
        self.guard_slots = rng.integers(0, 256, S * 128, dtype=np.uint8)
        self.guard_pay = rng.integers(0, 256, R, dtype=np.uint8)
        self.cmds = rng.integers(0, 256, 1 << 18, dtype=np.uint8)
        self.d_slots, self.d_pay, self.d_cmds = cuda(self.guard_slots), cuda(self.guard_pay), cuda(self.cmds)
        self.words = torch.zeros(8 + 5, dtype=torch.int64, device="cuda")   # state[8], doorbell, consumed, committed, stop
        self.pay_end = torch.zeros(S, dtype=torch.int64, device="cuda")
        p = self.words.data_ptr()
        self.view = E.SubmitterView(self.d_slots.data_ptr(), self.d_pay.data_ptr(), p + 64, S, R, p, self.pay_end.data_ptr(),
                                    p + 72, p + 80, p + 88, EPOCH)

    def setup(self, submitted, head, consumed=None, leader=None, wrap_next=0, doorbell=None, committed=0, stop=EPOCH,
              tail=None):
        """a fresh ring: guard bytes everywhere, `submitted` tickets handed out and published, `consumed` of them taken
        (the cached count; `leader`: the leader's word), the payload counter at `head`, free from `tail` on"""
        assert head % 16 == 0, "the payload counter moves in 16 B units: images are 16 B aligned"
        consumed = submitted if consumed is None else consumed
        leader = consumed if leader is None else leader
        self.d_slots.copy_(cuda(self.guard_slots))
        self.d_pay.copy_(cuda(self.guard_pay))
        st = [0, submitted, head, wrap_next, consumed, 0, (1 << 64) - 1, 0]
        w = st + [submitted if doorbell is None else doorbell, leader, committed, stop, 0]
        self.words.copy_(cuda(np.array(w, dtype=np.uint64).view(np.int64)))
        pe = np.full(self.S, head, dtype=np.int64)
        if tail is not None and consumed:
            pe[(consumed - 1) % self.S] = tail
        self.pay_end.copy_(cuda(pe))
        self.model = HP.Placement(self.S, self.R, submitted, head, consumed, wrap_next)
        self.model.pay_end = list(pe)
        self.leader = leader
        self.puts = []                                 # (ticket, pos or None, wrap, type, conn, req_id, cmd_off, len)
        self.reserved = set()

    def state(self):
        w = [int(x) for x in self.words.cpu().numpy().view(np.uint64)]
        return dict(zip(("lock", "submitted", "pay_head", "wrap_next", "consumed", "rejected", "first_rejected"), w[:7]),
                    doorbell=w[8])

    def run(self, scripts, reqs, threads=32):
        """run one script per CTA; returns [[Out of each step] per CTA]"""
        import torch
        steps, first = [], [0]
        for sc in scripts:
            steps += sc
            first.append(len(steps))
        sa = (HP.Step * len(steps))(*steps)
        ra = (HP.Req * max(len(reqs), 1))(*[HP.Req(*r) for r in reqs])
        d_steps = cuda(np.frombuffer(bytes(sa), dtype=np.uint8))
        d_first = cuda(np.array(first, dtype=np.int32))
        d_reqs = cuda(np.frombuffer(bytes(ra), dtype=np.uint8))
        d_out = torch.zeros(len(steps) * C.sizeof(HP.Out), dtype=torch.uint8, device="cuda")
        d_order = torch.zeros(1, dtype=torch.int64, device="cuda")
        assert HP.lib().hp_submit(C.byref(self.view), d_steps.data_ptr(), d_first.data_ptr(), d_reqs.data_ptr(),
                                  self.d_cmds.data_ptr(), d_out.data_ptr(), d_order.data_ptr(), len(scripts), threads,
                                  stream()) == 0
        ob = d_out.cpu().numpy().tobytes()
        outs = [HP.Out.from_buffer_copy(ob, k * C.sizeof(HP.Out)) for k in range(len(steps))]
        return [outs[first[b]:first[b + 1]] for b in range(len(scripts))]

    def expect(self, res, step, reqs):
        """the model's reservation for a reserve step, checked against the probe's Out `res`; records its puts"""
        n, req0 = step.n, step.req0
        need = sum(HP.ext_bytes(reqs[req0 + k][0], reqs[req0 + k][2]) for k in range(n)) \
            if step.ext == HP.EXT_OF_REQUESTS else step.ext
        want = self.model.reserve(n, need, self.leader)
        got = (res.outcome, res.first_ticket, res.pos, res.wrap)
        if want[0] == HP.OK:
            assert got == want and res.n == n, (got, want)
        else:
            assert res.outcome == want[0], (got, want)
        if res.outcome == HP.OK:
            self.reserved |= {res.first_ticket + k for k in range(n)}
            if step.flags & HP.PUT:
                ext_off, first_ext = 0, True
                for k in range(n):
                    typ, conn, ln, _, rid, co = reqs[req0 + k]
                    typ, ln = HP.written(typ, ln)
                    xb = HP.ext_bytes(typ, ln)
                    pos = res.pos + ext_off if xb else None
                    self.puts.append((res.first_ticket + k, pos, int(bool(xb and first_ext and res.wrap)), typ, conn,
                                      rid, co, ln))
                    if xb:
                        first_ext = False
                    ext_off += xb
        return got

    def check_bytes(self):
        """every slot and payload byte: the slot writer's bytes where a put wrote, guard bytes everywhere else"""
        W = HP.writer()
        es, ep = self.guard_slots.copy(), self.guard_pay.copy()
        care_s = np.ones(self.S * 128, dtype=bool)
        care_p = np.ones(self.R, dtype=bool)
        for t, pos, wrap, typ, conn, rid, co, ln in self.puts:
            cmd = self.cmds[co:co + ln] if ln else np.zeros(1, dtype=np.uint8)
            nb = W.sw_put(es.ctypes.data, self.S, ep.ctypes.data, t, 0 if pos is None else pos, wrap, typ, conn, rid,
                          cmd.ctypes.data, ln)
            s0 = 128 * ((t - 1) % self.S)
            care_s[s0:s0 + 128] = False
            for a, b in ((0, 16), (48, 64), (112, 128)):
                care_s[s0 + a:s0 + b] = True
            if pos is None:
                for i in range(nb):
                    care_s[s0 + (16 + i if i < 32 else 32 + i)] = True
            else:
                care_p[pos + nb:pos + HP.round16(nb)] = False
        gs, gp = self.d_slots.cpu().numpy(), self.d_pay.cpu().numpy()
        bad = np.nonzero((gs != es) & care_s)[0]
        assert not len(bad), f"slot bytes differ at {bad[:16].tolist()} (slot {bad[0] // 128}, byte {bad[0] % 128})"
        bad = np.nonzero((gp != ep) & care_p)[0]
        assert not len(bad), f"payload bytes differ at {bad[:16].tolist()}"


def res_step(n, req0=0, ext=HP.EXT_OF_REQUESTS, put=True, timeout=SECOND):
    return HP.Step(HP.RESERVE, n, req0, HP.PUT if put else 0, ext, timeout, 0)


def pub_step(timeout=SECOND):
    return HP.Step(HP.PUBLISH, 0, 0, 0, 0, timeout, 0)


def wait_step(ticket, timeout=SECOND):
    return HP.Step(HP.WAIT, 0, 0, 0, 0, timeout, ticket)


def req(typ, ln, co=0, conn=3, rid=None):
    return (typ, conn, ln, 0, rid if rid is not None else 1000 + ln + 7 * co, co)


def run_checked(ring, scripts, reqs, threads=32):
    """run single-CTA scripts whose reserves the model predicts step by step"""
    outs = ring.run(scripts, reqs, threads)
    got = []
    for sc, oc in zip(scripts, outs):
        for st, o in zip(sc, oc):
            got.append(ring.expect(o, st, reqs) if st.op == HP.RESERVE else (o.outcome,))
    return got


@pytest.fixture(scope="module", params=RINGS, ids=["R2^17", "R33x4096"])
def ring(request, probe):
    return Ring(64, request.param)


def test_submitter_reserve_bounds(ring):
    """NEVER_FITS for n = 0, n = S + 1 and ext = R + 1; on an empty ring n = S and ext = R are OK -- the latter a
    reservation of requests whose images fill the whole payload ring, from 0"""
    S, R = ring.S, ring.R
    ring.setup(1000, 3 * R + 4096 + 48)
    got = run_checked(ring, [[res_step(0, ext=0, put=False), res_step(S + 1, ext=0, put=False),
                              res_step(1, ext=R + 1, put=False), res_step(S, ext=0, put=False)]], [])
    assert [g[0] for g in got] == [HP.NEVER_FITS] * 3 + [HP.OK]
    assert ring.state()["submitted"] == 1000 + S
    lens = [65534, 65534] + ([4094] if R % 65536 else [])
    reqs = [req(HP.SEND, ln, co=5 + k) for k, ln in enumerate(lens)]
    assert sum(HP.ext_bytes(HP.SEND, ln) for ln in lens) == R
    ring.setup(1000, 3 * R + 4096 + 48)
    got = run_checked(ring, [[res_step(len(lens)), pub_step()]], reqs)
    assert got[0] == (HP.OK, 1001, 0, 1) and got[1] == (HP.OK,)
    ring.check_bytes()
    st = ring.state()
    assert st["pay_head"] == 4 * R + R and st["doorbell"] == 1000 + len(lens) and st["lock"] == 0


def test_submitter_ring_end(ring):
    """a reservation that ends exactly at R, then one that starts the ring anew at 0 (WRAP); one whose image is one byte
    too long to end at R skips to 0 (WRAP), and so does a raw reservation one byte over"""
    R = ring.R
    head = 5 * R - 4096
    reqs = [req(HP.SEND, 4094, co=3), req(HP.CSM, 200, co=9), req(HP.SEND, 4095, co=1)]
    ring.setup(50, head)
    got = run_checked(ring, [[res_step(1, 0), pub_step(), res_step(1, 1), pub_step()]], reqs)
    assert got[0] == (HP.OK, 51, R - 4096, 0) and got[2] == (HP.OK, 52, 0, 1)
    ring.check_bytes()
    ring.setup(50, head)
    got = run_checked(ring, [[res_step(1, 2), pub_step(), res_step(1, ext=16, put=False)]], reqs)
    assert got[0] == (HP.OK, 51, 0, 1) and got[2] == (HP.OK, 52, 4112, 0)
    ring.check_bytes()
    ring.setup(50, head)
    got = run_checked(ring, [[res_step(1, ext=4097, put=False), res_step(1, ext=4096, put=False)]], [])
    assert got == [(HP.OK, 51, 0, 1), (HP.OK, 52, 4097, 0)]


def test_submitter_wrap_next_survives_an_inline_reservation(ring):
    """wrap_next set (as a device batch or a detach leaves it): an all-inline reservation keeps it, and the next
    reservation's first external image carries WRAP although it is not its request 0; the one after carries none"""
    reqs = [req(HP.SEND, 300, co=2), req(HP.SEND, 120, co=4),                               # A: two external
            req(HP.CSM, 10, co=1), req(HP.SEND, 78, co=3), req(HP.CLOSE, 0),               # B: inline only
            req(HP.CONNECT, 20, co=6), req(HP.SEND, 79, co=7), req(HP.SEND, 200, co=8),    # C: inline, ext, ext
            req(HP.SEND, 500, co=11)]                                                      # D: ext
    ring.setup(200, 2 * ring.R + 1024)
    got = run_checked(ring, [[res_step(2, 0), pub_step()]], reqs)
    assert got[0][3] == 0
    ring.words[3] = 1
    ring.model.wrap_next = 1
    got = run_checked(ring, [[res_step(3, 2), pub_step(), res_step(3, 5), pub_step(), res_step(1, 8), pub_step()]], reqs)
    assert [g[3] for g in got[0::2]] == [0, 1, 0]
    assert [p[2] for p in ring.puts] == [0, 0, 0, 0, 0, 0, 1, 0, 0]
    ring.check_bytes()
    assert ring.state()["wrap_next"] == 0


def test_submitter_rereads_consumed_only_when_full(ring):
    """a full ring whose leader word has moved while the cached count has not: the reserve succeeds through the
    re-read and caches the new count; a ring that is not full keeps its cache"""
    S = ring.S
    ring.setup(1000 + S, 10 * ring.R, consumed=1000, leader=1005)
    reqs = [req(HP.SEND, k, co=k) for k in range(5)]
    got = run_checked(ring, [[res_step(5), pub_step()]], reqs)
    assert got[0] == (HP.OK, 1001 + S, 0, 0)
    assert ring.state()["consumed"] == 1005
    ring.check_bytes()
    ring.setup(1010, 10 * ring.R, consumed=1000, leader=1020)
    got = run_checked(ring, [[res_step(3), pub_step()]], reqs)
    assert got[0][0] == HP.OK and ring.state()["consumed"] == 1000


def test_submitter_full_ring_times_out_unchanged(ring):
    """a full slot ring, and then a full payload ring, whose leader word has not moved: TIMED_OUT, with submitted,
    pay_head, pay_end, the cache and the lock as they were"""
    S, R = ring.S, ring.R
    for kw, ext in ((dict(submitted=1000 + S, head=7 * R, consumed=1000), 0),
                    (dict(submitted=1010, head=7 * R, consumed=1000, tail=6 * R + 32), 48)):
        ring.setup(**kw)
        before, pe = ring.state(), ring.pay_end.cpu().clone()
        out = ring.run([[res_step(1, ext=ext, put=False, timeout=SHORT)]], [])
        assert out[0][0].outcome == HP.TIMED_OUT
        assert ring.state() == before and bool((ring.pay_end.cpu() == pe).all())
        ring.check_bytes()


def test_submitter_stopped(ring):
    """the stop word no longer holds stop_epoch: a reserve on a full ring, a publish whose turn never comes and a wait
    for a ticket not committed all end STOPPED; commit waits end OK at or below the committed word, and TIMED_OUT
    above it while the stop word holds its epoch"""
    S = ring.S
    ring.setup(1000 + S, 0, consumed=1000, stop=EPOCH + 1)
    assert ring.run([[res_step(1, ext=0, put=False, timeout=60 * SECOND)]], [])[0][0].outcome == HP.STOPPED
    ring.setup(1000, 0, doorbell=999, committed=990, stop=EPOCH + 1)
    out = ring.run([[res_step(1, ext=0, put=False), pub_step(60 * SECOND), wait_step(990), wait_step(991, 60 * SECOND)]],
                   [])[0]
    assert [o.outcome for o in out] == [HP.OK, HP.STOPPED, HP.OK, HP.STOPPED]
    assert ring.state()["doorbell"] == 999
    ring.setup(1000, 0, committed=990)
    out = ring.run([[wait_step(989), wait_step(991, SHORT)]], [])[0]
    assert [o.outcome for o in out] == [HP.OK, HP.TIMED_OUT]


def test_submitter_lengths_types_and_alignments(ring):
    """cmd lengths 77..80 (the inline limit), 65535, 65536 and 70000; types 0, 2, 3 and 9, which become counted NOOPs
    as the cmds above 65535 B do; cmd pointers at every alignment mod 16"""
    reqs = [req(HP.SEND, ln, co=3 + ln) for ln in (77, 78, 79, 80)]
    reqs += [req(HP.SEND, 65535, co=1), req(HP.SEND, 65536, co=2), req(HP.SEND, 70000, co=0)]
    reqs += [req(t, ln, co=5) for t in (0, 2, 3, 9) for ln in (0, 10, 200)]
    reqs += [req((HP.CSM, HP.CONNECT, HP.SEND, HP.CLOSE)[a % 4], 40 + 37 * a, co=1024 + a) for a in range(16)]
    ring.setup(300, 11 * ring.R + 512)
    got = run_checked(ring, [[res_step(7, 0), pub_step(), res_step(len(reqs) - 7, 7), pub_step()]], reqs, threads=8)
    assert got[0][0] == HP.OK and got[2][0] == HP.OK
    rejected = [t for t, r in zip(range(301, 301 + len(reqs)), reqs) if not HP.accepted(r[0], r[2])]
    st = ring.state()
    assert st["rejected"] == len(rejected) == 14 and st["first_rejected"] == min(rejected) == 306
    assert st["doorbell"] == 300 + len(reqs)
    ring.check_bytes()


def multi_scripts(rng, ctas, per, reqs, hold=None):
    scripts = []
    for b in range(ctas):
        sc = []
        for r in range(per):
            n = int(rng.integers(1, 9))
            req0 = len(reqs)
            for _ in range(n):
                typ = int(rng.choice([HP.SEND, HP.SEND, HP.CSM, HP.CONNECT, HP.CLOSE, 0, 9]))
                ln = int(rng.integers(0, 300))
                reqs.append(req(typ, ln, co=int(rng.integers(0, 1 << 17)), conn=int(rng.integers(0, 9)),
                                rid=len(reqs) + 1))
            sc.append(res_step(n, req0))
            if (b, r) != hold:
                sc.append(pub_step(20_000_000 if hold else SECOND))
        scripts.append(sc)
    return scripts


@pytest.mark.parametrize("R", RINGS)
def test_submitter_many_ctas(probe, R):
    """eight CTAs reserve, put and publish at once, across the payload ring's end: the tickets partition the range, the
    publishes happen in ticket order and the doorbell ends at the last ticket, the reservations are the model's in ticket
    order, consecutive external images are contiguous unless the later one carries WRAP, the rejections are counted
    with the lowest rejected ticket, and every byte is the slot writer's"""
    ring = Ring(1024, R, seed=11)
    rng = np.random.default_rng(R)
    reqs = []
    scripts = multi_scripts(rng, 8, 4, reqs)
    s0 = 5000
    ring.setup(s0, 6 * R - 3008)
    outs = ring.run(scripts, reqs, threads=64)
    done = []
    for sc, oc in zip(scripts, outs):
        for st, o in zip(sc, oc):
            assert o.outcome == HP.OK, (st.op, o.outcome)
            if st.op == HP.RESERVE:
                done.append((o.first_ticket, st, o))
            else:
                done[-1] += (o.order,)
    done.sort(key=lambda d: d[0])
    total = sum(st.n for _, st, _, _ in done)
    assert [d[0] for d in done] == list(np.cumsum([s0 + 1] + [st.n for _, st, _, _ in done[:-1]]))
    assert [d[3] for d in done] == list(range(len(done)))
    for _, st, o, _ in done:
        ring.expect(o, st, reqs)
    st = ring.state()
    assert st["doorbell"] == st["submitted"] == s0 + total and st["lock"] == 0
    ext = [(p[1], HP.ext_bytes(p[3], p[7]), p[2]) for p in sorted(ring.puts) if p[1] is not None]
    wraps = 0
    for (pa, xa, _), (pb, xb, wb) in zip(ext, ext[1:]):
        assert wb or pb == pa + xa, (pa, xa, pb)
        wraps += wb
    assert wraps >= 1
    rej = [first + k for first, st_, _, _ in done for k in range(st_.n)
           if not HP.accepted(reqs[st_.req0 + k][0], reqs[st_.req0 + k][2])]
    assert st["rejected"] == len(rej) > 0 and st["first_rejected"] == min(rej)
    ring.check_bytes()


def test_submitter_held_reservation(probe):
    """a reservation reserved and put but never published holds back every later one: their publishes end TIMED_OUT and
    the doorbell stays at the held reservation's first ticket - 1; earlier ones publish (one CTA, then eight)"""
    ring = Ring(1024, 1 << 17, seed=12)
    reqs = [req(HP.SEND, 10 * k, co=k) for k in range(12)]
    ring.setup(100, 0)
    out = ring.run([[res_step(3, 0), pub_step(), res_step(3, 3), res_step(3, 6), pub_step(SHORT)]], reqs)[0]
    assert [o.outcome for o in out] == [HP.OK, HP.OK, HP.OK, HP.OK, HP.TIMED_OUT]
    assert ring.state()["doorbell"] == 103
    rng = np.random.default_rng(3)
    reqs = []
    scripts = multi_scripts(rng, 8, 3, reqs, hold=(0, 1))
    ring.setup(100, 0)
    outs = ring.run(scripts, reqs, threads=32)
    held = outs[0][2].first_ticket
    pubs = []
    for sc, oc in zip(scripts, outs):
        last = None
        for st, o in zip(sc, oc):
            if st.op == HP.RESERVE:
                assert o.outcome == HP.OK
                last = o.first_ticket
            else:
                pubs.append((last, o.outcome))
    assert pubs and all((oc == HP.OK) == (t < held) for t, oc in pubs), (held, sorted(pubs))
    assert any(oc == HP.TIMED_OUT for _, oc in pubs)
    assert ring.state()["doorbell"] == held - 1


# ---------------------------------------------------------------------------------
# one end-to-end leg: a payload ring whose size is not a power of two
# ---------------------------------------------------------------------------------
def test_ring_of_33_pages_laps_with_every_writer(eng, orc):
    """ring_bytes = 33 * 4096 and APUS_F_AUTOPRUNE: host batches, packed device batches and a resident submitter take
    turns until the payload ring has lapped several times; every byte of every replica is the oracle's replay"""
    import torch
    import streams as S
    n, L, R = 3, 1 << 18, 33 * 4096
    flags = MODES["index_earlyack"] | E.F_AUTOPRUNE
    SB.lib()
    rp = AR.Replay(orc, n, L)
    try:
        with eng.Group(n, devices=devices_for(eng, n), log_size=L, flags=flags, leader_ctas=4, ring_mode=eng.RING_DEVICE,
                       ring_slots=1 << 11, ring_bytes=R) as g:
            g.prologue()
            ordered, prev, ext, rid = [(O.CONFIG, 0, 0, b"")], 0, 0, 1 << 20
            st = torch.cuda.Stream(device=g.leader.device)
            for rnd in range(6):
                host = S.ragged_stream(120, 600, conns=3, seed=300 + rnd)
                dev = S.ragged_stream(120, 600, conns=3, seed=400 + rnd)
                sub = SB.mixed_requests(200, seed=500 + rnd, max_len=600, reject_every=37, conns=3, first_req_id=rid)
                rid += len(sub)
                submit_host(g, host)
                g.submit_device_packed(*_packed(dev, g.leader.device))
                g.run()
                ordered += host + dev
                end = g.leader.offsets()["end"]
                rp.launch(AR.read_launch(g.leader, prev, end, L), ordered)
                prev = end
                v = g.leader.submitter_attach(st)
                s = SB.Submitter(v, st, sub, batch=16, ctas=4, timeout_s=30.0)
                g.tickets += len(sub)
                g.launch()
                s.start()
                fail, pub, tickets = s.result()
                assert fail is None and pub == len(sub), (fail, pub)
                g.wait(60_000)
                g.leader.submitter_detach()
                part = SB.ticket_order(sub, tickets)[0]
                ordered += part
                ext += sum(HP.round16(len(p) + 2) for _, _, _, p in host + dev + part if len(p) + 2 > 80)
                end = g.leader.offsets()["end"]
                rp.launch(AR.read_launch(g.leader, prev, end, L), ordered)
                prev = end
                check_heads(g.replicas, rp, f"after round {rnd}")
            assert rp.pos == len(ordered) and ext >= 4 * R and rp.written >= 2 * L
            EU.compare_group_to_oracle(g, rp.c, exact=True)
            assert g.leader.stats()["auto_heads"] == len(rp.heads) > 0
            assert g.leader.committed() == len(ordered)
    finally:
        rp.close()


def _packed(part, device):
    import torch
    offs = np.concatenate([[0], np.cumsum([len(p) for *_, p in part])]).astype(np.int64)
    vals = np.frombuffer(b"".join(p for *_, p in part) + b"\0", dtype=np.uint8)
    dev = torch.device("cuda", device)
    return (torch.from_numpy(np.array([t for t, *_ in part], dtype=np.uint8)).to(dev),
            torch.from_numpy(np.array([c for _, c, _, _ in part], dtype=np.uint16).view(np.int16)).to(dev),
            torch.from_numpy(np.array([r for _, _, r, _ in part], dtype=np.uint64).view(np.int64)).to(dev),
            torch.from_numpy(offs).to(dev), torch.from_numpy(vals[:max(int(offs[-1]), 1)].copy()).to(dev))
