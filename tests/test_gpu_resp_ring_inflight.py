"""The RESP ring driven as a server drives it, against ONE oracle store and no other GPU decision.

A server keeps several slots in flight: while slot j's replies are formatted on the out stream, slot j+1's
connections are parsed on the in stream, and stage 2 of its batch may overlap the residue tail of slot j's batch
behind PEND bits (over a segmented batch view, since a RESP batch's row count exists only on the device).  Here every
submit's expected outcome is computed on the host before it is submitted: for each connection in table order,
gcra_resp_parse_throttle at the row cap the connections before it leave (the header's contract) gives the rows,
consumed, n_frames and stop; the rows are appended, in submission order, to one sequence that one oracle store
replays; the expected replies are gcra_resp_format_replies of those rows and the oracle's results.  After each wait
the outcome (with reply_off and reply_len), the reply bytes and the slot's rows and results must be bit-exact.

A RESP batch always takes the index-order pipeline: plan_pipelined sends every batch over a view of more than one
segment there, and the adaptive switch and GCRA_INDEX_MIN only act on single-segment batches.  So these tests pin
k1_path to "auto"; "index" and "sort" would run the same kernels.

The engine statistics asserted on (index_batches, residue_rows, drains, grows, purges) prove that the machinery
under test was really exercised."""
import ctypes as C
from collections import deque

import numpy as np
import pytest

import oracle
import throttlecrab_b200 as tc
from throttlecrab_b200.resp import RespError, RespParser, RespSerializer, _plan_command, _throttle_reply
from test_gpu_pipelined_runs import assert_counters
from test_resp import _cmd, _raw_throttle

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000 * 10**9
MS = 1_000_000
SIP = (0x0706050403020100, 0x0f0e0d0c0b0a0908)
SEEDS = pytest.mark.parametrize("seed", [(0, 0), SIP], ids=["unkeyed", "siphash"])
AUTO = pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
MIN_FRAME = 45                          # gcra_resp::MIN_FRAME_BYTES: the submit's row bound is sum(len // 45)
PING = _cmd("PING")


def geometry(row_capacity):
    """gcra_resp_ring_create's view of a slot: nseg segments of 2^shift rows,
    shift = max(10, ceil_log2(ceil(row_capacity / 16))), nseg = max(2, ceil(row_capacity / 2^shift))"""
    shift = max(10, (-(-row_capacity // 16) - 1).bit_length())
    return shift, max(2, -(-row_capacity // (1 << shift)))


def host_parse(lim, seg, now, cap):
    req = np.zeros(max(1, min(cap, len(seg) // MIN_FRAME + 1)), tc.REQ_DTYPE)
    used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
    assert lim._L.gcra_resp_parse_throttle(lim._h, seg, len(seg), now, cap, req.ctypes.data, C.byref(used),
                                           C.byref(cnt), C.byref(stop)) == 0
    return req[:cnt.value], used.value, cnt.value, stop.value


def format_replies(lim, req, res):
    buf = C.create_string_buffer(max(len(req), 1) * tc.RESP_REPLY_MAX)
    w = lim._L.gcra_resp_format_replies(req.ctypes.data, res.ctypes.data, len(req), buf, len(buf))
    return buf.raw[:w]


class Server:
    """A RespRing and the host reference of everything it does: `expected` per slot in flight, one oracle store fed
    every decision in the order the engine makes them, and the keys seen (their hashes must be distinct)."""

    def __init__(self, lim, ring, ora):
        self.lim, self.ring, self.ora = lim, ring, ora
        self.rows, self.res = [], []               # every decision, in order
        self.pending = {}
        self.batches = 0                           # submits whose row bound is above 0: one pipelined batch each
        self.keys = {}                             # key hash -> key bytes

    def note_key(self, kb):
        h = self.lim.store.hash_key(kb)
        assert self.keys.setdefault(h, kb) == kb, "two keys of the trace share a key hash"
        return h

    def decide(self, rows):
        """the oracle's results of rows the engine decides next"""
        o = np.zeros(len(rows), oracle.REQ_DTYPE)
        o["key"] = rows["key_hash"]
        for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
            o[f] = rows[f]
        res = self.ora.replay(o).view(tc.RES_DTYPE)
        self.rows.append(rows)
        self.res.append(res)
        return res

    def submit(self, slot, segs, now, offsets=None):
        ring = self.ring
        inp = ring.input[slot]
        if offsets is None:                        # gaps of 0 .. 15 bytes: every residue mod 16 shows up
            offsets, at = [], 0
            for c, s in enumerate(segs):
                offsets.append(at)
                at += len(s) + c % 16
        for c, (s, off) in enumerate(zip(segs, offsets)):
            inp[off:off + len(s)] = np.frombuffer(s, np.uint8)
            ring.conns[slot][c] = (off, len(s))
        outs, rows, base = [], [], 0
        for s in segs:
            r, used, cnt, stop = host_parse(self.lim, s, now, ring.row_capacity - base)
            outs.append((used, cnt, stop))
            rows.append(r)
            base += cnt
        want = np.concatenate(rows) if rows else np.zeros(0, tc.REQ_DTYPE)
        res = self.decide(want)
        replies, b = [], 0
        for _, cnt, _ in outs:
            replies.append(format_replies(self.lim, want[b:b + cnt], res[b:b + cnt]) if cnt else b"")
            b += cnt
        self.batches += sum(len(s) // MIN_FRAME for s in segs) > 0
        ring.submit(slot, len(segs), now)
        self.pending[slot] = (outs, want, res, replies)
        return outs

    def wait(self, slot):
        ring = self.ring
        ring.wait(slot)
        outs, want, res, replies = self.pending.pop(slot)
        got = ring.outcome[slot][:len(outs)]
        lens = np.array([len(r) for r in replies], np.uint64)
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64) if len(lens) else lens
        exp = np.zeros(len(outs), tc.RESP_OUTCOME_DTYPE)
        if len(outs):
            exp["consumed"], exp["n_frames"], exp["stop"] = np.array(outs).T
        exp["reply_off"], exp["reply_len"] = offs, lens
        bad = np.nonzero(got != exp)[0]
        assert len(bad) == 0, "connection %d: %s != %s" % (bad[0], got[bad[0]], exp[bad[0]])
        # (comparisons outside `assert`: pytest's diff of megabytes would take minutes)
        total = int(lens.sum())
        same = ring.replies[slot][:total].tobytes() == b"".join(replies)
        assert same, "reply bytes differ"
        rows, rres = ring.rows(slot)
        same = len(rows) == len(want) and rows.tobytes() == want.tobytes()
        assert same, "rows differ: %d rows, %d expected" % (len(rows), len(want))
        if rres.tobytes() != res.tobytes():
            i = int(np.nonzero(rres != res)[0][0])
            raise AssertionError("row %d of %d: engine %s, oracle %s, row %s" % (i, len(res), rres[i], res[i], rows[i]))
        return outs

    def blocking(self, kb, b, c, p, q, now):
        """a THROTTLE the general parser took (RESP-integer arguments): decided on its own by a blocking
        rate_limit_batch, which orders itself after the RESP batches still in flight"""
        row = np.zeros(1, tc.REQ_DTYPE)
        row[0] = (self.note_key(kb), b, c, p, q, now)
        got = self.lim.rate_limit_batch(row)
        want = self.decide(row)
        assert got.tobytes() == want.tobytes(), (got, want, row)
        return RespSerializer.serialize(_throttle_reply(got[0], b, q))

    def all_results(self):
        return np.concatenate(self.res) if self.res else np.zeros(0, tc.RES_DTYPE)

    def check_entries(self, exact_counters=True, require_expired=True):
        st = self.lim.store
        for h in self.keys:
            assert st.peek(h) == self.ora.entry("k:%d" % h), self.keys[h]
        if exact_counters:
            assert_counters(st, self.all_results().view(oracle.RES_DTYPE), self.ora, require_expired)


class Conn:
    """One client connection: a stream of frames, read in pieces of any size (frames split anywhere), and the bytes
    the server still holds for it (what it has not consumed, carried to its next submit)."""

    def __init__(self, frames):
        self.frames = frames                      # callable -> the next frame
        self.out = deque()                        # frames not yet read; out[0] may be the rest of a split one
        self.split = False
        self.buf = b""

    def read(self, n):
        n = min(n, tc.RESP_MAX_CONN_BYTES - len(self.buf))
        got = []
        while n > 0:
            if not self.out:
                self.out.append(self.frames())
                self.split = False
            f = self.out.popleft()
            if len(f) > n:
                self.out.appendleft(f[n:])
                f = f[:n]
                self.split = True
            else:
                self.split = False
            got.append(f)
            n -= len(f)
        self.buf += b"".join(got)
        return self.buf

    def close(self):
        """after a protocol error: the connection ends, and a new one starts at the next whole frame"""
        self.buf = b""
        if self.split:
            self.out.popleft()
            self.split = False


def serve_stop2(srv, conn, now, parser=RespParser()):
    """the ONE frame at the start of conn.buf that is not a plain THROTTLE, as a server's general parser handles it"""
    try:
        r = parser.parse(conn.buf)
    except RespError:
        conn.close()
        return "closed"
    if r is None:
        return "incomplete"
    conn.buf = conn.buf[r[1]:]
    plan = _plan_command(r[0])
    if plan[0] == "throttle":
        srv.blocking(plan[1].encode(), plan[2], plan[3], plan[4], plan[5], now)
        return "throttle"
    return "reply"


def run_paced(srv, groups, n_submits, read_size, clock, rng, at_boundary=None):
    """Submit n_submits times, slot t % S taking connection group t % S, paced like ring_run: after submitting t,
    wait for t - S + 1 and serve its connections' frames that stop 2 -- while the slots after it are in flight."""
    S = len(groups)
    counts = {"stop3": 0, "stop1": 0, "blocking": 0, "closed": 0}
    now = [T0]

    def collect(j):
        outs = srv.wait(j % S)
        for conn, (_, _, stop) in zip(groups[j % S], outs):
            counts["stop3"] += stop == 3
            counts["stop1"] += stop == 1
            if stop == 2:
                what = serve_stop2(srv, conn, now[0])
                counts["blocking"] += what == "throttle"
                counts["closed"] += what == "closed"

    for t in range(n_submits):
        now[0] = clock(t, now[0])
        if at_boundary is not None:
            at_boundary(t, now[0])
        g = groups[t % S]
        segs = [c.read(read_size(rng)) for c in g]
        outs = srv.submit(t % S, segs, now[0])
        for c, (used, _, _) in zip(g, outs):
            c.buf = c.buf[used:]
        if t - S + 1 >= 0:
            collect(t - S + 1)
    for j in range(max(n_submits - S + 1, 0), n_submits):
        collect(j)
    return counts


# ---------------------------------------------------------------------------------------------------------------
# scenario 1: slots in flight on shared keys
# ---------------------------------------------------------------------------------------------------------------
HOT = (20, 50, 1)                  # 20 ms per token: the hot key changes state now and then, at every clock step
SPEND = (100, 1000, 60)            # fresh keys that spend a burst: every allowed row changes the state (residue)
TOGGLE = (1, 3, 3600)              # max_burst = 1, q = 0: the state toggles on every row, from tail to tail
COLD = (2, 10, 1)                  # entries expire 200 ms after their last allowed row: expired writes


def shared_key_frames(srv, rng, phase):
    """frames of every connection: the hot key, the current burst spenders (phase[0] moves on), the toggler, cold
    keys; a few with quantity -1, and a few frames that are not plain (PING, unknown, RESP-integer THROTTLE,
    garbage that closes the connection)"""
    cache = {}

    def frame(kb, pol, q):
        k = (kb, pol, q)
        f = cache.get(k)
        if f is None:
            srv.note_key(kb)
            f = cache[k] = _raw_throttle(kb, *pol, q)
        return f

    def nxt():
        u = rng.random()
        if u < 0.25:
            return frame(b"hot", HOT, 1)
        if u < 0.25 + phase[1]:
            return frame(b"spend:%d" % (phase[0] * 8 + int(rng.integers(0, 8))), SPEND, 1)
        if u < 0.27 + phase[1]:
            return frame(b"toggle", TOGGLE, 0)
        if u < 0.9996:          # (rare enough that most batches follow a pipelined batch, not a blocking one)
            kb = b"cold:%d" % int(rng.integers(0, 3000))
            q = int(rng.choice([1, 1, 1, 2, 0, -1])) if rng.random() < 0.1 else 1
            return frame(kb, COLD, q)
        v = rng.random()
        if v < 0.4:
            return PING
        if v < 0.6:
            return _cmd("UNKNOWN", "x")
        if v < 0.9:
            kb = b"hot" if rng.random() < 0.5 else b"cold:%d" % int(rng.integers(0, 3000))
            srv.note_key(kb)
            return _cmd("THROTTLE", kb.decode(), *COLD, 1)
        return b"?garbage\r\n"
    return nxt


def phase_clock(rng):
    def clock(t, now):
        return now + int(rng.choice([0, 0, 1 * MS, 7 * MS, 30 * MS, 250 * MS]))
    return clock


@AUTO
@SEEDS
@pytest.mark.parametrize("slots", [2, 3, 4])
def test_slots_in_flight_on_shared_keys(slots, seed, k1_path):
    """A few hundred submits, each slot with its own connection group (a connection is never in two slots in flight),
    the groups sharing every key: the parse of slot j+1 overlaps the replies of slot j, stage 2 of its batch overlaps
    slot j's residue tail, the drains fire, and blocking calls for the general parser's THROTTLEs order themselves
    after the slots in flight.  The row cap is below what a group holds, so stop 3 is frequent."""
    rng = np.random.default_rng(31 + slots)
    cap, n_conns, n_submits = 2048, 48, 240
    lim = tc.RateLimiter(tc.ManualStore(capacity=50_000, created_ns=T0, max_batch=cap, hash_seed=seed))
    per = n_conns // slots
    ring = tc.RespRing(lim, slots, per, per * (tc.RESP_MAX_CONN_BYTES + 16), cap)
    srv = Server(lim, ring, oracle.OracleStore(oracle.PERIODIC, capacity=50_000, created_ns=T0, p0=10**9))
    phase = [0, 0.3]
    frames = shared_key_frames(srv, rng, phase)
    conns = [Conn(frames) for _ in range(n_conns)]
    groups = [conns[g::slots] for g in range(slots)]
    mean = int(1.3 * cap * 52 / per)              # a group's reads hold ~1.3 row caps of frames

    def boundary(t, now):
        if t % 6 == 0:
            phase[0] += 1                         # new spenders; the share moves the residue across 1/8 and 1/4
            phase[1] = float(rng.choice([0.02, 0.1, 0.3, 0.5]))

    counts = run_paced(srv, groups, n_submits, lambda r: int(r.integers(0, 2 * mean)), phase_clock(rng), rng,
                       boundary)
    srv.check_entries()
    s = lim.store.stats()
    print("%d slots: %s %s" % (slots, counts, {f: s[f] for f in ("index_batches", "residue_rows", "drains")}))
    assert s["index_batches"] == srv.batches and s["residue_rows"] > 0, s
    assert 0 < s["drains"] < s["index_batches"] - 1, s
    assert counts["stop3"] > n_submits // 4 and counts["stop1"] > 0 and counts["blocking"] > 0 and counts["closed"] > 0


# ---------------------------------------------------------------------------------------------------------------
# scenario 2: a tight table grows and purges while slots are in flight
# ---------------------------------------------------------------------------------------------------------------
def arriving_frames(srv, rng, t_now):
    """keys arrive progressively (the id range grows with the submit count), and fresh keys asked for more than
    their burst are only ever denied: they take a slot and leave no entry, which a purge gives back"""
    def nxt():
        u = rng.random()
        if u < 0.05:
            kb = b"deny:%d" % int(rng.integers(0, 1 << 40))
            srv.note_key(kb)
            return _raw_throttle(kb, *COLD, 5)
        if u < 0.06:
            return PING
        kb = b"a:%d" % int(rng.integers(0, 40 + 60 * t_now[0]))
        srv.note_key(kb)
        return _raw_throttle(kb, *COLD, int(rng.choice([0, 1, 1, 1, 2])))
    return nxt


@AUTO
@pytest.mark.parametrize("store", ["manual", "periodic"])
def test_tight_table_grows_and_purges_with_slots_in_flight(store, k1_path):
    """GCRA_FLAG_TIGHT_TABLE from 16 entries: the table grows (sized from each submit's byte bound, not its real
    row count) and purges between submits while other slots are in flight.  With the ManualStore, sweeps at some
    boundaries run on both sides; the PeriodicStore sweeps by itself at submits when the counters are ready, which
    the timing decides, so only what sweeps cannot change is compared: rows and results, then len and entries after
    one final sweep of both."""
    rng = np.random.default_rng(41)
    cap, slots, per, n_submits = 1024, 3, 6, 150
    cls = tc.ManualStore if store == "manual" else tc.PeriodicStore
    st = cls(capacity=16, created_ns=T0, max_batch=cap, flags=tc._native.FLAG_TIGHT_TABLE, p0=1)
    lim = tc.RateLimiter(st)
    ring = tc.RespRing(lim, slots, per, per * (tc.RESP_MAX_CONN_BYTES + 16), cap)
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=16, created_ns=T0, p0=10**9)
    srv = Server(lim, ring, ora)
    t_now = [0]
    frames = arriving_frames(srv, rng, t_now)
    groups = [[Conn(frames) for _ in range(per)] for _ in range(slots)]
    swept = []

    def boundary(t, now):
        t_now[0] = t
        if store == "manual" and t % 10 == 9:
            swept.append((st.sweep(now), ora.force_sweep(now)))

    def clock(t, now):
        return now + int(rng.choice([0, 2 * MS, 90 * MS, 700 * MS]))

    run_paced(srv, groups, n_submits, lambda r: int(r.integers(0, 9000)), clock, rng, boundary)
    s = st.stats()
    print("%s: %s" % (store, {f: s[f] for f in ("grows", "purges", "sweeps", "len", "index_batches", "drains")}))
    assert s["grows"] > 0 and s["purges"] > 0, s
    if store == "manual":
        assert all(a == b for a, b in swept) and sum(a for a, _ in swept) > 0, swept
        srv.check_entries()
    else:
        assert s["sweeps"] > 0, s
        last = int(np.concatenate(srv.rows)["now_ns"].max())
        st.sweep(last)
        ora.force_sweep(last)
        assert st.len() == ora.len()
        srv.check_entries(exact_counters=False)


# ---------------------------------------------------------------------------------------------------------------
# scenario 3: every view geometry, and totals on the batch edges
# ---------------------------------------------------------------------------------------------------------------
# row capacity -> (shift, nseg) by the formula in `geometry`: 1 .. 1,025 rows view 2 x 2^10 (ceil(1025 / 16) = 65
# still gives shift 10); 16,384 -> 16 x 2^10; 16,385 -> 9 x 2^11 (ceil(16385 / 16) = 1,025 rounds up to 2^11);
# 131,073 -> 9 x 2^14; 2^20 -> 16 x 2^16.
GEOMETRIES = {1: (10, 2), 255: (10, 2), 256: (10, 2), 257: (10, 2), 1023: (10, 2), 1024: (10, 2), 1025: (10, 2),
              16384: (10, 16), 16385: (11, 9), 131073: (14, 9), 1 << 20: (16, 16)}
EDGE_KEYS = 5000


def edge_totals(cap):
    """(name, rows, where the cap cuts) of each fill: PINGs only (row bound > 0, no row), 1 row, whole reply tiles,
    one and two whole segments, exactly the cap, and past the cap cut inside a connection and at a boundary"""
    shift, _ = geometry(cap)
    out = [("pings", 0), ("one", 1)]
    out += [("tile%d" % m, 256 * m) for m in sorted({1, cap // 256}) if 0 < 256 * m <= cap]
    out += [("seg%d" % k, k << shift) for k in (1, 2) if k << shift <= cap]
    out += [("cap", cap), ("over-inside", cap + 1 + cap // 3), ("over-boundary", cap + 57)]
    seen = set()
    return [(name, n) for name, n in out if not (n in seen or seen.add(n))]


def edge_fill(rng, pool, name, n, cap):
    """connections of plain frames (sizes 0 .. ~1,000 frames) holding n rows; 'over-boundary' makes the first
    connections hold exactly `cap` rows, 'over-inside' keeps every connection boundary away from it"""
    if name == "pings":
        return [PING * 4, b"", PING * 9]
    sizes, left = [], n
    while left:
        k = min(left, int(rng.integers(0, 1000)))
        if name == "over-boundary" and sum(sizes) < cap < sum(sizes) + k:
            k = cap - sum(sizes)
        if name == "over-inside" and sum(sizes) + k == cap:
            k += 1 if left > k else -1
        sizes.append(k)
        left -= k
    ids = rng.integers(0, len(pool), n)
    segs, at = [], 0
    for k in sizes:
        segs.append(b"".join(pool[i] for i in ids[at:at + k]))
        at += k
    return segs


@AUTO
@pytest.mark.parametrize("cap", list(GEOMETRIES))
def test_view_geometry_and_batch_edges(cap, k1_path):
    """Each row capacity's (shift, nseg) view, filled with totals that end on the kernels' edges: on a 256-row reply
    tile (row + 1 == total, and the tiles past the total), on a segment end (the segment counts of the last
    connection's CTA), at the cap and past it.  Two slots, one in flight while the next is filled."""
    assert geometry(cap) == GEOMETRIES[cap]
    rng = np.random.default_rng(cap)
    lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 16, created_ns=T0, max_batch=max(cap, 4096)))
    fills = edge_totals(cap)
    n_max = max(n for _, n in fills)
    pool = [_raw_throttle(b"e:%d" % i, 5, 10, 60) for i in range(EDGE_KEYS)]
    n_conns = n_max // 250 + 64
    in_cap = n_max * max(len(f) for f in pool) + n_conns * 16 + 4096
    ring = tc.RespRing(lim, 2, n_conns, in_cap, cap)
    srv = Server(lim, ring, oracle.OracleStore(oracle.PERIODIC, capacity=1 << 16, created_ns=T0, p0=10**9))
    for i in range(EDGE_KEYS):
        srv.note_key(b"e:%d" % i)
    now = T0
    for t, (name, n) in enumerate(fills):
        segs = edge_fill(rng, pool, name, n, cap)
        assert len(segs) <= n_conns
        now += 50 * MS
        outs = srv.submit(t % 2, segs, now)
        assert sum(o[1] for o in outs) == min(n, cap), name
        if name.startswith("over"):                  # the first stop 3 took part of its connection, or none of it
            first = next(o for o in outs if o[2] == 3)
            assert (first[1] > 0) == (name == "over-inside"), (name, first)
        if t:
            srv.wait((t - 1) % 2)
    srv.wait((len(fills) - 1) % 2)
    srv.check_entries(require_expired=False)


@AUTO
def test_max_batch_below_the_view_with_a_large_residue(k1_path):
    """max_batch = row_capacity = 300 against a 2 x 2^10 view: the residue tail's n_max and nres_rows are clamped to
    max_batch while the per-row buffers are indexed in view space.  Burst-spending keys put most rows in the
    residue; three slots in flight."""
    rng = np.random.default_rng(300)
    cap = 300
    lim = tc.RateLimiter(tc.ManualStore(capacity=10_000, created_ns=T0, max_batch=cap))
    ring = tc.RespRing(lim, 3, 4, 4 * (tc.RESP_MAX_CONN_BYTES + 16), cap)
    srv = Server(lim, ring, oracle.OracleStore(oracle.PERIODIC, capacity=10_000, created_ns=T0, p0=10**9))
    phase = [0, 0.6]
    frames = shared_key_frames(srv, rng, phase)
    groups = [[Conn(frames) for _ in range(4)] for _ in range(3)]

    def boundary(t, now):
        phase[0] += t % 3 == 0

    run_paced(srv, groups, 120, lambda r: int(r.integers(0, 6000)), phase_clock(rng), rng, boundary)
    srv.check_entries(require_expired=False)
    s = lim.store.stats()
    assert s["index_batches"] == srv.batches and s["residue_rows"] > 120 * cap // 8, s


# ---------------------------------------------------------------------------------------------------------------
# scenario 4: full size
# ---------------------------------------------------------------------------------------------------------------
def zipf_conns(rng, n_conns, size):
    """tools/resp_ring_e2e.py's workload: plain frames over Zipf(1.1) keys of 1 M ids, up to `size` bytes each"""
    segs, used = [], set()
    for _ in range(n_conns):
        ids = np.minimum(rng.zipf(1.1, size // 40 + 1), 1_000_000)
        fr = [b"*5\r\n$8\r\nTHROTTLE\r\n$%d\r\nk:%d\r\n$2\r\n10\r\n$3\r\n100\r\n$2\r\n60\r\n" % (len(b"k:%d" % i), i)
              for i in ids]
        lens = np.cumsum([len(f) for f in fr])
        k = int(np.searchsorted(lens, size, side="right"))
        segs.append(b"".join(fr[:k]))
        used.update(int(i) for i in ids[:k])
    return segs, used


@AUTO
def test_full_size_slots_in_flight(k1_path):
    """row_capacity = max_batch = 2^20 (a 16 x 2^16 view): 4,096 connections of ~10 KiB and 256 of 64 KiB, two
    slots in flight, every row against the oracle"""
    rng = np.random.default_rng(2020)
    cap = 1 << 20
    lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 21, created_ns=T0, max_batch=cap))
    ring = tc.RespRing(lim, 2, 4096, 4096 * (10240 + 16), cap)
    srv = Server(lim, ring, oracle.OracleStore(oracle.PERIODIC, capacity=1 << 21, created_ns=T0, p0=10**9))
    all_ids, now, t = set(), T0, 0
    for n_conns, size in ((4096, 10240), (256, 65536)):
        for _ in range(3):
            segs, ids = zipf_conns(rng, n_conns, size)
            all_ids |= ids
            now += 3 * MS
            srv.submit(t % 2, segs, now)
            if t:
                srv.wait((t - 1) % 2)
            t += 1
    srv.wait((t - 1) % 2)
    ids = np.array(sorted(all_ids), np.uint64)
    hashes = tc.hash_key_ids(ids)
    assert len(np.unique(hashes)) == len(ids)
    srv.keys = {int(h): b"k:%d" % int(i) for h, i in zip(hashes[::61], ids[::61])}   # entries of a sample of keys
    srv.check_entries(require_expired=False)
    assert sum(len(r) for r in srv.rows) > 2_000_000


# ---------------------------------------------------------------------------------------------------------------
# scenario 5: 65,536 connections in one submit
# ---------------------------------------------------------------------------------------------------------------
@AUTO
@SEEDS
def test_65536_connections_in_one_submit(seed, k1_path):
    """max_conns = 65,536: 65,536 parse CTAs through the ticket look-back and 256 outcome blocks.  Most connections
    are empty or hold one frame; a few hold 64 KiB or end inside a frame; their offsets cover every residue mod 16,
    and the last one ends exactly at in_capacity."""
    rng = np.random.default_rng(65536)
    n = 65536
    lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 17, created_ns=T0, max_batch=1 << 16, hash_seed=seed))
    keys = [b"c:%d" % i for i in range(20_000)]
    one = [_raw_throttle(k, 3, 10, 60) for k in keys]
    full = b"".join(one[i] for i in range(1500))
    segs = []
    for c in range(n):
        u = rng.random()
        if c % 8192 == 77:
            segs.append(full[:65536])                                   # 64 KiB, cut inside a frame
        elif c % 8192 == 78:
            f = one[c % 20_000]
            segs.append(f * (65536 // len(f)))                          # whole frames up to 64 KiB
        elif u < 0.5:
            segs.append(b"")
        elif u < 0.97:
            segs.append(one[int(rng.integers(0, 20_000))])
        elif u < 0.99:
            f = one[int(rng.integers(0, 20_000))]
            segs.append(f[:int(rng.integers(1, len(f)))])               # a frame cut anywhere: stop 1
        else:
            segs.append(PING + one[int(rng.integers(0, 20_000))])       # stop 2 at once
    segs[-1] = one[5]
    offsets, at, big = [], 0, 0
    for c, s in enumerate(segs):
        if c % 8192 in (77, 78):
            at += (big - at) % 16                                       # the 16 large ones: every residue
            big += 1
        else:
            at += (c * 7) % 16
        offsets.append(at)
        at += len(s)
    ring = tc.RespRing(lim, 1, n, at, 1 << 16)
    srv = Server(lim, ring, oracle.OracleStore(oracle.PERIODIC, capacity=1 << 17, created_ns=T0, p0=10**9))
    for k in keys:
        srv.note_key(k)
    outs = srv.submit(0, segs, T0, offsets)
    assert {o % 16 for o in offsets} == set(range(16)) and offsets[-1] + len(segs[-1]) == ring.in_capacity
    srv.wait(0)
    assert {o[2] for o in outs} == {0, 1, 2} and sum(o[1] for o in outs) > 30_000
    srv.check_entries(require_expired=False)


# ---------------------------------------------------------------------------------------------------------------
# scenario 6: the parse kernel's key hash at every key length class and shared-memory offset
# ---------------------------------------------------------------------------------------------------------------
@AUTO
@SEEDS
def test_key_hash_from_shared_memory(seed, k1_path):
    """Keys of 0 .. 300 bytes, 4,095, 4,096, 4,097 and ~65,400 bytes (every len % 8 of both hashes' tails), each
    starting at every offset mod 16 of the staged segment (the connection's `off`, and 0 .. 2 frames before the
    key's).  Every row's key_hash is gcra_engine_hash_key of the key bytes, and everything else is checked as in the
    other scenarios."""
    rng = np.random.default_rng(6)
    lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 15, created_ns=T0, max_batch=1 << 14, hash_seed=seed))
    ring = tc.RespRing(lim, 2, 8192, 1 << 22, 1 << 14)
    srv = Server(lim, ring, oracle.OracleStore(oracle.PERIODIC, capacity=1 << 15, created_ns=T0, p0=10**9))
    pre = _raw_throttle(b"", 5, 5, 5)

    def key(n):
        return bytes(rng.integers(33, 127, n).astype(np.uint8))

    small = [(n, r) for n in range(301) for r in range(16)]
    big = [(n, r) for n in (4095, 4096, 4097, 65400) for r in range(16)]
    srv.note_key(b"")
    for t, cases in enumerate((small, big)):
        segs, offsets, keys, at = [], [], [], 0
        for n, r in cases:
            kb = key(n) if n else b""
            if n:
                srv.note_key(kb)
            lead = (n + r) % 3 if n < 60000 else 0
            at += (r - at) % 16                                # off % 16 == r
            segs.append(pre * lead + _raw_throttle(kb, 4, 10, 60))
            offsets.append(at)
            keys += [b""] * lead + [kb]
            at += len(segs[-1])
        srv.submit(t, segs, T0 + t * MS, offsets)
        srv.wait(t)
        rows, _ = ring.rows(t)
        want = np.array([lim.store.hash_key(k) for k in keys], np.uint64)
        assert len(rows) == len(want)
        bad = np.nonzero(rows["key_hash"] != want)[0]
        assert len(bad) == 0, "row %d: key of %d bytes" % (bad[0], len(keys[bad[0]]))
    srv.check_entries(require_expired=False)
