"""The RESP ring (gcra_resp_ring_*, csrc/gcra_resp_ring.cu): connections' read buffers parsed on the GPU, decided as
one batch, replies formatted on the GPU.  Every connection must give exactly what the host parser
gcra_resp_parse_throttle gives at the row cap the connections before it leave -- the same rows, consumed, n_frames
and stop -- and its replies must be the bytes gcra_resp_format_replies writes for a twin engine that decided the
host-parsed rows."""
import ctypes as C

import numpy as np
import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import resp
from test_resp import NOW, OracleEngine, _cmd, _raw_throttle, _throttle

SIP = (0x0706050403020100, 0x0f0e0d0c0b0a0908)
MINIMAL = _raw_throttle(b"", 5, 5, 5)
assert len(MINIMAL) == 45


def _engine(seed=(0, 0), max_batch=1 << 16):
    return tc.RateLimiter(tc.PeriodicStore(capacity=1000, created_ns=NOW, max_batch=max_batch, hash_seed=seed))


def _host_parse(lim, seg, cap):
    req = np.zeros(max(cap, 1), tc.REQ_DTYPE)
    used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
    assert lim._L.gcra_resp_parse_throttle(lim._h, seg, len(seg), NOW, cap, req.ctypes.data, C.byref(used),
                                           C.byref(cnt), C.byref(stop)) == 0
    return req[:cnt.value], used.value, cnt.value, stop.value


def _format(lim, req, res):
    buf = C.create_string_buffer(max(len(req), 1) * tc.RESP_REPLY_MAX)
    w = lim._L.gcra_resp_format_replies(req.ctypes.data, res.ctypes.data, len(req), buf, len(buf))
    return buf.raw[:w]


def _fuzz_frames(rng):
    """test_resp.test_native_pipeline_fuzz_against_the_general_pipeline's frame generator, same distribution"""
    keys = [b"a", b"user:1", "kéy".encode(), b"", b"x" * 70, b"\xff\xfe", b"with\r\ncrlf", b"-1", b"*5", b"$3"]
    nums = [0, 1, 2, 3, 5, 60, 100, -1, -5, 2**31, 2**63 - 1, -2**63, 2**63, "abc", "", "+7", "007", " 5", "5 ", "1e3"]
    kind = int(rng.integers(0, 10))
    if kind <= 5:
        args = [nums[int(rng.integers(0, len(nums)))] if rng.random() < 0.15 else int(rng.integers(1, 200))
                for _ in range(int(rng.choice([3, 3, 3, 4, 4, 2, 5])))]
        f = _raw_throttle(keys[int(rng.integers(0, len(keys)))], *args)
        if rng.random() < 0.1:
            f = f.replace(b"THROTTLE", rng.choice([b"throttle", b"Throttle", b"THROTTLF", b"THROTTL"]).item(), 1)
        return f
    if kind == 6:
        return _cmd(*[["PING"], ["PING", "hello"], ["QUIT"], ["UNKNOWN"], ["throttle", "k", 3, 100, 60],
                      ["THROTTLE", "k", 3, 100, 60, 2]][int(rng.integers(0, 6))])
    if kind == 7:
        f = bytearray(_raw_throttle(b"dmg", 3, 100, 60))
        for _ in range(int(rng.integers(1, 3))):
            op, pos = int(rng.integers(0, 3)), int(rng.integers(0, len(f)))
            if op == 0:
                f[pos] = int(rng.integers(0, 256))
            elif op == 1:
                del f[pos]
            else:
                f.insert(pos, int(rng.choice([0x0d, 0x0a, 0x24, 0x2a, 0x3a, 0x2d, 0x30, 0x39, 0xff])))
        return bytes(f)
    if kind == 8:
        return [b"+OK\r\n", b":5\r\n", b"$-1\r\n", b"*0\r\n", b"*-1\r\n", b"$5\r\nab\r\n",
                b"*5\r\n$8\r\nTHROTTLE\r\n$99999999999\r\n", b"*5\r\n$8\r\nTHROTTLE\r\n$-3\r\n", b"*99999999999\r\n",
                b"\r\n"][int(rng.integers(0, 10))]
    return bytes(rng.integers(0, 256, int(rng.integers(1, 12))).astype(np.uint8))


def _plain_prefix_of_fuzz(rng, n_frames):
    """mostly plain THROTTLE frames (so the GPU has rows to take), then fuzz"""
    fr = [_throttle("u%d" % int(rng.integers(0, 50)), 3, 100, 60) for _ in range(int(rng.integers(0, n_frames)))]
    fr += [_fuzz_frames(rng) for _ in range(int(rng.integers(0, 6)))]
    buf = b"".join(fr)
    if rng.random() < 0.3 and len(buf) > 1:
        buf = buf[:int(rng.integers(1, len(buf)))]
    return buf


def _run_and_check(lim, twin, ring, slot, segs, offsets=None, track=False):
    """place `segs` (neighbouring bytes: plain frames, so a read past a segment would show), submit, and check the
    contract, the replies against the twin, the results against the oracle"""
    inp = ring.input[slot]
    filler = np.frombuffer((_throttle("spill", 1, 1, 1) * (len(inp) // 40 + 1))[:len(inp)], np.uint8)
    inp[:] = filler
    if offsets is None:
        offsets, at = [], 0
        for s in segs:
            at += 7 if len(offsets) % 3 == 1 else 0            # gaps: every residue mod 16 shows up
            offsets.append(at)
            at += len(s)
    for c, (s, off) in enumerate(zip(segs, offsets)):
        inp[off:off + len(s)] = np.frombuffer(s, np.uint8)
        ring.conns[slot][c] = (off, len(s))
    if track:
        lim.store.track_denied(1 << 16)
    ring.submit(slot, len(segs), NOW)
    ring.wait(slot)
    rows, res = ring.rows(slot)
    out = ring.outcome[slot][:len(segs)].copy()
    host_rows = []
    for c, s in enumerate(segs):
        base = sum(len(r) for r in host_rows)
        r, used, cnt, stop = _host_parse(lim, s, ring.row_capacity - base)
        assert (int(out[c]["consumed"]), int(out[c]["n_frames"]), int(out[c]["stop"])) == (used, cnt, stop), c
        host_rows.append(r)
    want = np.concatenate(host_rows) if host_rows else np.zeros(0, tc.REQ_DTYPE)
    assert rows.tobytes() == want.tobytes()
    # the twin decides the host-parsed rows through a plain ring, in the same order
    tres = np.zeros(0, tc.RES_DTYPE)
    if len(want):
        tring = twin._resp_twin_ring
        tring.req[0][:len(want)] = want
        tring.submit(0, len(want), NOW)
        tring.wait(0)
        tres = tring.res[0][:len(want)].copy()
    assert res.tobytes() == tres.tobytes()
    base = 0
    for c in range(len(segs)):
        n = int(out[c]["n_frames"])
        got = ring.replies[slot][int(out[c]["reply_off"]):int(out[c]["reply_off"]) + int(out[c]["reply_len"])]
        assert got.tobytes() == _format(twin, want[base:base + n], tres[base:base + n]), c
        base += n
    if len(want):                                          # one oracle store replaying the rows, row for row
        ores = lim._resp_oracle(want)
        for f in ("status", "allowed", "remaining", "reset_after_ns", "retry_after_ns"):
            assert np.array_equal(ores[f], res[f]), f
    if track:
        dn = {}
        for r, x in zip(want, res):
            if int(x["status"]) == tc.OK and not x["allowed"]:
                dn[int(r["key_hash"])] = dn.get(int(r["key_hash"]), 0) + 1
        top, dropped = lim.store.top_denied(1 << 16)
        assert dropped == 0 and dict(top) == dn
    return rows, res, out


def _pair(seed, row_capacity, max_conns=512, in_capacity=1 << 22, slots=2):
    lim, twin = _engine(seed), _engine(seed)
    ring = tc.RespRing(lim, slots, max_conns, in_capacity, row_capacity)
    twin._resp_twin_ring = tc.Ring(twin, 1, row_capacity)
    lim._resp_oracle = OracleEngine()
    return lim, twin, ring


def _same_state(lim, twin, rows):
    for k in set(int(x) for x in rows["key_hash"]):
        assert lim.store.peek(k) == twin.store.peek(k)
    a, b = lim.store.stats(), twin.store.stats()
    for f in ("len", "allowed", "denied", "errors"):
        assert a[f] == b[f], f


@pytest.mark.gpu
# (auto only: every RESP batch takes the index-order pipeline, see test_gpu_resp_ring_inflight.py)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("seed", [(0, 0), SIP], ids=["unkeyed", "siphash"])
def test_parse_contract_over_fuzz_and_connection_counts(seed, k1_path):
    lim, twin, ring = _pair(seed, row_capacity=1 << 14)
    rng = np.random.default_rng(20260923)
    all_rows = []
    for i, n_conns in enumerate([1, 7, 300, 512]):
        segs = [_plain_prefix_of_fuzz(rng, 40) for _ in range(n_conns)]
        segs[n_conns // 2] = b""                                   # an empty connection
        rows, _, _ = _run_and_check(lim, twin, ring, i % 2, segs, track=(i == 2))
        all_rows.append(rows)
    _same_state(lim, twin, np.concatenate(all_rows))


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("seed", [(0, 0), SIP], ids=["unkeyed", "siphash"])
def test_adversarial_connections(seed, k1_path):
    lim, twin, ring = _pair(seed, row_capacity=1 << 14)
    inner = _raw_throttle(b"k", 3, 100, 60)
    full = MINIMAL * (65536 // 45)
    segs = [
        _raw_throttle(b"\r\n" + inner * 3, 3, 100, 60) * 5,              # keys that hold complete frames
        _raw_throttle(b"\n*" * 32700, 3, 100, 60),                       # candidates nearly everywhere
        (b"*\n" * 32768),                                                 # 32 K candidates, no frame
        full + MINIMAL[:65536 - len(full)],                               # 65,536 bytes of minimal frames, cut
        _raw_throttle(b"a" * 65400, 3, 100, 60),                          # one key of ~64 KiB
        inner * 3 + inner[:-3],                                           # cut by the segment end: stop 1
        inner + _raw_throttle(b"bad\xff", 3, 100, 60) + inner,            # not UTF-8: stop 2
        inner + _raw_throttle(b"d19", 10**18, 100, 60),                   # 19 digits: plain
        inner + _raw_throttle(b"d20", 10**19, 100, 60),                   # 20 digits: stop 2
        _raw_throttle(b"neg", -3, 100, 60, -1) + _throttle("q", 5, 10, 60, 2),
        b"",
    ]
    assert len(segs[3]) == 65536
    offs, at = [], 0
    for i, s in enumerate(segs):
        at += i % 16                                                      # every residue mod 16
        offs.append(at)
        at += len(s)
    rows, _, out = _run_and_check(lim, twin, ring, 0, segs, offsets=offs)
    assert [int(x) for x in out["stop"]] == [0, 0, 2, 1, 0, 1, 2, 0, 2, 0, 0]
    assert int(out[3]["n_frames"]) == 65536 // 45
    _same_state(lim, twin, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_row_cap_inside_a_connection_and_at_a_boundary(k1_path):
    lim, twin, ring = _pair((0, 0), row_capacity=100)
    f = _throttle("cap", 1000, 100, 60)
    for segs in ([f * 60, f * 60, f * 10],            # the cap falls inside the second connection
                 [f * 60, f * 40, f * 5, b""],       # exactly at the end of the second: the third stops at once
                 [f * 60, f * 40 + _cmd("PING")]):   # exactly at a frame that is not plain: still stop 3
        _, _, out = _run_and_check(lim, twin, ring, 0, segs)
        assert 3 in [int(x) for x in out["stop"]]


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_refused_submits_enqueue_nothing(k1_path):
    lim, twin, ring = _pair((0, 0), row_capacity=1024, max_conns=4, in_capacity=1 << 18)
    f = _throttle("r", 5, 10, 60)
    bad = [[(0, 65537)], [((1 << 18) - 10, 11)], [(0, len(f))] * 4]
    for i, table in enumerate(bad):
        for c, (o, ln) in enumerate(table):
            ring.conns[0][c] = (o, ln)
        with pytest.raises(tc.Internal):
            ring.submit(0, len(table) + (i == 2), NOW)          # the last: more connections than max_conns
    assert lim.store.stats()["allowed"] == 0
    _run_and_check(lim, twin, ring, 0, [f * 3, f])
    ring.input[1][:len(f)] = np.frombuffer(f, np.uint8)
    ring.conns[1][0] = (0, len(f))
    ring.submit(1, 1, NOW)
    with pytest.raises(tc.Internal):
        ring.submit(1, 1, NOW)                                  # in flight
    ring.wait(1)
    one = _host_parse(lim, f, 1)[0]
    twin._resp_twin_ring.req[0][:1] = one
    twin._resp_twin_ring.submit(0, 1, NOW)
    twin._resp_twin_ring.wait(0)
    lim._resp_oracle(one)
    _run_and_check(lim, twin, ring, 0, [f * 2])


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_process_connections_equals_process_pipeline_on_disjoint_keys(k1_path):
    rng = np.random.default_rng(7)
    lim = _engine()
    ring = tc.RespRing(lim, 1, 64, 1 << 20, 4096)
    bufs = []
    for c in range(40):
        fr = [_throttle("c%d:%d" % (c, int(rng.integers(0, 4))), 3, 100, 60) for _ in range(int(rng.integers(0, 30)))]
        for _ in range(int(rng.integers(0, 4))):
            fr.insert(int(rng.integers(0, len(fr) + 1)), [
                _cmd("PING"), _cmd("throttle", "c%d:0" % c, 3, 100, 60), _cmd("UNKNOWN"),
                _throttle("c%d:1" % c, 3, 100, 60, -1), _raw_throttle(("c%d:é" % c).encode(), 3, 100, 60)][
                int(rng.integers(0, 5))])
        buf = b"".join(fr)
        if c % 7 == 3:
            buf += _cmd("QUIT") + fr[0] if fr else _cmd("QUIT")
        if c % 7 == 5:
            buf += b"?garbage\r\n" + (fr[0] if fr else b"")
        if c % 5 == 1 and buf:
            buf = buf[:-4]
        bufs.append(buf)
    got = resp.process_connections(bufs, lim, NOW, ring, 0)
    for c, b in enumerate(bufs):
        want = resp.process_pipeline(b, _engine().rate_limit_batch, NOW)
        assert got[c] == want, c


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_process_connections_shared_keys_in_the_documented_order(k1_path):
    """Three connections on the same keys, each with a PING in the middle: round 1 decides every connection's prefix
    (list order), then nothing for the PINGs; round 2 the rest, in list order.  An oracle replay in that order gives
    the same replies."""
    lim = _engine()
    ring = tc.RespRing(lim, 1, 8, 1 << 16, 1024)
    f = [_throttle("shared:%d" % (i % 2), 4, 10, 60) for i in range(6)]
    bufs = [b"".join(f[:2]) + _cmd("PING") + b"".join(f[2:4]), b"".join(f[:3]) + _cmd("PING") + f[4],
            b"".join(f[:1]) + _cmd("PING") + b"".join(f[:2])]
    got = resp.process_connections(bufs, lim, NOW, ring, 0)
    eng = OracleEngine()
    want = [bytearray() for _ in bufs]
    order = []                                   # (connection, frame bytes) in the documented order
    for c, b in enumerate(bufs):                 # round 1: the prefixes
        head = b.split(_cmd("PING"))[0]
        order.append((c, head))
    for c, b in enumerate(bufs):                 # round 2: after each PING
        order.append((c, b.split(_cmd("PING"))[1]))
    for rnd, (c, chunk) in enumerate(order):
        want[c] += resp.process_pipeline(chunk, eng, NOW)[0]
        if rnd < len(bufs):
            want[c] += b"+PONG\r\n"
    for c, b in enumerate(bufs):
        assert got[c][0] == bytes(want[c]) and got[c][1] == len(b) and got[c][3] is None, c
