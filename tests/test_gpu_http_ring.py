"""The HTTP ring (gcra_http_ring_create + the gcra_resp_ring_* calls, csrc/gcra_resp_ring.cu with HttpTraits):
connections' read buffers parsed on the GPU, decided as one batch, responses formatted on the GPU.  Every connection
must give exactly what the host walk gcra_http_parse_throttle gives at the row cap the connections before it leave,
and its responses must be the bytes gcra_http_format_replies writes for a twin engine that decided the host-parsed
rows."""
import ctypes as C

import numpy as np
import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import http
from test_http_cpu import NEAR_MISSES, README, _fuzz_request, body_of, request
from test_resp import NOW, OracleEngine

SIP = (0x0706050403020100, 0x0f0e0d0c0b0a0908)
MINIMAL = request(b'{"key":"","max_burst":5,"count_per_period":5,"period":5}',
                  [(b"content-length", b"56"), (b"content-type", b"application/json")]).replace(b": ", b":")
assert len(MINIMAL) == 133


def _engine(seed=(0, 0), max_batch=1 << 16):
    return tc.RateLimiter(tc.PeriodicStore(capacity=1000, created_ns=NOW, max_batch=max_batch, hash_seed=seed))


def _host_parse(lim, seg, cap):
    # (room for the rows `seg` can hold: a plain request has at least 133 bytes)
    req = np.zeros(max(min(cap, len(seg) // 133 + 1), 1), tc.REQ_DTYPE)
    used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
    assert lim._L.gcra_http_parse_throttle(lim._h, seg, len(seg), NOW, cap, req.ctypes.data, C.byref(used),
                                           C.byref(cnt), C.byref(stop)) == 0
    return req[:cnt.value], used.value, cnt.value, stop.value


def _conn(rng, n_req):
    """mostly plain requests (so the GPU has rows to take), then fuzz, sometimes cut"""
    fr = [request(body_of("u%d" % int(rng.integers(0, 50)), 3, 100, 60)) for _ in range(int(rng.integers(0, n_req)))]
    fr += [_fuzz_request(rng) for _ in range(int(rng.integers(0, 4)))]
    if rng.random() < 0.2:
        fr.append(list(NEAR_MISSES.values())[int(rng.integers(0, len(NEAR_MISSES)))])
    buf = b"".join(fr)
    if rng.random() < 0.3 and len(buf) > 1:
        buf = buf[:int(rng.integers(1, len(buf)))]
    return buf


def _run_and_check(lim, twin, ring, slot, segs, offsets=None, track=False):
    """place `segs` (neighbouring bytes: plain requests, so a read past a segment would show), submit, and check the
    contract, the responses against the twin, the results against the oracle"""
    inp = ring.input[slot]
    fill = request(body_of("spill", 1, 1, 1))
    inp[:] = np.frombuffer((fill * (len(inp) // len(fill) + 1))[:len(inp)], np.uint8)
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
    host_rows, base = [], 0
    for c, s in enumerate(segs):
        r, used, cnt, stop = _host_parse(lim, s, ring.row_capacity - base)
        assert (int(out[c]["consumed"]), int(out[c]["n_frames"]), int(out[c]["stop"])) == (used, cnt, stop), c
        host_rows.append(r)
        base += cnt
    want = np.concatenate(host_rows) if host_rows else np.zeros(0, tc.REQ_DTYPE)
    assert rows.tobytes() == want.tobytes()
    tres = np.zeros(0, tc.RES_DTYPE)
    if len(want):
        tring = twin._http_twin_ring
        tring.req[0][:len(want)] = want
        tring.submit(0, len(want), NOW)
        tring.wait(0)
        tres = tring.res[0][:len(want)].copy()
    assert res.tobytes() == tres.tobytes()
    base = 0
    for c in range(len(segs)):
        n = int(out[c]["n_frames"])
        got = ring.replies[slot][int(out[c]["reply_off"]):int(out[c]["reply_off"]) + int(out[c]["reply_len"])]
        assert got.tobytes() == http.format_replies(want[base:base + n], tres[base:base + n]), c
        base += n
    if len(want):
        ores = lim._http_oracle(want)
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
    ring = tc.HttpRing(lim, slots, max_conns, in_capacity, row_capacity)
    twin._http_twin_ring = tc.Ring(twin, 1, row_capacity)
    lim._http_oracle = OracleEngine()
    return lim, twin, ring


def _same_state(lim, twin, rows):
    for k in set(int(x) for x in rows["key_hash"]):
        assert lim.store.peek(k) == twin.store.peek(k)
    a, b = lim.store.stats(), twin.store.stats()
    for f in ("len", "allowed", "denied", "errors"):
        assert a[f] == b[f], f


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("seed", [(0, 0), SIP], ids=["unkeyed", "siphash"])
def test_parse_contract_over_fuzz_and_connection_counts(seed, k1_path):
    lim, twin, ring = _pair(seed, row_capacity=1 << 14)
    rng = np.random.default_rng(20261017)
    all_rows = []
    for i, n_conns in enumerate([1, 7, 300, 512]):
        segs = [_conn(rng, 20) for _ in range(n_conns)]
        segs[n_conns // 2] = b""                                   # an empty connection
        rows, _, _ = _run_and_check(lim, twin, ring, i % 2, segs, track=(i == 2))
        all_rows.append(rows)
    _same_state(lim, twin, np.concatenate(all_rows))


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("seed", [(0, 0), SIP], ids=["unkeyed", "siphash"])
def test_adversarial_connections(seed, k1_path):
    lim, twin, ring = _pair(seed, row_capacity=1 << 14)
    inner = request(README)
    head = inner.split(b"\r\n\r\n")[0]
    full = MINIMAL * (65536 // 133)
    big = request(body_of("a" * 65000))
    segs = [
        request(body_of(head.decode().replace("\r\n", " ") * 3)) * 5,    # keys that hold "POST " and whole heads
        request(body_of("POST " * 12000)),                               # candidates nearly everywhere
        b"POST " * 13107,                                                # 13 K candidates, no request
        full + MINIMAL[:65536 - len(full)],                              # 65,536 bytes of minimal requests, cut
        big,                                                             # one key of ~64 KiB
        inner * 3 + inner[:-3],                                          # cut by the segment end: stop 1
        inner + NEAR_MISSES["escape"] + inner,                           # an escape: stop 2
        inner + request(body_of("d19", 10**18, 100, 60)),                # 19 digits: plain
        inner + request(body_of("d20", 10**19, 100, 60)),                # 20 digits: stop 2
        request(body_of("neg", -3, 100, 60, -1)) + request(body_of("q", 5, 10, 60, 2)),
        inner + b"POS",                                                  # a request line cut after 3 bytes
        b"",
    ]
    assert len(segs[3]) == 65536 and len(big) <= 65536
    offs, at = [], 0
    for i, s in enumerate(segs):
        at += i % 16                                                     # every residue mod 16
        offs.append(at)
        at += len(s)
    rows, _, out = _run_and_check(lim, twin, ring, 0, segs, offsets=offs)
    assert [int(x) for x in out["stop"]] == [0, 0, 2, 1, 0, 1, 2, 0, 2, 0, 1, 0]
    assert int(out[3]["n_frames"]) == 65536 // 133
    _same_state(lim, twin, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_row_cap_inside_a_connection_and_at_a_boundary(k1_path):
    lim, twin, ring = _pair((0, 0), row_capacity=100)
    f = request(body_of("cap", 1000, 100, 60))
    for segs in ([f * 60, f * 60, f * 10],
                 [f * 60, f * 40, f * 5, b""],
                 [f * 60, f * 40 + b"GET /health HTTP/1.1\r\n\r\n"]):
        _, _, out = _run_and_check(lim, twin, ring, 0, segs)
        assert 3 in [int(x) for x in out["stop"]]


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_65536_connections_with_one_request_each(k1_path):
    n = 65536
    rng = np.random.default_rng(5)
    keys = rng.zipf(1.2, n) % 5000
    segs = [request(body_of("z:%d" % k, 5, 10, 60)) for k in keys]
    total = sum(len(s) for s in segs)
    lim, twin, ring = _pair(SIP, row_capacity=n, max_conns=n, in_capacity=total, slots=1)
    offs = list(np.cumsum([0] + [len(s) for s in segs[:-1]]))
    rows, _, out = _run_and_check(lim, twin, ring, 0, segs, offsets=offs)
    assert len(rows) == n and set(int(x) for x in out["stop"]) == {0}
    _same_state(lim, twin, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_refused_submits_enqueue_nothing(k1_path):
    lim, twin, ring = _pair((0, 0), row_capacity=1024, max_conns=4, in_capacity=1 << 18)
    f = request(README)
    bad = [[(0, 65537)], [((1 << 18) - 10, 11)], [(0, len(f))] * 4]
    for i, table in enumerate(bad):
        for c, (o, ln) in enumerate(table):
            ring.conns[0][c] = (o, ln)
        with pytest.raises(tc.Internal):
            ring.submit(0, len(table) + (i == 2), NOW)
    with pytest.raises(tc.Internal):                                  # an HTTP ring takes gcra_resp_ring_submit
        lim.store._check(lim._L.gcra_ring_submit(lim._h, 0, 1, NOW))
    assert lim.store.stats()["allowed"] == 0
    _run_and_check(lim, twin, ring, 0, [f * 3, f])
    ring.input[1][:len(f)] = np.frombuffer(f, np.uint8)
    ring.conns[1][0] = (0, len(f))
    ring.submit(1, 1, NOW)
    with pytest.raises(tc.Internal):
        ring.submit(1, 1, NOW)                                          # in flight
    ring.wait(1)
    one = _host_parse(lim, f, 1)[0]
    twin._http_twin_ring.req[0][:1] = one
    twin._http_twin_ring.submit(0, 1, NOW)
    twin._http_twin_ring.wait(0)
    lim._http_oracle(one)
    _run_and_check(lim, twin, ring, 0, [f * 2])


def _mixed(rng, c, shared):
    """a connection's requests: plain ones and every kind the general path answers"""
    key = (lambda i: "shared:%d" % (i % 3)) if shared else (lambda i: "c%d:%d" % (c, i % 4))
    ct = (b"Content-Type", b"application/json")
    kinds = [
        lambda i: request(body_of(key(i), 4, 10, 60)),
        lambda i: b"GET /health HTTP/1.1\r\nHost: x\r\n\r\n",
        lambda i: b"GET /nope HTTP/1.1\r\n\r\n",
        lambda i: request(README, [(b"Content-Length", b"%d" % len(README))]),                 # 415
        lambda i: request(b'{"key": "x", "max_burst": NaN}', [ct, (b"Content-Length", b"30")]),   # 400
        lambda i: request(b'{"key": "x"}', [ct, (b"Content-Length", b"12")]),                    # 422
        lambda i: request(body_of(key(i), 4, 10, 60).replace(b'": "', b'": "\\u00', 1).replace(  # escaped key
            b'\\u00' + key(i)[:1].encode(), b'\\u00%02x' % ord(key(i)[0]), 1)),
        lambda i: request(body_of(key(i), 4, 10, 60)[:-1] + b', "extra": [1, {"a": null}]}'),    # unknown field
        lambda i: request(body_of(key(i), 4, 10, 60, -1)),                                         # 500
    ]
    out = []
    for i in range(int(rng.integers(0, 12))):
        k = 0 if rng.random() < 0.5 else int(rng.integers(1, len(kinds)))
        out.append(kinds[k](i))
    if c % 7 == 3:
        out.append(NEAR_MISSES["connection close"].replace(b"test", key(0).encode().ljust(4, b"_")[:4]))
        out.append(request(body_of(key(1), 4, 10, 60)))                # after the close: never answered
    if c % 11 == 5:
        out.append(b"garbage\r\n\r\n" + request(README))
    buf = b"".join(out)
    if c % 5 == 1 and buf:
        buf = buf[:-4]
    return buf


def _pure_python(bufs, limiter_factory, shared):
    """every request through the general path, decided by rate_limit_batch; with shared keys, in the documented
    order (rounds: each connection's plain prefix, then one general request per connection)"""
    lim = limiter_factory()
    n = len(bufs)
    pos, n_thr, close, out = [0] * n, [0] * n, [None] * n, [[] for _ in range(n)]
    live = [c for c in range(n) if bufs[c]]
    while live:
        nxt = []
        gen = {}
        for c in live:                                    # the GPU's share of the round: the plain prefix
            while pos[c] < len(bufs[c]):
                used, cnt, stop = _host_parse(lim, bufs[c][pos[c]:], 1)[1:]
                if cnt == 0:
                    gen[c] = stop
                    break
                g = http.parse_request(bufs[c][pos[c]:])
                o, k, _ = http.handle_request(g, lim, NOW)
                out[c].append(o)
                n_thr[c] += k
                pos[c] += g.consumed
            else:
                gen[c] = 0
        for c in live:
            if gen[c] != 2:
                continue
            g = http.parse_request(bufs[c][pos[c]:])
            if g is None:
                continue
            o, k, cl = http.handle_request(g, lim, NOW)
            out[c].append(o)
            n_thr[c] += k
            pos[c] += g.consumed
            if cl:
                close[c] = "error" if g.bad is not None else "close"
            elif pos[c] < len(bufs[c]):
                nxt.append(c)
        live = nxt
    return [(b"".join(out[c]), pos[c], n_thr[c], close[c]) for c in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("shared", [False, True], ids=["disjoint", "shared"])
def test_process_connections_equals_the_general_path(shared, k1_path):
    rng = np.random.default_rng(11 + shared)
    bufs = [_mixed(rng, c, shared) for c in range(60)]
    lim = _engine()
    ring = tc.HttpRing(lim, 1, 64, 1 << 20, 4096)
    got = http.process_connections(bufs, lim, NOW, ring, 0)
    want = _pure_python(bufs, _engine, shared)
    for c in range(len(bufs)):
        assert got[c] == want[c], c
    assert any(g[3] == "close" for g in got) and any(g[3] == "error" for g in got)
    assert sum(g[2] for g in got) > 100
