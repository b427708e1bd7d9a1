"""Ring metrics (gcra_ring_metrics, gcra_ring_transport_counts, gcra_denied_names) and metrics.Metrics on the GPU.

Each ring kind (RESP, HTTP, gRPC, mixed) serves connections whose keys the test knows -- shared hot keys, keys of 0, 1,
255, 256 and 257 bytes, rows with status other than OK, a 64 KiB connection -- in rounds of two slots in flight, with
stop-3 resubmits.  The counts must be the reference's rules applied to ring.rows(slot), every denied hash must be
named with exactly its key's bytes (GCRA_NAME_TOO_LONG past 256 bytes), and everything the rings return must equal a
twin engine's with metrics off, whose launches per submit are the ring's own.  Then: pruning keeps names, the
max_keys refusals leave the engine usable, and mixed.process_connections with a Metrics serves GET /metrics text equal
to an independent model of metrics.rs fed by the requests' transports, keys and outcomes read from the replies."""
import copy
import json
import random
import re

import numpy as np
import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import grpc_transport as gt
from throttlecrab_b200 import mixed
from throttlecrab_b200.metrics import Metrics
from throttlecrab_b200.resp import RespParser
import grpc_streams as gs
from grpc_server import request_bytes
from test_http_cpu import body_of, request
from test_resp import _cmd, _throttle

pytestmark = [pytest.mark.gpu, pytest.mark.parametrize("k1_path", ["auto"], indirect=True)]
NS = 10**9
NOW = 1_700_000_000 * NS
P = {"resp": tc.PROTO_RESP, "http": tc.PROTO_HTTP, "grpc": tc.PROTO_GRPC}
T = {"resp": 0, "http": 1, "grpc": 2}
HOT = ["hot:%d" % i for i in range(4)]
KEYS = HOT + ["", "a", "L" * 255, "M" * 256, "N" * 257] + ["k%d" % i for i in range(8)]


def _engine(max_batch=1 << 16):
    return tc.RateLimiter(tc.PeriodicStore(capacity=1 << 14, created_ns=NOW, max_batch=max_batch))


class Conn:
    """a connection of protocol p: its bytes and position, or (gRPC) its Connection"""

    def __init__(self, p, data):
        self.p, self.pos, self.stop = p, 0, None
        self.data = data if p != "grpc" else None
        self.cn = data if p == "grpc" else None

    def rest(self):
        return bytes(self.cn.buf) if self.p == "grpc" else self.data[self.pos:]


def _args(rng):
    return rng.choice([1, 2, 5]), rng.choice([1, 10, 100]), 60, rng.choice([None, 1, 1, 2, 5, -1])


def _make(rng, p, n, keys=KEYS):
    if p == "resp":
        return Conn(p, b"".join(_throttle(rng.choice(keys), *_args(rng)) for _ in range(n)))
    if p == "http":
        return Conn(p, b"".join(request(body_of(rng.choice(keys), *_args(rng))) for _ in range(n)))
    cn = gs.established()
    cn.buf += gs.steady_stream(rng, cn, n, keys, extras=False)
    return Conn(p, cn)


def _conns(rng, kind, n):
    ps = ["resp", "http", "grpc"] if kind == "mixed" else [kind]
    out = [_make(rng, rng.choice(ps), rng.randrange(0, 30)) for _ in range(n)]
    big = "grpc" if kind == "grpc" else "http" if kind == "http" else "resp"
    k = 65536 // len(_make(rng, big, 1, ["hot:0"]).rest())
    while True:                                                 # a connection of nearly 64 KiB
        c = _make(rng, big, k, HOT)
        if len(c.rest()) <= 65536:
            break
        k -= max(1, k // 50)
    out.insert(n // 2, c)
    return out


def _submit(ring, slot, kind, conns, now=NOW):
    at, k = 0, 0
    for j, c in enumerate(conns):
        b = c.rest()
        ring.input[slot][at:at + len(b)] = np.frombuffer(b, np.uint8)
        row = ring.conns[slot][j]
        if kind == "mixed":
            row["off"], row["len"], row["protocol"], row["grpc_state"] = at, len(b), P[c.p], k if c.p == "grpc" else 0
            if c.p == "grpc":
                c.cn.state(ring.grpc_conns[slot][k])
                k += 1
        else:
            row["off"], row["len"] = at, len(b)
            if kind == "grpc":
                c.cn.state(row)
        at += len(b)
    ring.submit(slot, len(conns), now)


def _collect(ring, slot, kind, conns, counts, denied, key_of):
    """after wait: advance the connections; tally the slot's rows by the reference's rules"""
    rows, res = ring.rows(slot)
    base, k = 0, 0
    for j, c in enumerate(conns):
        o = ring.outcome[slot][j]
        n, consumed = int(o["n_frames"]), int(o["consumed"])
        for i in range(base, base + n):
            ok, allowed = int(res[i]["status"]) == tc.OK, bool(res[i]["allowed"])
            cls = 1 if ok and not allowed else 0 if ok or c.p == "resp" else 2
            counts[T[c.p], cls] += 1
            if cls == 1:
                h = int(rows[i]["key_hash"])
                assert h in key_of
                denied[h] = denied.get(h, 0) + 1
        base += n
        if c.p == "grpc":
            go = o
            if kind == "mixed":
                go = ring.grpc_outcome[slot][k]
                k += 1
            off, ln = int(go["reply_off"]), int(go["reply_len"])
            c.cn.out += ring.replies[slot][off:off + ln].tobytes()
            c.cn.take_outcome(go)
            del c.cn.buf[:consumed]
        else:
            c.pos += consumed
        c.stop = int(o["stop"])
    assert base == len(rows)
    return rows, res


def _slot_bytes(ring, slot, n_conns):
    """everything a slot returns: rows, results, outcomes and reply bytes"""
    rows, res = ring.rows(slot)
    out = ring.outcome[slot][:n_conns]
    end = max([int(o["reply_off"]) + int(o["reply_len"]) for o in out] + [0])
    extra = ring.grpc_outcome[slot][:n_conns].tobytes() if ring.protocol == "mixed" else b""
    return rows.tobytes() + res.tobytes() + out.tobytes() + ring.replies[slot][:end].tobytes() + extra


def _ring(lim, kind, row_capacity):
    return tc.RespRing(lim, 2, 128, 1 << 21, row_capacity, protocol=kind)


# ---- 1. counts, names, results and launches per ring kind -------------------------------------------------------------
@pytest.mark.parametrize("kind", ["resp", "http", "grpc", "mixed"])
def test_counts_and_names_match_the_rows(kind, k1_path):
    rng = random.Random(["resp", "http", "grpc", "mixed"].index(kind))
    lim, twin = _engine(), _engine()
    key_of = {lim.store.hash_key(k.encode()): k.encode() for k in KEYS}
    for e in (lim, twin):
        e.store.track_denied(1024)
    lim.store.ring_metrics(True)
    ring, tring = _ring(lim, kind, 400), _ring(twin, kind, 400)
    conns = _conns(rng, kind, 40)
    tconns = copy.deepcopy(conns)
    counts, denied = np.zeros((3, 3), np.uint64), {}
    live = [j for j, c in enumerate(conns) if c.rest()]
    rounds = 0
    while live:
        halves = [live[:len(live) // 2 + 1], live[len(live) // 2 + 1:]]   # two slots in flight on shared keys
        halves = [hv for hv in halves if hv]
        l0, t0 = lim.store.launch_count(), twin.store.launch_count()
        for s, hv in enumerate(halves):
            _submit(ring, s, kind, [conns[j] for j in hv])
            _submit(tring, s, kind, [tconns[j] for j in hv])
        nrows = []
        for s, hv in enumerate(halves):
            ring.wait(s)
            tring.wait(s)
            assert _slot_bytes(ring, s, len(hv)) == _slot_bytes(tring, s, len(hv))
            rows, _ = _collect(ring, s, kind, [conns[j] for j in hv], counts, denied, key_of)
            _collect(tring, s, kind, [tconns[j] for j in hv], np.zeros((3, 3), np.uint64), {}, key_of)
            nrows.append(len(rows))
        got = lim.store.launch_count() - l0
        assert got == twin.store.launch_count() - t0 + sum(1 for n in nrows if n)
        live = [j for j in live if conns[j].stop == 3]
        rounds += 1
    assert rounds > 1                                          # (stop 3 happened: resubmits)
    assert counts[:, 1].sum() > 0 and counts[1:, 2].sum() + counts[0, 0] > 0
    assert (lim.store.ring_transport_counts() == counts).all()
    assert (twin.store.ring_transport_counts() == 0).all()
    top, dropped = lim.store.top_denied(1 << 12)
    assert dropped == 0 and dict(top) == denied
    assert top == twin.store.top_denied(1 << 12)[0]
    names = lim.store.denied_names([h for h, _ in top])
    long_seen = False
    for (h, _), nm in zip(top, names):
        key = key_of[h]
        if len(key) > tc.DENIED_NAME_MAX:
            assert nm == tc.NAME_TOO_LONG
            long_seen = True
        else:
            assert nm == key, (key, nm)
    assert long_seen
    assert twin.store.denied_names([h for h, _ in top]) == [tc.NAME_UNKNOWN] * len(top)

    # off: no kernel, counts kept, names released
    lim.store.ring_metrics(False)
    again = [_make(rng, "grpc" if kind == "grpc" else "resp" if kind != "http" else "http", 10, HOT)
             for _ in range(3)]
    l0, t0 = lim.store.launch_count(), twin.store.launch_count()
    _submit(ring, 0, kind, again)
    _submit(tring, 0, kind, copy.deepcopy(again))
    ring.wait(0)
    tring.wait(0)
    assert lim.store.launch_count() - l0 == twin.store.launch_count() - t0
    assert (lim.store.ring_transport_counts() == counts).all()
    assert lim.store.denied_names([h for h, _ in top]) == [tc.NAME_UNKNOWN] * len(top)


# ---- 2. pruning -------------------------------------------------------------------------------------------------------
def _deny(ring, lim, keys_times):
    """one RESP slot: key k denied n times (quantity 5 over a burst of 1)"""
    buf = b"".join(_throttle(k, 1, 1, 60, 5) * n for k, n in keys_times)
    ring.input[0][:len(buf)] = np.frombuffer(buf, np.uint8)
    ring.conns[0][0] = (0, len(buf))
    ring.submit(0, 1, NOW)
    ring.wait(0)
    assert int(ring.outcome[0][0]["consumed"]) == len(buf)


def test_pruning_keeps_names(k1_path):
    lim = _engine()
    lim.store.track_denied(4)
    lim.store.ring_metrics(True)
    ring = tc.RespRing(lim, 1, 4, 1 << 20, 4096)
    _deny(ring, lim, [("p:%d" % i, i + 1) for i in range(20)])
    top, _ = lim.store.top_denied(100)                          # 20 keys > 3 x 4: pruned to the top 4
    assert len(top) == 20
    top, _ = lim.store.top_denied(100)
    assert [c for _, c in top] == [20, 19, 18, 17]
    assert lim.store.denied_names([h for h, _ in top]) == [b"p:%d" % i for i in (19, 18, 17, 16)]
    _deny(ring, lim, [("p:0", 30)])                             # a pruned key, denied again
    top, _ = lim.store.top_denied(100)
    assert top[0] == (lim.store.hash_key(b"p:0"), 30)
    assert lim.store.denied_names([h for h, _ in top]) == [b"p:%d" % i for i in (0, 19, 18, 17, 16)]


# ---- 3. the refusals -------------------------------------------------------------------------------------------------
def test_max_keys_refusals_leave_the_engine_usable(k1_path):
    lim = _engine()
    lim.store.track_denied(20_000)
    with pytest.raises(tc.Internal):
        lim.store.ring_metrics(True)
    lim.store.track_denied(10_000)
    lim.store.ring_metrics(True)
    with pytest.raises(tc.Internal):
        lim.store.track_denied(10_001)
    ring = tc.RespRing(lim, 1, 4, 1 << 20, 4096)
    _deny(ring, lim, [("r:a", 3), ("r:b", 2)])
    top, _ = lim.store.top_denied(10)
    assert [c for _, c in top] == [3, 2]
    assert lim.store.denied_names([h for h, _ in top]) == [b"r:a", b"r:b"]
    assert lim.store.ring_transport_counts().tolist() == [[0, 5, 0], [0, 0, 0], [0, 0, 0]]
    lim.store.track_denied(100)                                 # a new table: names start over
    lim.store.ring_metrics(True)                                # on again: counts zeroed
    _deny(ring, lim, [("r:c", 1)])
    top, _ = lim.store.top_denied(10)
    assert lim.store.denied_names([h for h, _ in top]) == [b"r:c"]
    assert lim.store.ring_transport_counts().tolist() == [[0, 1, 0], [0, 0, 0], [0, 0, 0]]


# ---- 4. end to end: mixed.process_connections with a Metrics, GET /metrics against a model of metrics.rs -------------
SPECIAL = 'q"\\\x01\x7f\x85é'


def _e2e_conns(rng):
    """(protocol, conn) and per connection its requests: (kind, key) with kind "cmd" (a RESP command other than
    THROTTLE, counted), "throttle", or "uncounted" (HTTP: /health, a bad body)"""
    conns, reqs = [], []
    S = ["shared:%d" % i for i in range(4)]
    for c in range(6):
        p = ["resp", "http", "grpc"][c % 3]
        items = [("throttle", rng.choice(S), rng.choice([None, 1, 2])) for _ in range(rng.randrange(8, 20))]
        if p == "resp":
            extra = [("cmd", _cmd("PING")), ("cmd", _cmd("NOPE")), ("raw", _cmd("THROTTLE", "shared:0", 2, 1, 60)),
                     ("throttle", "neg", -1), ("throttle", SPECIAL, 5)]
        elif p == "http":
            extra = [("esc", b'{"key": "shared:\\u0030", "max_burst": 2, "count_per_period": 1, "period": 60}'),
                     ("uncounted", b"GET /health HTTP/1.1\r\nHost: x\r\n\r\n"),
                     ("uncounted", request(b'{"key": ')), ("throttle", "neg", -1)]
        else:
            extra = [("throttle", "neg", -1)]
        for e in extra:
            items.insert(rng.randrange(len(items) + 1), e)
        if p == "resp":
            buf, rq = b"", []
            for it in items:
                if it[0] == "throttle":
                    buf += _throttle(it[1], 2, 1, 60, it[2])
                    rq.append(("throttle", it[1]))
                elif it[0] == "raw":
                    buf += it[1]
                    rq.append(("throttle", "shared:0"))
                else:
                    buf += it[1]
                    rq.append(("cmd", None))
            conns.append(("resp", buf))
        elif p == "http":
            buf, rq = b"", []
            for it in items:
                if it[0] == "throttle":
                    buf += request(body_of(it[1], 2, 1, 60, it[2]))
                    rq.append(("throttle", it[1]))
                elif it[0] == "esc":
                    buf += request(it[1])
                    rq.append(("throttle", "shared:0"))
                else:
                    buf += it[1]
                    rq.append(("uncounted", None))
            conns.append(("http", buf))
        else:
            cn = gs.established()
            blk = gs.steady_block(cn.hpack)
            sid, rq = 3, {}
            for it in items:
                q = 1 if it[2] is None else it[2]
                cn.buf += gs.call(sid, blk, request_bytes(it[1], 2, 1, 60, q))
                rq[sid] = it[1]
                sid += 2
            # last, a call on the general HTTP/2 path: its header block inserts into the HPACK table
            rq[sid] = rng.choice(S)
            cn.buf += gs.call(sid, gs.lit(b"x-new", b"v", 0x40) + blk, request_bytes(rq[sid], 2, 1, 60, 1))
            conns.append(("grpc", cn))
        reqs.append(rq)
    return conns, reqs


def _http_responses(out):
    i, got = 0, []
    while i < len(out):
        head_end = out.index(b"\r\n\r\n", i)
        head = out[i:head_end].decode()
        n = int(re.search(r"content-length: (\d+)", head).group(1))
        got.append((int(head.split(" ")[1]), out[head_end + 4:head_end + 4 + n]))
        i = head_end + 4 + n
    return got


def _events(conns, reqs, got):
    """(transport, key, outcome) per counted request, outcome "allowed", "denied" or "error", read from the replies"""
    ev = []
    for (p, cn), rq, g in zip(conns, reqs, got):
        if p == "resp":
            out, pos, k = g[0], 0, 0
            while pos < len(out):
                v, n = RespParser().parse(out[pos:])
                pos += n
                kind, key = rq[k]
                k += 1
                denied = v[0] == "array" and v[1][0][1] == 0
                ev.append(("redis", key, "denied" if denied else "allowed"))
            assert k == len(rq)
        elif p == "http":
            resps = _http_responses(g[0])
            assert len(resps) == len(rq)
            for (kind, key), (status, body) in zip(rq, resps):
                if kind != "throttle":
                    continue
                if status == 500:
                    ev.append(("http", key, "error"))
                else:
                    assert status == 200
                    ev.append(("http", key, "allowed" if json.loads(body)["allowed"] else "denied"))
        else:
            out, i, seen = bytes(cn.out), 0, set()
            while i < len(out):
                n = int.from_bytes(out[i:i + 3], "big")
                ftype, sid = out[i + 3], int.from_bytes(out[i + 5:i + 9], "big") & 0x7fffffff
                payload = out[i + 9:i + 9 + n]
                if sid in rq and sid not in seen:
                    if ftype == gt.DATA:
                        seen.add(sid)
                        ev.append(("grpc", rq[sid], "allowed" if payload[5:7] == b"\x08\x01" else "denied"))
                    elif ftype == gt.HEADERS and b"Rate%20limiter%20error" in payload:
                        seen.add(sid)
                        ev.append(("grpc", rq[sid], "error"))
                i += 9 + n
            assert seen == set(rq)
    return ev


def _model_text(ev):
    """metrics.rs:233-310 over the events (uptime masked; top keys as (escaped key, count))"""
    by = {"http": 0, "grpc": 0, "redis": 0}
    tot = {"allowed": 0, "denied": 0, "error": 0}
    den = {}
    for t, key, o in ev:
        by[t] += 1
        tot[o] += 1
        if o == "denied" and key is not None and len(key.encode()) <= 256:
            den[key] = den.get(key, 0) + 1
    head = ("# HELP throttlecrab_uptime_seconds Time since server start in seconds\n"
            "# TYPE throttlecrab_uptime_seconds gauge\nthrottlecrab_uptime_seconds U\n\n"
            "# HELP throttlecrab_requests_total Total number of requests processed\n"
            "# TYPE throttlecrab_requests_total counter\nthrottlecrab_requests_total %d\n\n"
            "# HELP throttlecrab_requests_by_transport Total requests by transport type\n"
            "# TYPE throttlecrab_requests_by_transport counter\n"
            'throttlecrab_requests_by_transport{transport="http"} %d\n'
            'throttlecrab_requests_by_transport{transport="grpc"} %d\n'
            'throttlecrab_requests_by_transport{transport="redis"} %d\n\n'
            "# HELP throttlecrab_requests_allowed Total requests allowed\n"
            "# TYPE throttlecrab_requests_allowed counter\nthrottlecrab_requests_allowed %d\n\n"
            "# HELP throttlecrab_requests_denied Total requests denied\n"
            "# TYPE throttlecrab_requests_denied counter\nthrottlecrab_requests_denied %d\n\n"
            "# HELP throttlecrab_requests_errors Total internal errors\n"
            "# TYPE throttlecrab_requests_errors counter\nthrottlecrab_requests_errors %d\n\n"
            "# HELP throttlecrab_top_denied_keys Top keys by denial count\n"
            "# TYPE throttlecrab_top_denied_keys gauge\n") % (
        len(ev), by["http"], by["grpc"], by["redis"], tot["allowed"], tot["denied"], tot["error"])

    def esc(s):
        return "".join({'"': '\\"', "\\": "\\\\", "\n": "\\n", "\r": "\\r", "\t": "\\t"}.get(
            ch, "\\x%02x" % (ord(ch) & 0xff) if ord(ch) < 0x20 or 0x7f <= ord(ch) <= 0x9f else ch) for ch in s)
    return head, {(esc(k), n) for k, n in den.items()}


def test_end_to_end_metrics_text_of_the_mixed_driver(k1_path):
    rng = random.Random(7)
    lim = _engine()
    m = Metrics(lim, 100)
    ring = tc.MixedRing(lim, 1, 64, 1 << 20, 4096)
    conns, reqs = _e2e_conns(rng)
    got = mixed.process_connections(conns, lim, NOW, ring, metrics=m)
    ev = _events(conns, reqs, got)
    assert {o for _, _, o in ev} == {"allowed", "denied", "error"}
    scrape = mixed.process_connections([("http", b"GET /metrics HTTP/1.1\r\nHost: x\r\n\r\n")], lim, NOW, ring,
                                       metrics=m)
    (status, body), = _http_responses(scrape[0][0])
    assert status == 200
    text = re.sub(r"throttlecrab_uptime_seconds \d+\n", "throttlecrab_uptime_seconds U\n", body.decode())
    head, top = _model_text(ev)
    assert text.startswith(head)
    lines = text[len(head):].splitlines()
    parsed = [re.fullmatch(r'throttlecrab_top_denied_keys\{key="(.*)",rank="(\d+)"\} (\d+)', ln) for ln in lines]
    assert all(parsed) and [int(x.group(2)) for x in parsed] == list(range(1, len(lines) + 1))
    counts = [int(x.group(3)) for x in parsed]
    assert counts == sorted(counts, reverse=True)                # (tied ranks: compared as a set)
    assert {(x.group(1), int(x.group(3))) for x in parsed} == top
    assert any(k.startswith("q") for k, _ in top)               # the escaped key, named on the GPU
