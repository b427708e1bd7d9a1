"""mixed.process_connections without a GPU (ring=None: each connection's host walk, decided by an oracle-backed
limiter): every protocol's connections answered as their own paths answer them, and one key's limit shared by RESP,
HTTP and gRPC connections in the documented decision order (the reference's multi_transport.rs:159-225)."""
import copy
import json
import random

import pytest

import oracle
import throttlecrab_b200 as tc
from throttlecrab_b200 import grpc_transport as gt
from throttlecrab_b200 import http, mixed
from throttlecrab_b200.resp import RespParser, process_pipeline
import grpc_streams as gs
from grpc_server import request_bytes
from test_http_cpu import NEAR_MISSES, body_of, request
from test_resp import OracleEngine, _FakeLimiter, _FakeStore, _cmd, _throttle

NS = 10**9
NOW = 1_700_000_000 * NS


class _Store(_FakeStore):
    def hash_key(self, kb):
        return tc.hash_key(kb)


class Limiter(_FakeLimiter):
    """test_resp's _FakeLimiter (the oracle standing in for the engine) with the store's hash_key, which the general
    paths use"""

    def __init__(self):
        super().__init__()
        self.store = _Store()


# ---- connections of each protocol ------------------------------------------------------------------------------------
def resp_conn(rng, tag, n, general=True):
    """n THROTTLE frames on keys of its own, some for the general path (PING, RESP integers), maybe a split tail"""
    frames = [_throttle("%s:%d" % (tag, rng.randrange(3)), rng.choice([1, 3, 5]), 10, 60,
                        rng.choice([None, 1, 2, -1])) for _ in range(n)]
    if general and n:
        for _ in range(rng.randrange(3)):
            frames.insert(rng.randrange(len(frames) + 1),
                          rng.choice([_cmd("PING"), _cmd("THROTTLE", "%s:int" % tag, 3, 10, 60), _cmd("UNKNOWN")]))
    buf = b"".join(frames)
    if general and rng.random() < 0.2:
        buf += _throttle("%s:tail" % tag, 3, 10, 60)[:-3]
    return buf


def http_conn(rng, tag, n, general=True):
    """n POST /throttle requests on keys of its own, some for the general path (/health, 404, quantity null,
    escapes), maybe a split tail"""
    reqs = [request(body_of("%s:%d" % (tag, rng.randrange(3)), rng.choice([1, 3, 5]), 10, 60,
                            rng.choice([None, 1, 2]))) for _ in range(n)]
    if general and n:
        for _ in range(rng.randrange(3)):
            reqs.insert(rng.randrange(len(reqs) + 1), rng.choice([
                b"GET /health HTTP/1.1\r\nHost: x\r\n\r\n", b"GET /nope HTTP/1.1\r\nHost: x\r\n\r\n",
                request(b'{"key": "%s:\\u0065", "max_burst": 3, "count_per_period": 10, "period": 60}'
                        % tag.encode())]))
    buf = b"".join(reqs)
    if general and rng.random() < 0.2:
        buf += request(body_of("%s:tail" % tag))[:-4]
    return buf


def grpc_conn(rng, tag, n, general=True):
    """an established connection with n calls on keys of its own; maybe a SETTINGS frame (the general path) and a
    call whose header block inserts into the HPACK table"""
    cn = gs.established()
    data = gs.steady_stream(rng, cn, n, ["%s:%d" % (tag, i) for i in range(3)])
    if general and rng.random() < 0.4:
        data += gt.frame(gt.SETTINGS, 0, 0)
        data += gs.call(cn.last_stream + 2 * n + 2, gs.lit(b"x-new", b"v", 0x40) + gs.steady_block(cn.hpack),
                        request_bytes("%s:ins" % tag, 3, 10, 60, 1))
    cn.buf += data
    return cn


def mix(rng, n_conns, per_conn=(0, 12), general=True):
    out = []
    for c in range(n_conns):
        p = rng.choice(["resp", "http", "grpc"])
        n = rng.randint(*per_conn)
        tag = "%s%d" % (p, c)
        out.append((p, {"resp": resp_conn, "http": http_conn, "grpc": grpc_conn}[p](rng, tag, n, general)))
    return out


def copy_conns(conns):
    """the same connections, gRPC ones as copies of their Connection objects"""
    return [(p, copy.deepcopy(cn) if p == "grpc" else cn) for p, cn in conns]


# ---- tests -----------------------------------------------------------------------------------------------------------
def _http_general(buf, lim):
    """an HTTP connection through the general path alone, one request after another"""
    pos, out, n, close = 0, [], 0, None
    while pos < len(buf) and close is None:
        g = http.general(buf[pos:], lim, NOW)
        if g is None:
            break
        used, reply, k, close = g
        pos += used
        out.append(reply)
        n += k
    return b"".join(out), pos, n, close


def test_each_protocol_as_its_own_path_on_disjoint_keys():
    """with keys of its own, every connection gets what its protocol's own path gives it over the same bytes"""
    rng = random.Random(5)
    for rnd in range(4):
        conns = mix(rng, 24)
        if rnd == 0:
            conns.append(("http", b"".join(NEAR_MISSES[k] for k in sorted(NEAR_MISSES)[:12])))
            conns.append(("resp", _throttle("q:1", 3, 10, 60) + _cmd("QUIT") + _throttle("q:1", 3, 10, 60)))
            conns.append(("resp", _throttle("g:1", 3, 10, 60) + b"?garbage\r\n"))
            conns.append(("resp", b""))
        ref = copy_conns(conns)
        got = mixed.process_connections(conns, Limiter(), NOW, None)
        lim = Limiter()
        for c, ((p, cn), (_, rc)) in enumerate(zip(conns, ref)):
            if p == "resp":
                assert got[c] == process_pipeline(cn, OracleEngine(), NOW), (rnd, c)
            elif p == "http":
                assert got[c] == _http_general(cn, lim), (rnd, c)
            else:
                n = gt.process_connections([rc], lim, NOW, None)[0]
                assert got[c] == n and bytes(cn.out) == bytes(rc.out) and bytes(cn.buf) == bytes(rc.buf), (rnd, c)
                assert (cn.last_stream, cn.send_window, cn.closed) == (rc.last_stream, rc.send_window, rc.closed)
                assert cn.hpack.classes() == rc.hpack.classes()


def _allowed_resp(out):
    p, flags, pos = RespParser(), [], 0
    while pos < len(out):
        v, k = p.parse(out[pos:])
        flags.append(v[1][0][1] == 1)
        pos += k
    return flags


def _allowed_http(out):
    return [json.loads(part.split(b"}", 1)[0] + b"}")["allowed"] for part in out.split(b"\r\n\r\n")[1::1]
            if part.startswith(b"{")]


def _allowed_grpc(out):
    flags, i = [], 0
    while i < len(out):
        n = int.from_bytes(out[i:i + 3], "big")
        if out[i + 3] == gt.DATA:
            flags.append(out[i + 14:i + 16] == b"\x08\x01")
        i += 9 + n
    return flags


def shared_key_conns(n_conns, n_requests, health_at=None):
    """n_requests for shared_test_key (max_burst 100, 10 per 60 s, quantity 1), request i on connection i % n_conns,
    connection c of protocol c % 3 (RESP, HTTP, gRPC); health_at: an HTTP connection index that gets a GET /health
    after its first request.  Returns the connections and each connection's request numbers."""
    per = [[i for i in range(n_requests) if i % n_conns == c] for c in range(n_conns)]
    conns = []
    for c in range(n_conns):
        k = len(per[c])
        if c % 3 == 0:
            conns.append(("resp", _throttle("shared_test_key", 100, 10, 60, 1) * k))
        elif c % 3 == 1:
            one = request(body_of("shared_test_key", 100, 10, 60, 1))
            buf = one * k
            if c == health_at:
                buf = one + b"GET /health HTTP/1.1\r\nHost: x\r\n\r\n" + one * (k - 1)
            conns.append(("http", buf))
        else:
            cn = gs.established()
            blk = gs.steady_block(cn.hpack)
            cn.buf += b"".join(gs.call(3 + 2 * j, blk, request_bytes("shared_test_key", 100, 10, 60, 1))
                               for j in range(k))
            conns.append(("grpc", cn))
    return conns, per


def allowed_flags(conns, got):
    flags = []
    for (p, cn), g in zip(conns, got):
        flags.append(_allowed_resp(g[0]) if p == "resp" else _allowed_http(g[0]) if p == "http"
                     else _allowed_grpc(bytes(cn.out)))
    return flags


def decision_order(per, health_at=None):
    """the documented order: every connection's plain prefix in list order, then (after the /health the general path
    answers) the rest of the connection that stopped there"""
    order = []
    for c, reqs in enumerate(per):
        order += reqs[:1] if c == health_at else reqs
    if health_at is not None:
        order += per[health_at][1:]
    return order


def test_one_limit_shared_by_all_three_transports():
    """200 requests for one key, round-robin over RESP, HTTP and gRPC connections at one now: the per-request allowed
    flags are a sequential oracle replay in the documented order, and exactly 100 are limited"""
    for n_conns, health_at in ((3, None), (6, None), (200, None), (6, 4)):
        conns, per = shared_key_conns(n_conns, 200, health_at)
        got = mixed.process_connections(conns, Limiter(), NOW, None)
        flags = allowed_flags(conns, got)
        assert [len(f) for f in flags] == [len(r) for r in per]
        ora = oracle.OracleStore(oracle.PERIODIC, capacity=1000, created_ns=NOW, p0=NS)
        want = {}
        for i in decision_order(per, health_at):
            want[i] = ora.rate_limit("shared_test_key", 100, 10, 60, 1, NOW)[1]
        for c, reqs in enumerate(per):
            assert flags[c] == [bool(want[i]) for i in reqs], (n_conns, c)
        assert sum(not a for f in flags for a in f) == 100, n_conns


def test_refuses_unknown_protocols_and_long_buffers():
    with pytest.raises(ValueError):
        mixed.process_connections([("smtp", b"HELO")], Limiter(), NOW, None)
    with pytest.raises(ValueError):
        mixed.process_connections([("resp", b"x" * 65537)], Limiter(), NOW, None)
    assert mixed.process_connections([], Limiter(), NOW, None) == []
    assert mixed.PROTOCOLS == {"resp": tc.PROTO_RESP, "http": tc.PROTO_HTTP, "grpc": tc.PROTO_GRPC} == {
        "resp": 1, "http": 2, "grpc": 3}
