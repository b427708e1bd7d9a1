"""The native server (gcra_server_*, throttlecrab_b200.server.Server) on 127.0.0.1 with ephemeral ports and a fixed
clock, driven by raw-socket clients (and grpcio).  A serve over the buffered bytes must be exactly
mixed.process_connections over those connections in accept order at the same clock: every client must receive the
bytes a replay engine's process_connections gives them, with the same ring geometry and metrics.  Then the bytes
split across many reads and serves, grpcio calls, the connections' lifecycle (half-close, backpressure, a full buffer
without progress, a port in use, no descriptor left behind) and the subprocess CLI."""
import os
import random
import re
import select
import signal
import socket
import subprocess
import sys
import threading
import time
import types

import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import grpc_transport as gt
from throttlecrab_b200 import mixed
from throttlecrab_b200 import server as S
from throttlecrab_b200.metrics import Metrics
import grpc_streams as gs
from grpc_server import request_bytes, throttle_stub
from test_http_cpu import body_of, request
from test_mixed_cpu import http_conn, resp_conn
from test_resp import _cmd, _throttle

pytestmark = [pytest.mark.gpu, pytest.mark.parametrize("k1_path", ["auto"], indirect=True)]
NS = 10**9
NOW = 1_700_000_000 * NS
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROTO = {"resp": "redis", "http": "http", "grpc": "grpc"}


def _engine(max_conns=512, in_capacity=1 << 22, row_capacity=1 << 14):
    lim = tc.RateLimiter(tc.PeriodicStore(capacity=1 << 14, created_ns=NOW, max_batch=1 << 16))
    ring = tc.MixedRing(lim, 1, max_conns, in_capacity, row_capacity)
    return lim, ring, Metrics(lim, 100)


def _server(geometry=None, metrics=True):
    lim, ring, m = _engine(**(geometry or {}))
    srv = S.Server(ring, [(t, "127.0.0.1", 0) for t in ("redis", "http", "grpc")], m if metrics else None)
    return srv, lim, m


# ---- client traffic --------------------------------------------------------------------------------------------------
def grpc_client(rng, keys, n, tail=True):
    """what a client sends on a new connection: the preface, SETTINGS, a first call whose block inserts into the
    HPACK table, n plain calls (with a PING and split DATA), maybe a SETTINGS and a call with one more insert"""
    dec = gt.Decoder()
    first = gs.first_block()
    dec.decode(first)
    out = gt.PREFACE + gt.frame(gt.SETTINGS, 0, 0) + gs.call(1, first, request_bytes(rng.choice(keys), 3, 10, 60, 1))
    st = types.SimpleNamespace(last_stream=1, hpack=dec)
    out += gs.steady_stream(rng, st, n, keys)
    if tail and rng.random() < 0.5:
        out += gt.frame(gt.SETTINGS, 0, 0)
        out += gs.call(3 + 2 * n, gs.lit(b"x-new", b"v", 0x40) + gs.steady_block(dec),
                       request_bytes(rng.choice(keys), 3, 10, 60, 1))
    return out


def traffic(rng, n_conns, shared=True, per_conn=(0, 12), metrics=True, closers=True):
    """[(protocol, bytes)]: plain and general requests; keys shared across protocols, or distinct per connection;
    closers: some connections end with a request that closes them (QUIT, a protocol error, HTTP/1.0, GOAWAY)"""
    out = []
    for c in range(n_conns):
        p = rng.choice(["resp", "http", "grpc"])
        tag = "shared" if shared else "%s%d" % (p, c)
        n = rng.randint(*per_conn)
        if p == "resp":
            b = resp_conn(rng, tag, n)
            b += rng.choice([b"", _cmd("PING")] + ([_cmd("QUIT") + _throttle(tag + ":after", 3, 10, 60),
                                                   b"*1\r\n$x\r\n"] if closers else []))
        elif p == "http":
            b = http_conn(rng, tag, n)
            b += rng.choice([b"", b"GET /health HTTP/1.1\r\nHost: x\r\n\r\n"]
                            + ([request(body_of(tag + ":10", 3, 10, 60)).replace(b"HTTP/1.1", b"HTTP/1.0"),
                                b"POST /throttle HTTP/1.1\r\nContent-Length: 3\r\n\r\n{x}"] if closers else [])
                            + ([b"GET /metrics HTTP/1.1\r\nHost: x\r\n\r\n"] if metrics else []))
        else:
            b = grpc_client(rng, ["%s:%d" % (tag, i) for i in range(3)], n)
            if closers and rng.random() < 0.15:
                b += gt.frame(gt.DATA, 0, 0, b"x")                       # DATA on stream 0: GOAWAY
        out.append((p, b))
    return out


def replay(conns, geometry=None, metrics=True, now=NOW):
    """each connection's reply bytes from mixed.process_connections on a fresh engine of the same geometry"""
    lim, ring, m = _engine(**(geometry or {}))
    cs = [(p, gt.Connection()) if p == "grpc" else (p, b) for p, b in conns]
    for (p, b), (_, cn) in zip(conns, cs):
        if p == "grpc":
            cn.buf += b
    got = mixed.process_connections(cs, lim, now, ring, metrics=m if metrics else None)
    return [bytes(cn.out) if p == "grpc" else g[0] for (p, cn), g in zip(cs, got)], m


def split_replay(conns, points):
    """each connection's reply bytes from mixed.process_connections called at every serve over what it had buffered
    then (the keys are distinct per connection, so the connections' replays do not interact)"""
    lim, ring, _ = _engine()
    cs = [gt.Connection() if p == "grpc" else None for p, _ in conns]
    pos, out, closed = [0] * len(conns), [bytearray() for _ in conns], [False] * len(conns)
    for pt in points:
        for c, (p, b) in enumerate(conns):
            if closed[c]:
                continue
            if p == "grpc":
                cs[c].buf += b[pos[c]:pt[c]]
                pos[c] = pt[c]
                mixed.process_connections([(p, cs[c])], lim, NOW, ring)
                out[c] += cs[c].out
                cs[c].out.clear()
                closed[c] = cs[c].closed
            elif pt[c] > pos[c]:
                reply, used, _, close = mixed.process_connections([(p, b[pos[c]:pt[c]])], lim, NOW, ring)[0]
                out[c] += reply
                pos[c] += used
                closed[c] = close is not None
    return [bytes(o) for o in out]


def _uptime(b):
    return re.sub(rb"throttlecrab_uptime_seconds \d+", b"throttlecrab_uptime_seconds U", b)


# ---- a harness over one Server ---------------------------------------------------------------------------------------
class Clients:
    def __init__(self, srv):
        self.srv, self.socks, self.got, self.sent = srv, [], [], 0

    def connect(self, protocol):
        """a new client, accepted before the next one (so accept order is list order)"""
        s = socket.create_connection(("127.0.0.1", self.srv.port(PROTO[protocol])))
        s.setblocking(False)
        want = self.srv.stats()["accepted"] + 1
        self.until(lambda st: st["accepted"] >= want)
        self.socks.append(s)
        self.got.append(bytearray())
        return s

    def until(self, cond, timeout=20):
        t = time.time() + timeout
        while not cond(self.srv.stats()):
            assert time.time() < t, self.srv.stats()
            self.srv.read(5)

    def send(self, i, data):
        self.socks[i].setblocking(True)
        self.socks[i].sendall(data)
        self.socks[i].setblocking(False)
        self.sent += len(data)

    def buffered(self):
        """read until every byte sent is in the server's buffers"""
        self.until(lambda st: st["bytes_read"] >= self.sent)

    def drain(self, want_len=None, timeout=20):
        """read every client's socket until `want_len` bytes arrived on each (or nothing more comes for a while)"""
        t, quiet = time.time() + timeout, 0
        while time.time() < t:
            self.srv.read(0)
            r, _, _ = select.select([s for s in self.socks if s.fileno() >= 0], [], [], 0.02)
            for s in r:
                i = self.socks.index(s)
                try:
                    d = s.recv(1 << 20)
                except BlockingIOError:
                    continue
                except ConnectionResetError:
                    d = b""
                if not d:
                    s.close()
                self.got[i] += d
            if want_len is not None and all(len(g) >= n for g, n in zip(self.got, want_len)):
                return
            quiet = quiet + 1 if not r else 0
            if want_len is None and quiet > 25:
                return

    def close(self):
        for s in self.socks:
            s.close()


def _equivalence(seed, n_conns, geometry=None, per_conn=(0, 12)):
    rng = random.Random(seed)
    conns = traffic(rng, n_conns, per_conn=per_conn)
    srv, _, m = _server(geometry)
    cl = Clients(srv)
    try:
        for p, _ in conns:
            cl.connect(p)
        for i, (_, b) in enumerate(conns):
            cl.send(i, b)
        cl.buffered()
        srv.serve(NOW)
        want, m2 = replay(conns, geometry)
        cl.drain([len(w) for w in want])
        for i, (w, g) in enumerate(zip(want, cl.got)):
            assert _uptime(bytes(g)) == _uptime(w), (i, conns[i][0])
        st = srv.stats()
        assert st["general_errors"] == 0 and st["submits"] >= 1
        # GET /metrics over the HTTP port: the text the replay engine's Metrics gives
        k = len(cl.socks)
        cl.connect("http")
        cl.send(k, b"GET /metrics HTTP/1.1\r\nHost: x\r\n\r\n")
        cl.buffered()
        srv.serve(NOW)
        cl.drain()
        body = bytes(cl.got[k]).split(b"\r\n\r\n", 1)[1]
        assert _uptime(body) == _uptime(m2().encode())
        assert b"throttlecrab_requests_denied" in body
        return st
    finally:
        cl.close()
        srv.close()


def test_serve_is_process_connections_over_accept_order():
    st = _equivalence(1, 24)
    assert st["general_calls"] > 0


def test_more_connections_than_max_conns():
    st = _equivalence(2, 40, {"max_conns": 7})
    assert st["submits"] >= 6


def test_more_bytes_than_in_capacity():
    st = _equivalence(3, 12, {"in_capacity": 1 << 16}, per_conn=(100, 200))
    assert st["submits"] > st["rounds"]


def test_row_capacity_forcing_stop_3():
    st = _equivalence(4, 16, {"row_capacity": 5})
    assert st["rounds"] > 3


def test_byte_splits_across_reads_and_serves():
    rng = random.Random(5)
    conns = traffic(rng, 18, shared=False, metrics=False, closers=False)   # (every byte sent is read)
    srv, _, _ = _server(metrics=False)
    cl = Clients(srv)
    try:
        for p, _ in conns:
            cl.connect(p)
        at, points = [0] * len(conns), []                 # points: each serve's bytes per connection
        while any(a < len(b) for a, (_, b) in zip(at, conns)):
            i = rng.choice([c for c in range(len(conns)) if at[c] < len(conns[c][1])])
            n = rng.randint(1, 400)
            cl.send(i, conns[i][1][at[i]:at[i] + n])
            at[i] = min(at[i] + n, len(conns[i][1]))
            if rng.random() < 0.4:
                cl.buffered()
                srv.serve(NOW)
                points.append(list(at))
        cl.buffered()
        srv.serve(NOW)
        points.append(list(at))
        want = split_replay(conns, points)
        cl.drain([len(w) for w in want])
        for i, (w, g) in enumerate(zip(want, cl.got)):
            assert bytes(g) == w, (i, conns[i][0])
        assert srv.stats()["general_errors"] == 0
    finally:
        cl.close()
        srv.close()


def test_grpcio_unary_calls():
    grpc = pytest.importorskip("grpc")
    srv, _, _ = _server()
    keys = ["g%d" % (i % 5) for i in range(60)]
    reqs = [request_bytes(k, 3, 10, 60, 1) for k in keys]
    results, errors = [], []

    def client():
        try:
            with grpc.insecure_channel("127.0.0.1:%d" % srv.port("grpc")) as ch:
                stub = throttle_stub(ch)
                for r in reqs:
                    results.append(stub(r, timeout=10))
        except Exception as e:                             # (reported below)
            errors.append(e)
    th = threading.Thread(target=client, daemon=True)
    th.start()
    try:
        t = time.time() + 60
        while th.is_alive() and time.time() < t:
            srv.poll(5, NOW)
        th.join(5)
        assert not th.is_alive() and not errors, errors
        # the same calls one by one on a replay engine
        lim, ring, m = _engine()
        want = []
        for k in keys:
            row = tc.np.zeros(1, tc.REQ_DTYPE)
            row[0] = (lim.store.hash_key(k.encode()), 3, 10, 60, 1, NOW)
            res = lim.rate_limit_batch(row)
            out, _ = gt.format_replies(row, res, [1])
            h = 9 + int.from_bytes(out[0:3], "big")         # HEADERS, then DATA: the gRPC message
            n = int.from_bytes(out[h:h + 3], "big")
            want.append(out[h + 9 + 5:h + 9 + n])
        assert [bytes(r) for r in results] == want
    finally:
        srv.close()


def test_half_close_after_pipelined_requests():
    srv, _, _ = _server()
    cl = Clients(srv)
    try:
        cl.connect("resp")
        cl.send(0, b"".join(_throttle("hc:%d" % (i % 4), 3, 10, 60) for i in range(200)))
        cl.socks[0].shutdown(socket.SHUT_WR)
        t = time.time() + 20
        while cl.socks[0].fileno() >= 0 and time.time() < t:
            srv.poll(5, NOW)
            cl.drain()
        assert cl.got[0].count(b"*5\r\n") == 200
        assert srv.stats()["open"] == 0 and srv.stats()["closed"] == 1
    finally:
        cl.close()
        srv.close()


def test_backpressure_on_a_client_that_does_not_read():
    srv, _, _ = _server()
    cl = Clients(srv)
    n = 100_000                                            # (HTTP: more replies than the sockets' buffers hold)
    data = b"".join(request(body_of("bp:%d" % (i % 50), 1000, 10, 60)) for i in range(n))
    s = cl.connect("http")
    sender = threading.Thread(target=lambda: cl.send(0, data))
    sender.start()
    try:
        last, still = -1, 0
        while still < 40:                                  # until the server stops reading
            srv.poll(5, NOW)
            b = srv.stats()["bytes_read"]
            still = still + 1 if b == last else 0
            last = b
        st = srv.stats()
        assert st["bytes_read"] < len(data)
        assert 0 < st["peak_unsent"] < S.OUT_BOUND
        got, k = bytearray(), 0
        t = time.time() + 120
        while k < n and time.time() < t:
            srv.poll(1, NOW)
            while select.select([s], [], [], 0)[0]:       # (the sender thread keeps the socket blocking)
                d = s.recv(1 << 20)
                got += d
                if not d or len(d) < 1 << 20:
                    break
            k = got.count(b"HTTP/1.1 ")
        sender.join(20)
        assert k == n
        assert srv.stats()["peak_unsent"] < S.OUT_BOUND
    finally:
        sender.join(20)
        cl.close()
        srv.close()


def test_full_buffer_without_progress_closes():
    srv, _, _ = _server()
    cl = Clients(srv)
    try:
        cl.connect("resp")
        cl.connect("http")
        cl.send(0, b"*2\r\n$4\r\nPING\r\n$70000\r\n" + b"x" * 65600)          # a bulk string past the buffer
        cl.send(1, b"GET /health HTTP/1.1\r\nX: " + b"y" * 70000)             # a header that never ends
        t = time.time() + 20
        while srv.stats()["full_closed"] < 2 and time.time() < t:
            srv.poll(5, NOW)
        cl.drain()
        assert srv.stats()["full_closed"] == 2 and srv.stats()["open"] == 0
        assert [s.fileno() for s in cl.socks] == [-1, -1]   # both saw EOF
    finally:
        cl.close()
        srv.close()


def _fds():
    return len(os.listdir("/proc/self/fd"))


def test_port_in_use_is_refused_and_ports_bind_again_after_destroy():
    lim, ring, m = _engine()

    def ping(srv):
        c = socket.create_connection(("127.0.0.1", srv.port("redis")))
        c.sendall(_cmd("PING"))
        srv.poll(50, NOW)
        srv.poll(50, NOW)
        assert c.recv(100) == b"+PONG\r\n"
        c.close()
    warm = S.Server(ring, [("redis", "127.0.0.1", 0)], m)    # (the device's first work opens what it opens)
    ping(warm)
    warm.close()
    before = _fds()
    busy = socket.socket()
    busy.bind(("127.0.0.1", 0))
    busy.listen(1)
    with pytest.raises(tc.Internal, match="bind"):
        S.Server(ring, [("redis", "127.0.0.1", 0), ("http", "127.0.0.1", busy.getsockname()[1])])
    busy.close()
    assert _fds() == before
    with pytest.raises(tc.Internal, match="twice"):
        S.Server(ring, [("redis", "127.0.0.1", 0), ("redis", "127.0.0.1", 0)])
    srv = S.Server(ring, [(t, "127.0.0.1", 0) for t in ("redis", "http", "grpc")], m)
    ports = [srv.port(t) for t in ("redis", "http", "grpc")]
    ping(srv)
    srv.close()
    assert _fds() <= before
    again = S.Server(ring, [(t, "127.0.0.1", p) for t, p in zip(("redis", "http", "grpc"), ports)], m)
    assert [again.port(t) for t in ("redis", "http", "grpc")] == ports
    again.close()
    assert _fds() <= before
    # a ring that is not mixed is refused
    lim2 = tc.RateLimiter(tc.PeriodicStore(capacity=64, created_ns=NOW, max_batch=1024))
    r2 = tc.RespRing(lim2, 1, 8, 1 << 16, 64)
    with pytest.raises(tc.Internal, match="not a mixed ring"):
        S.Server(r2, [("redis", "127.0.0.1", 0)])


def test_general_path_exception_closes_only_its_connection(monkeypatch):
    srv, _, _ = _server()
    cl = Clients(srv)
    try:
        cl.connect("resp")
        cl.connect("resp")
        real = S._resp.general

        def boom(data, *a):
            if b"boom" in data:
                raise ValueError("boom")
            return real(data, *a)
        monkeypatch.setattr(S._resp, "general", boom)
        cl.send(0, _throttle("e:0", 3, 10, 60) + _cmd("ECHO", "boom"))
        cl.send(1, _throttle("e:1", 3, 10, 60) + _cmd("PING"))
        cl.buffered()
        with pytest.raises(S.GeneralPathError, match="connection 0"):
            srv.serve(NOW)
        cl.drain()
        assert cl.socks[0].fileno() == -1 and cl.got[0] == b""
        assert cl.got[1].endswith(b"+PONG\r\n") and cl.got[1].startswith(b"*5\r\n")
        assert srv.stats()["general_errors"] == 1 and srv.stats()["open"] == 1
    finally:
        cl.close()
        srv.close()


def test_subprocess_cli_answers_and_exits_on_sigterm():
    args = [sys.executable, "-m", "throttlecrab_b200.server", "--redis", "--http", "--grpc",
            "--buffer-size", "4096", "--store-capacity", "1000"]
    for t in ("redis", "http", "grpc"):
        args += ["--%s-host" % t, "127.0.0.1", "--%s-port" % t, "0"]
    p = subprocess.Popen(args, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        ports, lines, t = {}, [], time.time() + 120
        while len(ports) < 3 and time.time() < t:
            ln = p.stdout.readline()
            assert ln, "".join(lines)
            lines.append(ln)
            m = re.search(r"Starting (\w+) transport on 127\.0\.0\.1:(\d+)", ln)
            if m:
                ports[m.group(1)] = int(m.group(2))
        assert sorted(ports) == ["HTTP", "Redis", "gRPC"], lines

        def ask(port, data, until):
            with socket.create_connection(("127.0.0.1", port), timeout=20) as s:
                s.sendall(data)
                got = b""
                while not until(got):
                    d = s.recv(4096)
                    assert d, got
                    got += d
                return got
        assert ask(ports["Redis"], _cmd("PING"), lambda g: b"\r\n" in g) == b"+PONG\r\n"
        r = ask(ports["Redis"], _throttle("sub", 3, 10, 60), lambda g: g.count(b"\r\n") >= 6)
        assert r.startswith(b"*5\r\n:1\r\n:3\r\n")                          # allowed, limit 3
        h = ask(ports["HTTP"], b"GET /health HTTP/1.1\r\nHost: x\r\n\r\n", lambda g: g.endswith(b"OK"))
        assert h.startswith(b"HTTP/1.1 200")
        rng = random.Random(6)
        g = ask(ports["gRPC"], grpc_client(rng, ["sub"], 0, tail=False), lambda g: b"grpc-status" in g)
        assert gt.frame(gt.SETTINGS, 0, 0) in g
        p.send_signal(signal.SIGTERM)
        assert p.wait(20) == 0
    finally:
        if p.poll() is None:
            p.kill()
            p.wait(10)
        p.stdout.close()
