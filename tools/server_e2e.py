"""End-to-end load on the server (python -m throttlecrab_b200.server) against a Python selectors loop over
mixed.process_connections, both as subprocesses on 127.0.0.1, alternated over repetitions.

Two client shapes, each client a process of its own:
  - blocking: 32 clients per protocol, each one connection sending one request and waiting for its reply, --requests
    requests each (the reference's docs/benchmark-results.md shape): req/s and P50/P90/P99/P99.9 latency per protocol;
  - pipelined: 3 x --conns connections (RESP, HTTP, gRPC), each sending --depth requests at once and reading the replies.
Every request must get exactly one reply.  Prints the GPU, its power limit and the host CPU count, one JSON line per
run.  Usage: python tools/server_e2e.py [--reps 2] [--requests 10000] [--conns 4096] [--depth 8]
[--device 0 --device 0,1 ...]: with --device, the native server at each of the given --device values instead, the
servers alternated as above (rep 0 in the given order, rep 1 reversed, ...).
"""
import argparse
import json
import multiprocessing as mp
import os
import re
import resource
import selectors
import signal
import socket
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from throttlecrab_b200 import grpc_transport as gt  # noqa: E402
import grpc_streams as gs  # noqa: E402
from grpc_server import request_bytes  # noqa: E402

TRANSPORTS = ("Redis", "HTTP", "gRPC")
REPLY_MARK = {"Redis": b"*5\r\n", "HTTP": b"HTTP/1.1 ", "gRPC": b"grpc-status"}


# ---- requests ----------------------------------------------------------------------------------------------------------
def resp_req(key):
    parts = [b"THROTTLE", key.encode(), b"100000", b"1000000", b"60"]
    return b"*5\r\n" + b"".join(b"$%d\r\n%s\r\n" % (len(p), p) for p in parts)


def http_req(key):
    body = b'{"key": "%s", "max_burst": 100000, "count_per_period": 1000000, "period": 60}' % key.encode()
    return b"POST /throttle HTTP/1.1\r\nHost: x\r\nContent-Type: application/json\r\nContent-Length: %d\r\n\r\n%s" \
        % (len(body), body)


class GrpcCalls:
    """a client connection's HTTP/2 bytes: the opening (preface, SETTINGS, a first call that fills the HPACK table),
    then plain calls on the next odd streams"""

    def __init__(self, key):
        dec = gt.Decoder()
        first = gs.first_block()
        dec.decode(first)
        self.block, self.sid, self.key = gs.steady_block(dec), 1, key
        self.opening = gt.PREFACE + gt.frame(gt.SETTINGS, 0, 0) + gs.call(1, first, self._msg())

    def _msg(self):
        return request_bytes(self.key, 100000, 1000000, 60, 1)

    def next(self):
        self.sid += 2
        return gs.call(self.sid, self.block, self._msg())


# ---- clients -----------------------------------------------------------------------------------------------------------
def _recv_until(s, buf, mark, count):
    while buf.count(mark) < count:
        d = s.recv(1 << 16)
        if not d:
            raise ConnectionError("closed with %d of %d replies" % (buf.count(mark), count))
        buf += d
    return buf


def blocking_client(transport, port, n, key, q):
    """one connection, one request at a time -> (latencies in ns, replies)"""
    s = socket.create_connection(("127.0.0.1", port))
    s.setsockopt(socket.IPPROTO_TCP, socket.TCP_NODELAY, 1)
    mark, buf, lat = REPLY_MARK[transport], bytearray(), []
    g = GrpcCalls(key) if transport == "gRPC" else None
    if g:                                                  # (the opening call is not timed)
        s.sendall(g.opening)
        buf = _recv_until(s, buf, mark, 1)
    base = buf.count(mark)
    for i in range(n):
        req = resp_req(key) if transport == "Redis" else http_req(key) if transport == "HTTP" else g.next()
        t = time.perf_counter_ns()
        s.sendall(req)
        buf = _recv_until(s, buf, mark, base + i + 1)
        lat.append(time.perf_counter_ns() - t)
    s.close()
    q.put((lat, buf.count(mark) - base))


def pipelined_client(transport, port, conns, depth, tag, q):
    """`conns` connections, each sending `depth` requests at once -> replies per connection"""
    socks = []
    for c in range(conns):
        s = socket.create_connection(("127.0.0.1", port))
        key = "%s:%d" % (tag, c)
        if transport == "gRPC":
            g = GrpcCalls(key)
            data = g.opening + b"".join(g.next() for _ in range(depth - 1))
        else:
            one = resp_req(key) if transport == "Redis" else http_req(key)
            data = one * depth
        socks.append((s, data))
    t = time.perf_counter_ns()
    for s, data in socks:
        s.sendall(data)
    got = []
    for s, _ in socks:
        buf = _recv_until(s, bytearray(), REPLY_MARK[transport], depth)
        got.append(buf.count(REPLY_MARK[transport]))
        s.close()
    q.put((time.perf_counter_ns() - t, got))


def run_clients(target, argsets):
    q = mp.Queue()
    ps = [mp.Process(target=target, args=a + (q,)) for a in argsets]
    for p in ps:
        p.start()
    out = [q.get(timeout=600) for _ in ps]
    for p in ps:
        p.join(30)
        if p.is_alive():
            p.kill()
    return out


# ---- the baseline: a Python selectors loop over mixed.process_connections ------------------------------------------------
def baseline_server(buffer_size):
    import throttlecrab_b200 as tc
    from throttlecrab_b200 import mixed
    from throttlecrab_b200.metrics import Metrics
    from throttlecrab_b200.server import MAX_CONNS, IN_CAPACITY
    lim = tc.RateLimiter(tc.PeriodicStore(capacity=100_000))
    ring = tc.MixedRing(lim, 1, MAX_CONNS, IN_CAPACITY, buffer_size)
    metrics = Metrics(lim, 100)
    sel = selectors.DefaultSelector()
    for name, proto in zip(TRANSPORTS, ("resp", "http", "grpc")):
        ls = socket.socket()
        ls.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        ls.bind(("127.0.0.1", 0))
        ls.listen(1024)
        ls.setblocking(False)
        sel.register(ls, selectors.EVENT_READ, ("listen", proto))
        print("Starting %s transport on 127.0.0.1:%d" % (name, ls.getsockname()[1]), flush=True)
    stop = []
    signal.signal(signal.SIGTERM, lambda *_: stop.append(1))
    conns = {}                                             # socket -> [protocol, pending bytes or Connection, order]
    order = 0
    while not stop:
        ready = []
        for key, _ in sel.select(0.1):
            kind, proto = key.data
            if kind == "listen":
                while True:
                    try:
                        s, _ = key.fileobj.accept()
                    except BlockingIOError:
                        break
                    s.setblocking(False)
                    conns[s] = [proto, gt.Connection() if proto == "grpc" else bytearray(), order]
                    order += 1
                    sel.register(s, selectors.EVENT_READ, ("conn", proto))
                continue
            s = key.fileobj
            st = conns[s]
            room = 65536 - (len(st[1].buf) if proto == "grpc" else len(st[1]))
            if room:
                try:
                    d = s.recv(room)
                except (BlockingIOError, ConnectionError):
                    continue
                if not d:
                    sel.unregister(s)
                    s.close()
                    del conns[s]
                    continue
                (st[1].buf if proto == "grpc" else st[1]).extend(d)
            ready.append(s)
        if not ready:
            continue
        ready.sort(key=lambda s: conns[s][2])
        batch = [(conns[s][0], conns[s][1] if conns[s][0] == "grpc" else bytes(conns[s][1])) for s in ready]
        got = mixed.process_connections(batch, lim, time.time_ns(), ring, metrics=metrics)
        for s, (p, _), g in zip(ready, batch, got):
            st = conns[s]
            if p == "grpc":
                out, st[1].out = bytes(st[1].out), bytearray()
            else:
                out = g[0]
                del st[1][:g[1]]
            s.setblocking(True)
            s.sendall(out)
            s.setblocking(False)
    for s in conns:
        s.close()


# ---- runs --------------------------------------------------------------------------------------------------------------
def start(kind, buffer_size):
    if kind != "python":                                   # "native", or "native --device D"
        cmd = [sys.executable, "-m", "throttlecrab_b200.server", "--redis", "--http", "--grpc",
               "--buffer-size", str(buffer_size)] + kind.split()[1:]
        for t in ("redis", "http", "grpc"):
            cmd += ["--%s-host" % t, "127.0.0.1", "--%s-port" % t, "0"]
    else:
        cmd = [sys.executable, os.path.abspath(__file__), "--baseline-server", "--buffer-size", str(buffer_size)]
    p = subprocess.Popen(cmd, cwd=ROOT, stdout=subprocess.PIPE, text=True)
    ports = {}
    while len(ports) < 3:
        ln = p.stdout.readline()
        if not ln:
            p.kill()
            raise RuntimeError("%s server did not start" % kind)
        m = re.search(r"Starting (\S+) transport on 127\.0\.0\.1:(\d+)", ln)
        if m:
            ports[m.group(1)] = int(m.group(2))
    return p, ports


def stop(p):
    p.send_signal(signal.SIGTERM)
    try:
        p.wait(30)
    except subprocess.TimeoutExpired:
        p.kill()
        p.wait(10)
    p.stdout.close()


def pct(xs, q):
    return xs[min(len(xs) - 1, int(q * len(xs)))]


def one_run(kind, a, rep):
    p, ports = start(kind, a.buffer_size)
    try:
        res = {"server": kind, "rep": rep}
        for t in TRANSPORTS:
            t0 = time.perf_counter()
            out = run_clients(blocking_client, [(t, ports[t], a.requests, "b%d:%s:%d" % (rep, t, c))
                                                for c in range(a.clients)])
            wall = time.perf_counter() - t0
            lat = sorted(x for lt, _ in out for x in lt)
            assert all(n == a.requests for _, n in out), "a blocking client lost replies"
            res[t] = {"req_s": round(len(lat) / wall), "p50_us": pct(lat, .5) / 1e3, "p90_us": pct(lat, .9) / 1e3,
                      "p99_us": pct(lat, .99) / 1e3, "p999_us": pct(lat, .999) / 1e3}
        per = max(1, a.conns // a.procs)
        t0 = time.perf_counter()
        out = run_clients(pipelined_client, [(t, ports[t], per, a.depth, "p%d:%s:%d" % (rep, t, k))
                                             for t in TRANSPORTS for k in range(a.procs)])
        wall = time.perf_counter() - t0
        got = [n for _, g in out for n in g]
        assert all(n == a.depth for n in got), "a pipelined connection got a wrong number of replies"
        res["pipelined"] = {"conns": len(got), "requests": sum(got), "req_s": round(sum(got) / wall)}
        return res
    finally:
        stop(p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--clients", type=int, default=32)
    ap.add_argument("--requests", type=int, default=10_000)
    ap.add_argument("--conns", type=int, default=4096)
    ap.add_argument("--depth", type=int, default=8)
    ap.add_argument("--procs", type=int, default=8, help="client processes per protocol, pipelined shape")
    ap.add_argument("--buffer-size", type=int, default=100_000)
    ap.add_argument("--device", action="append", help="the native server's --device (repeat to compare several)")
    ap.add_argument("--baseline-server", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.baseline_server:
        return baseline_server(a.buffer_size)
    soft, hard = resource.getrlimit(resource.RLIMIT_NOFILE)
    resource.setrlimit(resource.RLIMIT_NOFILE, (hard, hard))     # (this process and its children only)
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True).stdout.strip()
    except OSError:
        gpu = "unknown"
    print(json.dumps({"gpu": gpu, "cpus": os.cpu_count(), "nofile": hard}), flush=True)
    kinds = ["native --device " + d for d in a.device] if a.device else ["native", "python"]
    for rep in range(a.reps):
        for kind in (kinds if rep % 2 == 0 else kinds[::-1]):
            print(json.dumps(one_run(kind, a, rep)), flush=True)


if __name__ == "__main__":
    main()
