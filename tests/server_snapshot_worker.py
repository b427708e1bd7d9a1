"""Child process of tests/test_gpu_server_snapshots.py: servers built by server.serve_config with --snapshot-dir, on
`world` engines of cuda:0, restarted into another world size, against a control server on one engine that never
restarts.  Every serve opens fresh RESP, HTTP and gRPC connections on both servers, sends the same bytes (Zipf keys in
one namespace per client, some with entries that live an hour and some that expire within seconds), serves at the
same clock and compares every reply byte.

    server_snapshot_worker.py restart OLD NEW    final save, then a background save whose cut is replayed
    server_snapshot_worker.py failed WORLD       a save that cannot create its generation

Prints "server snapshot ok"."""
import argparse
import json
import os
import random
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from throttlecrab_b200 import persist as P  # noqa: E402
from throttlecrab_b200 import server as S  # noqa: E402
from test_gpu_server import NOW, NS, Clients, grpc_client  # noqa: E402
from test_http_cpu import body_of, request  # noqa: E402
from test_resp import _throttle  # noqa: E402

ROUNDS, CUT, DOWNTIME = 6, 2, 10 * NS          # serves before the restart; the background save's serve; the clock jump


class Log:
    def __init__(self):
        self.lines = []

    def _add(self, kind, fmt, *a):
        self.lines.append((kind, fmt % a if a else fmt))

    def info(self, fmt, *a):
        self._add("info", fmt, *a)

    def warning(self, fmt, *a):
        self._add("warning", fmt, *a)


def config(world, snapshot_dir=None):
    argv = ["--redis", "--http", "--grpc", "--buffer-size", "4096", "--store-capacity", "4096",
            "--device", ",".join(["0"] * world)]
    for t in ("redis", "http", "grpc"):
        argv += ["--%s-host" % t, "127.0.0.1", "--%s-port" % t, "0"]
    if snapshot_dir:
        argv += ["--snapshot-dir", snapshot_dir]
    return S.parse_config(argv, {"CUDA_DEVICE_MAX_CONNECTIONS": "32"})


def _key(rng, c):
    """a Zipf-skewed key of client c; odd ranks are short-lived (burst 2, 1 per second), even ones live an hour"""
    k = min(int(rng.paretovariate(1.1)) - 1, 40)
    return "c%d:%d" % (c, k), ((2, 1, 1) if k % 2 else (3, 10, 3600))


def traffic(rng, clients=9):
    """one serve's connections: [(protocol, bytes)]; client c's keys are its own, so the order in which a sharded
    serve takes the connections does not change a decision"""
    out = []
    for c in range(clients):
        p = ("resp", "http", "grpc")[c % 3]
        n = rng.randint(4, 24)
        if p == "grpc":
            out.append((p, grpc_client(rng, ["c%d:g%d" % (c, min(int(rng.paretovariate(1.1)), 6)) for _ in range(8)],
                                       n, tail=False)))
            continue
        b = b""
        for _ in range(n):
            key, (mb, cnt, per) = _key(rng, c)
            b += _throttle(key, mb, cnt, per) if p == "resp" else request(body_of(key, mb, cnt, per))
        out.append((p, b))
    return out


class Served:
    """one server and its clients: serve(conns, now) -> each connection's reply bytes"""

    def __init__(self, srv, stores):
        self.srv, self.stores, self.cl = srv, stores, Clients(srv)

    def serve(self, conns, now, want=None):
        first = len(self.cl.socks)
        for p, _ in conns:
            self.cl.connect(p)
        for i, (_, b) in enumerate(conns):
            self.cl.send(first + i, b)
        self.cl.buffered()
        self.srv.serve(now)
        self.cl.drain(None if want is None else [len(g) for g in self.cl.got[:first]] + [len(w) for w in want])
        got = [bytes(g) for g in self.cl.got[first:]]
        for s in self.cl.socks[first:]:
            s.close()
        return got

    def close(self, stores=True):
        self.cl.close()
        self.srv.close()
        if stores:
            for st in reversed(self.stores):
                st.close()


def manifest(d):
    with open(os.path.join(d, "MANIFEST")) as f:
        return json.load(f)


def start(world, d, log):
    sd = P.SnapshotDir(d, "periodic", log)
    srv, stores = S.serve_config(config(world, d), log, sd)
    return Served(srv, stores), sd


def same(ctl, x, conns, now):
    want = ctl.serve(conns, now)
    got = x.serve(conns, now, want)
    for i, (w, g) in enumerate(zip(want, got)):
        assert g == w, (i, conns[i][0], now, w[:200], g[:200])
    return want


def scenario_restart(old, new):
    for mode in ("final", "background"):
        rng = random.Random(100 * old + new + (mode == "final"))
        log = Log()
        d = tempfile.mkdtemp(prefix="snap-")
        ctl = Served(*S.serve_config(config(1), log))
        a, sd = start(old, d, log)
        rounds = [traffic(rng) for _ in range(ROUNDS)]
        replies = []
        for i, conns in enumerate(rounds):
            replies.append(same(ctl, a, conns, NOW + i * NS // 10))
            if mode == "background":
                if i == CUT:
                    assert sd.begin()
                sd.poll()
        denied = b"".join(r for r, (p, _) in zip(replies[-1], rounds[-1]) if p == "resp").count(b"*5\r\n:0\r\n")
        assert denied > 0, "no key is denied at the restart"
        if mode == "final":
            a.srv.close()                                  # (as main: the sockets, then the save, then the stores)
            assert sd.save() == 1
            a.close()
        else:
            t = time.time() + 60
            while sd.in_flight():
                assert time.time() < t
                sd.poll()
                time.sleep(0.01)
            assert sd.generation == 1, log.lines
            a.close()                                      # (no shutdown save: the background one is restored)
        sd.close()
        m = manifest(d)
        assert m["world"] == old and m["generation"] == 1 and len(m["files"]) == old
        assert sorted(os.listdir(d)) == ["LOCK", "MANIFEST", "gen-1"]

        b, sd = start(new, d, log)
        assert sd.generation == 1 and any("Restored snapshot generation 1" in t for _, t in log.lines), log.lines
        if mode == "final":
            assert sum(st.len() for st in b.stores) == ctl.stores[0].len() > 0
        else:                                              # the cut is the serve boundary: replay what came after it
            for i in range(CUT + 1, ROUNDS):
                got = b.serve(rounds[i], NOW + i * NS // 10, replies[i])
                assert got == replies[i], i
        for i in range(ROUNDS, ROUNDS + 4):                # after the downtime: short-lived entries have expired
            same(ctl, b, traffic(rng), NOW + DOWNTIME + i * NS // 10)
        b.srv.close()
        assert sd.save() == 2
        b.close()
        sd.close()
        ctl.close()
        assert manifest(d)["world"] == new
        shutil.rmtree(d)
        print("%s %d -> %d: %d serves equal" % (mode, old, new, ROUNDS + 4))


def scenario_failed(world):
    rng = random.Random(7 + world)
    log = Log()
    d = tempfile.mkdtemp(prefix="snap-")
    ctl = Served(*S.serve_config(config(1), log))
    a, sd = start(world, d, log)
    rounds = [traffic(rng) for _ in range(ROUNDS)]
    replies = []
    for i, conns in enumerate(rounds):
        replies.append(same(ctl, a, conns, NOW + i * NS // 10))
        if i == CUT:
            assert sd.begin()
            t = time.time() + 60
            while sd.poll() is None:
                assert time.time() < t
                time.sleep(0.01)
            assert sd.generation == 1
            with open(os.path.join(d, "gen-2"), "w") as f:           # mkdir of the next generation fails
                f.write("in the way")
        if i == CUT + 1:
            assert not sd.begin()
            assert any(k == "warning" and "generation 2 failed" in t for k, t in log.lines), log.lines
    assert manifest(d)["generation"] == 1 and sd.generation == 1
    a.close()
    sd.close()
    ctl.close()
    b, sd = start(world, d, log)                           # the committed generation: the cut after serve CUT
    assert sd.generation == 1
    for i in range(CUT + 1, ROUNDS):
        assert b.serve(rounds[i], NOW + i * NS // 10, replies[i]) == replies[i], i
    b.close()
    sd.close()
    shutil.rmtree(d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("scenario", choices=["restart", "failed"])
    ap.add_argument("worlds", type=int, nargs="+")
    a = ap.parse_args()
    globals()["scenario_" + a.scenario](*a.worlds)
    print("server snapshot ok: %s %s" % (a.scenario, a.worlds))


if __name__ == "__main__":
    main()
