"""Child process of tests/test_gpu_sharded_server.py: the native server over `world` engines of one process
(gcra_server_create_sharded, throttlecrab_b200.server.Server over a list of rings), on cuda:0 or one engine per GPU
with --gpus, driven by raw-socket clients on 127.0.0.1 at a fixed clock.  Every serve must give every client exactly
the bytes that mixed.process_connections_sharded gives on fresh engines of the same geometry, with each serve's
connections placed on rank id % world and every rank's policy tick first.

    sharded_server_worker.py SCENARIO WORLD [--gpus]

SCENARIO: serve | splits | sweep | general | refusals.  Prints "sharded server ok"."""
import argparse
import ctypes as C
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
from throttlecrab_b200 import grpc_transport as gt  # noqa: E402
from throttlecrab_b200 import mixed  # noqa: E402
from throttlecrab_b200 import server as S  # noqa: E402
from throttlecrab_b200.metrics import ShardedMetrics  # noqa: E402
from throttlecrab_b200.sharded import connect_local  # noqa: E402
from test_gpu_server import NOW, NS, Clients, _fds, _uptime, traffic  # noqa: E402
from test_resp import _cmd, _throttle  # noqa: E402

GEOMETRY = {"max_conns": 512, "in_capacity": 1 << 22, "row_capacity": 1 << 14}
LISTENS = [(t, "127.0.0.1", 0) for t in ("redis", "http", "grpc")]
SCRAPE = b"GET /metrics HTTP/1.1\r\nHost: x\r\n\r\n"


def engines(world, gpus=False, geoms=None, store=tc.PeriodicStore, **kw):
    """`world` engines connected over peer memory, each with a mixed ring switched to peer-memory ticks; geoms[r]
    overrides rank r's ring geometry"""
    kw = dict(dict(capacity=1 << 14, created_ns=NOW, max_batch=1 << 16), **kw)
    lims = [tc.RateLimiter(store(device=r if gpus else 0, **kw)) for r in range(world)]
    gs = [dict(GEOMETRY, **((geoms or {}).get(r, {}))) for r in range(world)]
    connect_local(lims, max(g["row_capacity"] for g in gs))
    rings = [tc.MixedRing(lim, 1, g["max_conns"], g["in_capacity"], g["row_capacity"]) for lim, g in zip(lims, gs)]
    for ring in rings:
        ring.peer_memory(True)
    return lims, rings


def server(world, gpus=False, geoms=None, metrics=True, **kw):
    lims, rings = engines(world, gpus, geoms, **kw)
    m = ShardedMetrics(lims, 100) if metrics else None
    return S.Server(rings, LISTENS, m), lims, rings


class Replay:
    """the server's serves replayed on fresh engines of the same geometry: each serve is every rank's policy tick,
    then mixed.process_connections_sharded over the connections with pending bytes, connection id on rank id % world,
    in id order; bytes a serve did not take stay pending, and a closed connection takes nothing more"""

    def __init__(self, world, gpus=False, geoms=None, metrics=True, **kw):
        self.world = world
        self.lims, self.rings = engines(world, gpus, geoms, **kw)
        self.metrics = ShardedMetrics(self.lims, 100) if metrics else None
        self.pending, self.kind, self.closed = {}, {}, set()

    def serve(self, sent, now=NOW):
        """sent: {id: (protocol, new bytes)} -> ({id: reply bytes}, per rank the driver's result)"""
        for cid, (p, b) in sent.items():
            self.kind[cid] = p
            if p == "grpc":
                self.pending.setdefault(cid, gt.Connection()).buf += b
            else:
                self.pending[cid] = self.pending.get(cid, b"") + b
        for lim in self.lims:
            lim.store.policy_tick(now)
        per, ids = [[] for _ in range(self.world)], [[] for _ in range(self.world)]
        for cid in sorted(self.pending):
            x = self.pending[cid]
            if cid in self.closed or not (x.buf if self.kind[cid] == "grpc" else x):
                continue
            per[cid % self.world].append((self.kind[cid], x))
            ids[cid % self.world].append(cid)
        got = mixed.process_connections_sharded([(cs, lim, ring) for cs, lim, ring in zip(per, self.lims, self.rings)],
                                                now, metrics=self.metrics)
        out = {}
        for r in range(self.world):
            for cid, (p, x), g in zip(ids[r], per[r], got[r]):
                if p == "grpc":
                    out[cid] = bytes(x.out)
                    x.out.clear()
                    if x.closed:
                        self.closed.add(cid)
                else:
                    out[cid] = g[0]
                    self.pending[cid] = x[g[1]:]
                    if g[3] is not None:
                        self.closed.add(cid)
        return out, got


def check_p2p(lims):
    e = C.c_uint32()
    for r, lim in enumerate(lims):
        lim.store._check(lim._L.gcra_p2p_error(lim._h, C.byref(e)))
        assert e.value == 0, "rank %d: a wait gave up" % r


def hot_elsewhere(lim, world, rank):
    """a key whose owner is not `rank`"""
    L = tc._native.lib()
    return next(k for k in ("hot%d" % i for i in range(1000))
                if L.gcra_owner_of(lim.store.hash_key(k.encode()), world) != rank)


def one_serve(world, conns, gpus=False, geoms=None, metrics=True):
    """every connection's bytes sent and buffered, one serve; its replies against the replay -> (stats, server's
    per-rank counts, replay, clients, server)"""
    srv, lims, _ = server(world, gpus, geoms, metrics)
    cl = Clients(srv)
    for p, _ in conns:
        cl.connect(p)
    for i, (_, b) in enumerate(conns):
        cl.send(i, b)
    cl.buffered()
    srv.serve(NOW)
    rp = Replay(world, gpus, geoms, metrics)
    want, got = rp.serve({i: c for i, c in enumerate(conns)})
    cl.drain([len(want.get(i, b"")) for i in range(len(conns))])
    for i in range(len(conns)):
        assert _uptime(bytes(cl.got[i])) == _uptime(want.get(i, b"")), (i, conns[i][0], i % world)
    check_p2p(lims)
    for r in range(world):                             # each rank's GPU counted the rows of its own connections
        assert (lims[r].store.ring_transport_counts() == rp.lims[r].store.ring_transport_counts()).all(), r
    return srv, lims, rp, cl, got


def scenario_serve(world, gpus):
    """replay with metrics and a key denied on a rank that does not own it; the same serve against ONE engine where no
    slot fills; a rank with more connections than max_conns and more bytes than in_capacity"""
    rng = random.Random(40 + world)
    conns = traffic(rng, 8 * world)
    rank = 1 % world                                   # a rank that parses a key another rank owns, denied often
    probe = tc.RateLimiter(tc.PeriodicStore(capacity=64, created_ns=NOW, max_batch=1024))
    hot = hot_elsewhere(probe, world, rank)
    probe.store.close()
    conns[rank] = ("resp", _throttle(hot, 3, 10, 60) * 20)
    srv, lims, rp, cl, got = one_serve(world, conns, gpus)
    try:
        assert srv.stats()["general_calls"] > 0 and srv.stats()["general_errors"] == 0
        assert all(lims[r].store.ring_transport_counts().sum() > 0 for r in range(world))
        # GET /metrics: the replay's text, the hot key named although its owner parsed none of its bytes
        k = len(cl.socks)
        cl.connect("http")
        cl.send(k, SCRAPE)
        cl.buffered()
        srv.serve(NOW)
        cl.drain()
        want, _ = rp.serve({k: ("http", SCRAPE)})
        assert _uptime(bytes(cl.got[k])) == _uptime(want[k])
        assert ('throttlecrab_top_denied_keys{key="%s"' % hot).encode() in bytes(cl.got[k]), (hot, bytes(cl.got[k]))
    finally:
        cl.close()
        srv.close()
    # no slot fills: ONE engine deciding the joined list (rank-major) gives the same bytes
    conns = traffic(rng, 6 * world, metrics=False)
    srv, lims, rp, cl, got = one_serve(world, conns, gpus, metrics=False)
    try:
        one = tc.RateLimiter(tc.PeriodicStore(capacity=1 << 14, created_ns=NOW, max_batch=1 << 16))
        order = [i for r in range(world) for i in range(len(conns)) if i % world == r]
        joined = [(p, gt.Connection() if p == "grpc" else b) for p, b in (conns[i] for i in order)]
        for (p, cn), i in zip(joined, order):
            if p == "grpc":
                cn.buf += conns[i][1]
        ref = mixed.process_connections(joined, one, NOW, None)
        for (p, cn), g, i in zip(joined, ref, order):
            assert bytes(cl.got[i]) == (bytes(cn.out) if p == "grpc" else g[0]), (i, p)
    finally:
        cl.close()
        srv.close()
    # rank 0: more connections than max_conns and more bytes than in_capacity; the other ranks tick empty meanwhile
    conns = traffic(rng, 14 * world, per_conn=(100, 200))
    geoms = {0: {"max_conns": 5, "in_capacity": 1 << 16}}
    srv, lims, rp, cl, got = one_serve(world, conns, gpus, geoms)
    try:
        st = srv.stats()
        assert st["submits"] > st["rounds"] and st["general_errors"] == 0, st
    finally:
        cl.close()
        srv.close()


def scenario_splits(world, gpus):
    """bytes split across many reads and serves, against the replay of every serve"""
    rng = random.Random(50 + world)
    conns = traffic(rng, 6 * world, shared=False, metrics=False, closers=False)   # (every byte sent is read)
    srv, lims, _ = server(world, gpus, metrics=False)
    rp = Replay(world, gpus, metrics=False)
    cl = Clients(srv)
    try:
        for p, _ in conns:
            cl.connect(p)
        at, sent, want = [0] * len(conns), {}, [bytearray() for _ in conns]

        def serve():
            cl.buffered()
            srv.serve(NOW)
            got, _ = rp.serve(dict(sent))
            sent.clear()
            for i, b in got.items():
                want[i] += b
        while any(a < len(b) for a, (_, b) in zip(at, conns)):
            i = rng.choice([c for c in range(len(conns)) if at[c] < len(conns[c][1])])
            part = conns[i][1][at[i]:at[i] + rng.randint(1, 400)]
            cl.send(i, part)
            at[i] += len(part)
            p, b = sent.get(i, (conns[i][0], b""))
            sent[i] = (p, b + part)
            if rng.random() < 0.4:
                serve()
        serve()
        cl.drain([len(w) for w in want])
        for i, w in enumerate(want):
            assert bytes(cl.got[i]) == bytes(w), (i, conns[i][0])
        assert srv.stats()["general_errors"] == 0
        check_p2p(lims)
    finally:
        cl.close()
        srv.close()


def scenario_sweep(world, gpus):
    """a periodic store (cleanup every second): serves past the interval sweep every rank, decisions as the replay's"""
    rng = random.Random(60 + world)
    srv, lims, _ = server(world, gpus, metrics=False, p0=1)
    rp = Replay(world, gpus, metrics=False, p0=1)
    cl = Clients(srv)
    try:
        swept = []
        for t in range(3):
            now = NOW + t * 600 * NS
            conns = traffic(rng, 4 * world, shared=False, metrics=False, closers=False)
            first = len(cl.socks)
            for p, _ in conns:
                cl.connect(p)
            for i, (_, b) in enumerate(conns):
                cl.send(first + i, b)
            cl.buffered()
            srv.serve(now)
            want, _ = rp.serve({first + i: c for i, c in enumerate(conns)}, now)
            cl.drain([len(cl.got[i]) for i in range(first)] + [len(want.get(first + i, b"")) for i in range(len(conns))])
            for i in range(len(conns)):
                assert bytes(cl.got[first + i]) == want.get(first + i, b""), (t, i)
            assert [lim.store.len() for lim in lims] == [lim.store.len() for lim in rp.lims], t
            swept.append([lim.store.stats()["swept"] for lim in lims])
        # keys of earlier serves have expired: each serve's policy ticks removed some on every rank
        assert all(swept[t][r] > swept[t - 1][r] for t in (1, 2) for r in range(world)), swept
        before = [lim.store.len() for lim in lims]
        assert all(n > 0 for n in before), before
        srv.serve(NOW + 3 * 600 * NS)                   # (no pending bytes: the policy ticks alone)
        rp.serve({}, NOW + 3 * 600 * NS)
        after = [lim.store.len() for lim in lims]
        assert after == [lim.store.len() for lim in rp.lims] and all(a < b for a, b in zip(after, before)), \
            (before, after)
        check_p2p(lims)
    finally:
        cl.close()
        srv.close()


def scenario_general(world, gpus):
    """a failing general path on a rank-1 connection closes only it; the next serve works"""
    srv, lims, _ = server(world, gpus)
    cl = Clients(srv)
    real = S._resp.general

    def boom(data, *a):
        if b"boom" in data:
            raise ValueError("boom")
        return real(data, *a)
    S._resp.general = boom
    try:
        for _ in range(2 * world):
            cl.connect("resp")
        for i in range(2 * world):
            cl.send(i, _throttle("e:%d" % i, 3, 10, 60) + (_cmd("ECHO", "boom") if i == 1 else _cmd("PING")))
        cl.buffered()
        try:
            srv.serve(NOW)
        except S.GeneralPathError as e:
            assert "connection 1" in str(e), e
        else:
            raise AssertionError("no GeneralPathError")
        cl.drain()
        assert cl.socks[1].fileno() == -1 and cl.got[1] == b""
        for i in range(2 * world):
            if i != 1:
                assert cl.got[i].startswith(b"*5\r\n") and cl.got[i].endswith(b"+PONG\r\n"), (i, cl.got[i])
        assert srv.stats()["general_errors"] == 1 and srv.stats()["open"] == 2 * world - 1
        check_p2p(lims)
        n = len(cl.got[0])
        cl.send(0, _throttle("e:0", 3, 10, 60))
        cl.buffered()
        srv.serve(NOW)
        cl.drain([n + 1] + [len(g) for g in cl.got[1:]])
        assert cl.got[0][n:].startswith(b"*5\r\n:1\r\n")
        check_p2p(lims)
    finally:
        S._resp.general = real
        cl.close()
        srv.close()


def scenario_refusals(world, gpus):
    """every refusal of gcra_server_create_sharded: GCRA_INTERNAL, gcra_last_error(hs[0]) says why, no descriptor left
    open; the engines serve afterwards"""
    lims, rings = engines(world, gpus)
    warm = S.Server(rings, LISTENS)                     # (the device's first work opens what it opens)
    warm.close()
    before = _fds()
    L = tc._native.lib()

    def refused(hs, n, match):
        arr = (C.c_void_p * max(len(hs), 1))(*[h.value for h in hs])
        ls = (S._Listen * 1)()
        ls[0].protocol, ls[0].port, ls[0].host = tc.PROTO_RESP, 0, b"127.0.0.1"
        out = C.c_void_p()
        cb = S._GENERAL_FN(lambda *a: 0)
        assert L.gcra_server_create_sharded(arr, n, ls, 1, cb, None, C.byref(out)) == tc.INTERNAL, match
        assert not out.value
        err = L.gcra_last_error(hs[0]).decode()
        assert match in err, (match, err)
        assert _fds() == before, match
    hs = [lim._h for lim in lims]
    refused(hs, 0, "world 0")
    if world > 1:
        refused(hs[:-1], world - 1, "not peer-memory connected")
        refused(hs[::-1], world, "peer-memory rank")
    rings[-1].peer_memory(False)
    refused(hs, world, "not peer-memory ticks")
    rings[-1].peer_memory(True)
    lone = [tc.RateLimiter(tc.PeriodicStore(capacity=64, created_ns=NOW, max_batch=1024)) for _ in range(world)]
    for lim in lone:
        tc.MixedRing(lim, 1, 8, 1 << 16, 256)
    refused([lim._h for lim in lone], world, "not peer-memory connected")
    for kind, match in (("resp", "not a mixed ring"), ("small", "in_capacity")):
        ls = [tc.RateLimiter(tc.PeriodicStore(capacity=64, created_ns=NOW, max_batch=1024)) for _ in range(world)]
        connect_local(ls, 256)
        rs = [tc.RespRing(lim, 1, 8, 1 << 16, 256) if kind == "resp" else tc.MixedRing(lim, 1, 8, 1 << 15, 256)
              for lim in ls]
        for r in rs:
            r.peer_memory(True)
        refused([lim._h for lim in ls], world, match)
        for lim in ls[::-1]:
            lim.store.close()
    # the engines serve afterwards: one request per connection, one connection per rank
    srv = S.Server(rings, LISTENS)
    cl = Clients(srv)
    try:
        for i in range(world):
            cl.connect("resp")
            cl.send(i, _throttle("after:%d" % i, 3, 10, 60))
        cl.buffered()
        srv.serve(NOW)
        cl.drain([len(b"*5\r\n:1\r\n:3\r\n")] * world)
        assert all(g.startswith(b"*5\r\n:1\r\n:3\r\n") for g in cl.got), cl.got
        check_p2p(lims)
    finally:
        cl.close()
        srv.close()
    assert _fds() <= before


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("scenario", choices=["serve", "splits", "sweep", "general", "refusals"])
    ap.add_argument("world", type=int)
    ap.add_argument("--gpus", action="store_true", help="engine r on GPU r")
    a = ap.parse_args()
    globals()["scenario_" + a.scenario](a.world, a.gpus)
    print("sharded server ok: %s, world %d" % (a.scenario, a.world))


if __name__ == "__main__":
    main()
