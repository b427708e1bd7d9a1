"""The gRPC ring (gcra_grpc_ring_*) against the host walk (gcra_grpc_parse_throttle), and served to grpcio clients."""
import random
import threading

import numpy as np
import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import grpc_transport as gt
import grpc_streams as gs_
from grpc_server import Server, request_bytes, throttle_stub

pytestmark = pytest.mark.gpu
NS = 10**9
T0 = 1_700_000_000 * NS


def _ring(max_batch=1 << 14, row_capacity=4096, max_conns=64, in_capacity=1 << 20, seed=(0, 0)):
    lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 14, created_ns=T0, max_batch=max_batch, hash_seed=seed))
    return lim, tc.GrpcRing(lim, 1, max_conns, in_capacity, row_capacity)


def _conns(rng, n):
    """connections in several shapes: steady streams, cut anywhere, with near misses, windows nearly spent"""
    out = []
    keys = ["k%d" % i for i in range(20)] + ["été", ""]
    for c in range(n):
        cn = gs_.established()
        data = gs_.steady_stream(rng, cn, rng.randint(0, 40), keys)
        shape = c % 6
        if shape == 1:
            data = data[:rng.randint(0, len(data))]
        elif shape == 2:
            data += gt.frame(gt.SETTINGS, 0, 0) + data[:30]
        elif shape == 3:
            cn.send_window = rng.randint(0, 400)
        elif shape == 4:
            cn.init_window = rng.choice([0, 50, 51])
        elif shape == 5:
            data += gs_.call(cn.last_stream, gs_.steady_block(cn.hpack), b"")      # a stream id reused
        cn.buf += data
        out.append(cn)
    return out


def _expected(lim, conns, row_cap, now):
    """each connection's host walk at the row cap the earlier ones leave, keys hashed with the engine's seed"""
    L = tc._native.lib()
    exp, base = [], 0
    for cn in conns:
        row = cn.conn_row()
        data = bytes(cn.buf)
        req = np.zeros(len(data) // 26 + 1, tc.REQ_DTYPE)
        sids = np.zeros(len(req), np.uint32)
        o = np.zeros((), tc.GRPC_OUTCOME_DTYPE)
        assert L.gcra_grpc_parse_throttle(lim._h, data, len(data), now, row_cap - base, row.ctypes.data,
                                          req.ctypes.data, sids.ctypes.data, o.ctypes.data) == 0
        n = int(o["n_frames"])
        exp.append((o, req[:n].copy(), sids[:n].copy()))
        base += n
    return exp


@pytest.mark.parametrize("seed,row_cap,hash_seed", [(1, 4096, (0, 0)), (2, 37, (0, 0)), (3, 1, (5, 7)),
                                                    (4, 300, (5, 7))])
def test_ring_takes_what_the_host_walk_takes(seed, row_cap, hash_seed):
    import oracle
    rng = random.Random(seed)
    lim, ring = _ring(row_capacity=row_cap, seed=hash_seed)
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=1 << 14, created_ns=T0, p0=NS)
    allowed = denied = 0
    for rnd in range(3):
        conns = _conns(rng, 24)
        now = T0 + rnd * NS
        exp = _expected(lim, conns, row_cap, now)
        used = 0
        for j, cn in enumerate(conns):
            data = bytes(cn.buf)
            ring.input[0][used:used + len(data)] = np.frombuffer(data, np.uint8)
            ring.conns[0][j]["off"], ring.conns[0][j]["len"] = used, len(data)
            cn.state(ring.conns[0][j])
            used += len(data)
        ring.submit(0, len(conns), now)
        ring.wait(0)
        req, res = ring.rows(0)
        base = 0
        for j, (o, ereq, esids) in enumerate(exp):
            g = ring.outcome[0][j]
            for f in ("consumed", "n_frames", "stop", "data_octets", "last_stream", "send_window", "ping"):
                assert int(g[f]) == int(o[f]), (seed, rnd, j, f, int(g[f]), int(o[f]))
            assert bytes(g["ping_opaque"]) == bytes(o["ping_opaque"])
            n = len(ereq)
            assert np.array_equal(req[base:base + n], ereq), (seed, rnd, j)
            want, sent = gt.format_replies(req[base:base + n], res[base:base + n], esids)
            off, ln = int(g["reply_off"]), int(g["reply_len"])
            assert ring.replies[0][off:off + ln].tobytes() == want, (seed, rnd, j)
            assert int(g["data_sent"]) == sent
            base += n
        assert len(req) == base
        # the batch's decisions, replayed in row order on the oracle (a key is its hash under the engine's seed)
        for q, r in zip(req, res):
            want = ora.rate_limit("h%d" % int(q["key_hash"]), int(q["max_burst"]), int(q["count_per_period"]),
                                  int(q["period"]), int(q["quantity"]), int(q["now_ns"]))
            got = (int(r["status"]), bool(r["allowed"]), int(r["remaining"]), int(r["reset_after_ns"]),
                   int(r["retry_after_ns"]))
            assert got == want, (seed, rnd, q)
            allowed += want[0] == tc.OK and want[1]
            denied += want[0] == tc.OK and not want[1]
    st = lim.store.stats()
    assert (st["allowed"], st["denied"]) == (allowed, denied)


def test_refused_submits_leave_the_ring_usable():
    lim, ring = _ring()
    cn = gs_.established()
    cn.buf += gs_.steady_stream(random.Random(0), cn, 3, ["a"])
    data = bytes(cn.buf)
    ring.input[0][:len(data)] = np.frombuffer(data, np.uint8)
    ring.conns[0][0]["off"], ring.conns[0][0]["len"] = 0, len(data)
    cn.state(ring.conns[0][0])
    ring.conns[0][0]["n_dyn"] = 129
    with pytest.raises(Exception):
        ring.submit(0, 1, T0)
    ring.conns[0][0]["n_dyn"] = 6
    ring.conns[0][0]["len"] = 65537
    with pytest.raises(Exception):
        ring.submit(0, 1, T0)
    ring.conns[0][0]["len"] = len(data)
    ring.submit(0, 1, T0)
    ring.wait(0)
    assert int(ring.outcome[0][0]["n_frames"]) == 3 and int(ring.outcome[0][0]["stop"]) == 0


def _oracle_replies(calls):
    """the response messages the oracle gives for (key, max_burst, count, period, quantity) calls in order, all at T0"""
    import oracle
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=1000, created_ns=T0, p0=NS)
    req = np.zeros(len(calls), tc.REQ_DTYPE)
    res = np.zeros(len(calls), tc.RES_DTYPE)
    for i, (k, b, c, p, q) in enumerate(calls):
        s, a, rem, reset, retry = ora.rate_limit(k, b, c, p, q, T0)
        req[i] = (0, b, c, p, q, T0)
        res[i] = (rem, reset, retry, s, a, [0, 0, 0])
    out, _ = gt.format_replies(req, res, np.ones(len(calls), np.uint32))
    msgs, i = [], 0
    while i < len(out):
        n = int.from_bytes(out[i:i + 3], "big")
        if out[i + 3] == gt.DATA:
            msgs.append(out[i + 14:i + 9 + n])
        i += 9 + n
    return msgs


@pytest.mark.parametrize("seed", [(0, 0), (11, 13)])
def test_grpcio_clients_served_by_the_ring(seed):
    grpc = pytest.importorskip("grpc")
    lim, ring = _ring(row_capacity=1024, seed=seed)
    srv = Server(lim, ring, now_ns=lambda: T0)
    allowed, errors, shared, own = [], [], [], {}

    def client(i):
        try:
            ch = grpc.insecure_channel("127.0.0.1:%d" % srv.port)
            stub = throttle_stub(ch)
            own[i] = []
            for k in range(15):
                r = stub(request_bytes("shared", 5, 10, 3600, 1), timeout=10)
                shared.append(r)
                allowed.append(r[:2] == b"\x08\x01")
                own[i].append(stub(request_bytes("own%d" % i, 3, 10, 3600, 1), timeout=10))
            try:
                stub(request_bytes("neg", 3, 10, 3600, -2), timeout=10)
                errors.append("no error")
            except grpc.RpcError as e:
                if e.code() != grpc.StatusCode.INTERNAL or \
                        e.details() != "Rate limiter error: Rate limit check failed: negative quantity: -2":
                    errors.append((e.code(), e.details()))
            ch.close()
        except Exception as e:                         # noqa: BLE001  (reported below)
            errors.append(repr(e))

    ts = [threading.Thread(target=client, args=(i,)) for i in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(60)
    srv.close()
    assert not any(t.is_alive() for t in ts)
    assert not errors, errors
    assert len(allowed) == 60 and sum(allowed) == 5           # the reference's burst test, across shared clients
    # every response against the oracle: a client's own key in its order; the shared key's 60 responses as a multiset
    # (the server decides the clients' calls in the order they arrive)
    for i in range(4):
        assert own[i] == _oracle_replies([("own%d" % i, 3, 10, 3600, 1)] * 15), i
    assert sorted(shared) == sorted(_oracle_replies([("shared", 5, 10, 3600, 1)] * 60))


@pytest.mark.parametrize("use_ring", [False, True])
def test_seeded_engine_one_identity_per_key(use_ring):
    """a connection's first call (a table insert: the general path) and its later calls (the host walk or the ring)
    count against one entry under the engine's seed"""
    grpc = pytest.importorskip("grpc")
    lim, ring = _ring(row_capacity=256, seed=(123, 456))
    srv = Server(lim, ring if use_ring else None, now_ns=lambda: T0)
    try:
        ch = grpc.insecure_channel("127.0.0.1:%d" % srv.port)
        stub = throttle_stub(ch)
        got = [stub(request_bytes("rate_limit_test", 5, 10, 60, 1), timeout=10) for _ in range(15)]
        ch.close()
    finally:
        srv.close()
    assert sum(r[:2] == b"\x08\x01" for r in got) == 5
    assert got == _oracle_replies([("rate_limit_test", 5, 10, 60, 1)] * 15)


def test_captured_grpcio_stream_ring_against_host_walk():
    import os
    with open(os.path.join(os.path.dirname(__file__), "golden", "grpcio_throttle_stream.bin"), "rb") as f:
        raw = f.read()
    outs = []
    for use_ring in (False, True):
        lim, ring = _ring(row_capacity=64, seed=(3, 4))
        cn = gt.Connection()
        n = 0
        for i in range(0, len(raw), 500):
            cn.buf += raw[i:i + 500]
            n += gt.process_connections([cn], lim, T0, ring if use_ring else None)[0]
        assert n == 41 and not cn.closed
        outs.append(bytes(cn.out))
    assert outs[0] == outs[1]
