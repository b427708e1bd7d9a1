"""The mixed ring (gcra_mixed_ring_create + the gcra_resp_ring_* calls): RESP, HTTP and gRPC connections in one slot,
parsed on the GPU, decided as one batch, replies formatted on the GPU.  Every connection must give exactly what its
own protocol's host walk gives at the row cap the connections before it leave -- the same rows, consumed, n_frames
and stop, and for gRPC the whole outcome -- and its replies must be the bytes its protocol's formatter writes for a
twin engine that decided the host-walked rows as one batch."""
import ctypes as C
import random

import numpy as np
import pytest

import oracle
import throttlecrab_b200 as tc
from throttlecrab_b200 import grpc_transport as gt
from throttlecrab_b200 import mixed
import grpc_streams as gs
from test_gpu_grpc_ring import _conns as grpc_conns
from test_gpu_resp_ring import _plain_prefix_of_fuzz
from test_http_cpu import NEAR_MISSES, _fuzz_request, body_of, request
from test_mixed_cpu import allowed_flags, copy_conns, mix, shared_key_conns
from test_resp import _cmd, _throttle

# (auto only: every ring batch takes the index-order pipeline, see test_gpu_resp_ring_inflight.py)
pytestmark = [pytest.mark.gpu, pytest.mark.parametrize("k1_path", ["auto"], indirect=True)]
NS = 10**9
NOW = 1_700_000_000 * NS
SIP = (0x0706050403020100, 0x0f0e0d0c0b0a0908)
P = {"resp": tc.PROTO_RESP, "http": tc.PROTO_HTTP, "grpc": tc.PROTO_GRPC}
MIN_FRAME = {"resp": 45, "http": 133, "grpc": 26}


def _engine(seed=(0, 0), max_batch=1 << 16, capacity=1 << 14):
    return tc.RateLimiter(tc.PeriodicStore(capacity=capacity, created_ns=NOW, max_batch=max_batch, hash_seed=seed))


def _pair(seed, row_capacity, max_conns=512, in_capacity=1 << 22, slots=2):
    lim, twin = _engine(seed), _engine(seed)
    return lim, twin, tc.MixedRing(lim, slots, max_conns, in_capacity, row_capacity)


# ---- connections: (protocol, bytes, gRPC state row or None) -------------------------------------------------------
def _conn(rng, nrng, p):
    if p == "resp":
        return ("resp", _plain_prefix_of_fuzz(nrng, 30), None)
    if p == "http":
        reqs = [_fuzz_request(nrng) if nrng.random() < 0.3 else request(body_of("u%d" % rng.randrange(50)))
                for _ in range(rng.randrange(0, 20))]
        if rng.random() < 0.2:
            reqs.insert(rng.randrange(len(reqs) + 1), NEAR_MISSES[rng.choice(sorted(NEAR_MISSES))])
        buf = b"".join(reqs)
        if rng.random() < 0.3 and len(buf) > 1:
            buf = buf[:rng.randrange(1, len(buf))]
        return ("http", buf, None)
    cn = grpc_conns(rng, rng.randrange(1, 7))[-1]         # (every shape of test_gpu_grpc_ring._conns)
    return ("grpc", bytes(cn.buf), cn.conn_row())


def _fuzz_conns(rng, nrng, n):
    return [_conn(rng, nrng, rng.choice(["resp", "http", "grpc"])) for _ in range(n)]


def _expected(lim, conns, row_cap, now=NOW):
    """each connection's own host walk at the row cap the earlier ones leave: (outcome fields, rows, stream ids,
    gRPC outcome or None)"""
    L, exp, base = lim._L, [], 0
    for p, data, st in conns:
        room = row_cap - base
        req = np.zeros(min(room, len(data) // MIN_FRAME[p]) + 1, tc.REQ_DTYPE)
        if p == "grpc":
            sids = np.zeros(len(req), np.uint32)
            o = np.zeros((), tc.GRPC_OUTCOME_DTYPE)
            assert L.gcra_grpc_parse_throttle(lim._h, data, len(data), now, room, st.ctypes.data, req.ctypes.data,
                                              sids.ctypes.data, o.ctypes.data) == 0
            n = int(o["n_frames"])
            exp.append(((int(o["consumed"]), n, int(o["stop"])), req[:n].copy(), sids[:n].copy(), o))
        else:
            walk = L.gcra_resp_parse_throttle if p == "resp" else L.gcra_http_parse_throttle
            used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
            assert walk(lim._h, data, len(data), now, room, req.ctypes.data, C.byref(used), C.byref(cnt),
                        C.byref(stop)) == 0
            n = cnt.value
            exp.append(((used.value, n, stop.value), req[:n].copy(), None, None))
        base += n
    return exp


def _place(ring, slot, conns):
    """conns into the slot at offsets of every residue mod 16, neighbouring bytes plain requests (a read past a
    connection would show); the gRPC state rows' off and len are garbage (the mixed ring does not read them)"""
    inp = ring.input[slot]
    inp[:] = np.frombuffer((_throttle("spill", 1, 1, 1) * (len(inp) // 40 + 1))[:len(inp)], np.uint8)
    at, k = 0, 0
    for c, (p, data, st) in enumerate(conns):
        at += (5 * c) % 16
        inp[at:at + len(data)] = np.frombuffer(data, np.uint8)
        row = ring.conns[slot][c]
        row["off"], row["len"], row["protocol"], row["grpc_state"] = at, len(data), P[p], k if p == "grpc" else 7
        if p == "grpc":
            ring.grpc_conns[slot][k] = st
            ring.grpc_conns[slot][k]["off"], ring.grpc_conns[slot][k]["len"] = 0xffffffff, 0xfffffff0
            k += 1
        at += len(data)


def _format(p, req, res, sids):
    if p == "grpc":
        return gt.format_replies(req, res, sids)
    L = tc._native.lib()
    fmt = L.gcra_resp_format_replies if p == "resp" else L.gcra_http_format_replies
    buf = C.create_string_buffer(max(len(req), 1) * tc.HTTP_REPLY_MAX)
    w = fmt(np.ascontiguousarray(req).ctypes.data, np.ascontiguousarray(res).ctypes.data, len(req), buf, len(buf))
    return buf.raw[:w], 0


def _check(ring, slot, conns, exp, tres):
    """the slot's outcome, gRPC outcome, rows and replies against the host walks and the twin's results `tres`"""
    rows, res = ring.rows(slot)
    want = np.concatenate([e[1] for e in exp]) if exp else np.zeros(0, tc.REQ_DTYPE)
    assert rows.tobytes() == want.tobytes()
    assert res.tobytes() == tres.tobytes()
    base, k = 0, 0
    for c, ((p, _, _), (fields, req, sids, go)) in enumerate(zip(conns, exp)):
        o = ring.outcome[slot][c]
        assert (int(o["consumed"]), int(o["n_frames"]), int(o["stop"])) == fields, (c, p)
        n = len(req)
        want_bytes, sent = _format(p, req, tres[base:base + n], sids)
        off, ln = int(o["reply_off"]), int(o["reply_len"])
        assert ring.replies[slot][off:off + ln].tobytes() == want_bytes, (c, p)
        if p == "grpc":
            g = ring.grpc_outcome[slot][k]
            for f in ("consumed", "n_frames", "stop", "data_octets", "last_stream", "send_window", "ping"):
                assert int(g[f]) == int(go[f]), (c, f)
            assert bytes(g["ping_opaque"]) == bytes(go["ping_opaque"])
            assert (int(g["reply_off"]), int(g["reply_len"]), int(g["data_sent"])) == (off, ln, sent), c
            k += 1
        base += n
    return rows, res


def _run(lim, twin, ring, slot, conns, now=NOW):
    exp = _expected(lim, conns, ring.row_capacity, now)
    _place(ring, slot, conns)
    ring.submit(slot, len(conns), now)
    ring.wait(slot)
    want = np.concatenate([e[1] for e in exp]) if exp else np.zeros(0, tc.REQ_DTYPE)
    tres = twin.rate_limit_batch(want) if len(want) else np.zeros(0, tc.RES_DTYPE)
    return _check(ring, slot, conns, exp, tres), exp


# ---- 1. the contract over fuzzed mixes ---------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [(0, 0), SIP], ids=["unkeyed", "siphash"])
def test_contract_over_fuzzed_mixes(seed):
    rng, nrng = random.Random(7), np.random.default_rng(20261017)
    lim, twin, ring = _pair(seed, row_capacity=1 << 14)
    for rnd, n in enumerate([0, 1, 3, 17, 64, 200, 5]):
        conns = _fuzz_conns(rng, nrng, n)
        if rnd == 6:
            conns += [("resp", b"", None), ("http", b"", None), ("grpc", b"", gs.established().conn_row())]
            rng.shuffle(conns)
        _run(lim, twin, ring, rnd % 2, conns, NOW + rnd * NS)
    a, b = lim.store.stats(), twin.store.stats()
    assert (a["len"], a["allowed"], a["denied"], a["errors"]) == (b["len"], b["allowed"], b["denied"], b["errors"])


@pytest.mark.parametrize("where", ["resp", "http", "grpc"])
def test_row_cap_stops_inside_a_connection_of_each_protocol(where):
    """row_capacity lands inside the first long connection of `where`: it stops with 3, and every later connection
    takes no rows -- a RESP or HTTP one with bytes stops with 3, a gRPC one where its walk stops at max_frames 0 (3 at
    its first call, 2 at a frame that is not plain before it)"""
    rng, nrng = random.Random(11), np.random.default_rng(11)
    conns = _fuzz_conns(rng, nrng, 40)
    conns.insert(20, {"resp": ("resp", _throttle("cap", 3, 10, 60) * 9, None),
                      "http": ("http", request(body_of("cap")) * 9, None),
                      "grpc": ("grpc", *(lambda cn: (gs.steady_stream(rng, cn, 9, ["cap"]), cn.conn_row()))(
                          gs.established()))}[where])
    probe = _engine(SIP)
    base = sum(len(e[1]) for e in _expected(probe, conns[:20], 1 << 16))
    cap = base + 4
    lim, twin, ring = _pair(SIP, row_capacity=cap)
    _, exp = _run(lim, twin, ring, 0, conns)
    assert exp[20][0][1:] == (4, 3)
    later = [(p, e[0]) for (p, d, _), e in zip(conns[21:], exp[21:]) if d]
    assert all(f[1] == 0 for _, f in later)
    assert all(f[2] == 3 for p, f in later if p != "grpc") and any(f[2] == 3 for p, f in later if p == "grpc")


def test_one_64k_connection_of_each_protocol_in_one_slot():
    rng = random.Random(3)
    one = _throttle("big:r", 5, 10, 60)
    resp = one * (65536 // len(one))
    req = request(body_of("big:h"))
    http_ = req * (65536 // len(req))
    cn = gs.established()
    g = gs.steady_stream(rng, cn, 1200, ["big:g"], extras=False)[:65536]      # (the last call cut: stop 1)
    conns = [("resp", resp, None), ("grpc", g, cn.conn_row()), ("http", http_, None)]
    assert all(len(d) > 65000 for _, d, _ in conns)
    lim, twin, ring = _pair((0, 0), row_capacity=1 << 14, in_capacity=1 << 20)
    _, exp = _run(lim, twin, ring, 0, conns)
    assert all(e[0][1] > 300 for e in exp)


# ---- 2. keys shared across transports, slots in flight -------------------------------------------------------------
def _shared_conn(rng, p):
    keys = ["hot", "hot", "t1", "t2", "cold%d" % rng.randrange(1000)]
    n = rng.randrange(0, 12)
    if p == "resp":
        return ("resp", b"".join(_throttle(rng.choice(keys), rng.choice([1, 4]), 10, 60) for _ in range(n)), None)
    if p == "http":
        return ("http", b"".join(request(body_of(rng.choice(keys), rng.choice([1, 4]), 10, 60)) for _ in range(n)),
                None)
    cn = gs.established()
    return ("grpc", gs.steady_stream(rng, cn, n, keys), cn.conn_row())


@pytest.mark.parametrize("slots", [2, 3])
def test_shared_keys_with_slots_in_flight_against_one_oracle(slots):
    """every slot's results equal one oracle store replaying all rows in submission order and table order"""
    rng = random.Random(slots)
    lim = _engine(SIP)
    ring = tc.MixedRing(lim, slots, 256, 1 << 22, 700)
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=1 << 14, created_ns=NOW, p0=NS)
    for rnd in range(12):
        pending = []
        for s in range(slots):
            now = NOW + (rnd * slots + s) * NS // 3
            conns = [_shared_conn(rng, rng.choice(["resp", "http", "grpc"])) for _ in range(rng.randrange(1, 60))]
            exp = _expected(lim, conns, ring.row_capacity, now)
            _place(ring, s, conns)
            ring.submit(s, len(conns), now)
            want = np.concatenate([e[1] for e in exp])
            ores = np.zeros(len(want), tc.RES_DTYPE)
            for i, q in enumerate(want):
                st, a, rem, reset, retry = ora.rate_limit("h%d" % int(q["key_hash"]), int(q["max_burst"]),
                                                          int(q["count_per_period"]), int(q["period"]),
                                                          int(q["quantity"]), int(q["now_ns"]))
                ores[i] = (rem, reset, retry, st, a, [0, 0, 0])
            pending.append((s, conns, exp, ores))
        for s, conns, exp, ores in pending:
            ring.wait(s)
            _check(ring, s, conns, exp, ores)


# ---- 3. one protocol only ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", ["resp", "http", "grpc"])
def test_one_protocol_only_equals_its_own_ring(p):
    rng, nrng = random.Random(P[p]), np.random.default_rng(P[p])
    lim, twin = _engine(SIP), _engine(SIP)
    ring = tc.MixedRing(lim, 1, 128, 1 << 21, 500)
    own = tc.RespRing(twin, 1, 128, 1 << 21, 500, protocol=p)
    for rnd in range(4):
        conns = [_conn(rng, nrng, p) for _ in range(rng.randrange(1, 100))]
        _place(ring, 0, conns)
        used = 0
        for c, (_, data, st) in enumerate(conns):
            own.input[0][used:used + len(data)] = np.frombuffer(data, np.uint8)
            if p == "grpc":
                own.conns[0][c] = st
            own.conns[0][c]["off"], own.conns[0][c]["len"] = used, len(data)
            used += len(data)
        for r in (ring, own):
            r.submit(0, len(conns), NOW + rnd * NS)
            r.wait(0)
        a, b = ring.rows(0), own.rows(0)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
        total = int(ring.outcome[0][len(conns) - 1]["reply_off"] + ring.outcome[0][len(conns) - 1]["reply_len"])
        assert ring.replies[0][:total].tobytes() == own.replies[0][:total].tobytes()
        for c in range(len(conns)):
            mine, theirs = ring.outcome[0][c], own.outcome[0][c]
            for f in ("consumed", "n_frames", "stop", "reply_off", "reply_len"):
                assert int(mine[f]) == int(theirs[f]), (rnd, c, f)
            if p == "grpc":
                assert ring.grpc_outcome[0][c].tobytes() == theirs.tobytes(), (rnd, c)


# ---- 4. refusals ------------------------------------------------------------------------------------------------------
def test_refused_submits_leave_the_ring_usable():
    rng = random.Random(4)
    lim, twin, ring = _pair((0, 0), row_capacity=256, max_conns=8, in_capacity=1 << 18, slots=1)
    cn = gs.established()
    conns = [("resp", _throttle("v", 3, 10, 60) * 3, None), ("grpc", gs.steady_stream(rng, cn, 3, ["v"]),
                                                              cn.conn_row()),
             ("http", request(body_of("v")) * 3, None), ("grpc", gs.steady_stream(rng, cn, 2, ["w"]), cn.conn_row())]
    _place(ring, 0, conns)
    good = ring.conns[0][:4].copy()

    def refused(n=4):
        with pytest.raises(tc.CellError):
            ring.submit(0, n, NOW)
        ring.conns[0][:4] = good

    for bad in (0, 4, 0xffffffff):
        ring.conns[0][2]["protocol"] = bad
        refused()
    for states in ((1, 0), (0, 0), (0, 2), (1, 2)):
        ring.conns[0][1]["grpc_state"], ring.conns[0][3]["grpc_state"] = states
        refused()
    ring.grpc_conns[0][1]["n_dyn"] = 129
    refused()
    ring.grpc_conns[0][1]["n_dyn"] = conns[3][2]["n_dyn"]
    refused(9)                                              # n_conns > max_conns
    ring.conns[0][0]["len"] = 65537
    refused()
    ring.conns[0][0]["off"] = (1 << 18) - 10
    refused()
    assert lim._L.gcra_ring_submit(lim._h, 0, 1, NOW) != 0
    assert lim._L.gcra_resp_ring_conns(lim._h, 0) is None
    with pytest.raises(tc.CellError):
        tc.RespRing(lim, 1, 8, 1 << 10, 16)
    with pytest.raises(tc.CellError):
        tc.MixedRing(lim, 1, 8, 1 << 10, 16)
    ring.submit(0, 4, NOW)
    with pytest.raises(tc.CellError):                       # the slot is in flight
        ring.submit(0, 4, NOW)
    ring.wait(0)
    exp = _expected(twin, conns, 256)
    want = np.concatenate([e[1] for e in exp])
    _check(ring, 0, conns, exp, twin.rate_limit_batch(want))
    assert [int(ring.outcome[0][c]["n_frames"]) for c in range(4)] == [3, 3, 3, 2]


# ---- 5. the driver -------------------------------------------------------------------------------------------------
def _driver_mix(rng, rnd):
    conns = mix(rng, 30)
    if rnd == 0:
        conns += [("resp", _throttle("q:1", 3, 10, 60) + _cmd("QUIT") + _throttle("q:1", 3, 10, 60)),
                  ("resp", _throttle("g:1", 3, 10, 60) + b"?garbage\r\n" + _throttle("g:1", 3, 10, 60)),
                  ("http", request(body_of("c:1")) + b"GET /health HTTP/1.1\r\nConnection: close\r\n\r\n"
                   + request(body_of("c:1"))),
                  ("grpc", gt.Connection())]
        conns[-1][1].buf += gt.PREFACE + gt.frame(gt.SETTINGS, 0, 0) + gs.call(1, gs.first_block(),
                                                                              b"\x0a\x01k\x10\x05\x18\x0a\x20\x3c")
    return conns


@pytest.mark.parametrize("seed", [(0, 0), SIP], ids=["unkeyed", "siphash"])
def test_driver_equals_the_host_walks(seed):
    """mixed.process_connections through the ring equals its ring=None rounds on a twin engine, including the general
    paths (PING, QUIT, RESP integers, garbage, /health, 404, escapes, SETTINGS, an HPACK insert, a preface)"""
    rng = random.Random(21)
    lim, twin, ring = _pair(seed, row_capacity=1 << 14, max_conns=64)
    for rnd in range(5):
        conns = _driver_mix(rng, rnd)
        ref = copy_conns(conns)
        now = NOW + rnd * NS
        got = mixed.process_connections(conns, lim, now, ring, slot=rnd % 2)
        want = mixed.process_connections(ref, twin, now, None)
        assert got == want, rnd
        for (p, a), (_, b) in zip(conns, ref):
            if p == "grpc":
                assert (bytes(a.out), bytes(a.buf), a.last_stream, a.send_window, a.closed) == \
                    (bytes(b.out), bytes(b.buf), b.last_stream, b.send_window, b.closed)
    a, b = lim.store.stats(), twin.store.stats()
    assert (a["len"], a["allowed"], a["denied"], a["errors"]) == (b["len"], b["allowed"], b["denied"], b["errors"])


def test_reference_multi_transport_limit_through_the_ring():
    """multi_transport.rs:159-225 through the ring: 200 requests for one key alternating RESP, HTTP and gRPC, one
    limit: exactly 100 limited, the same flags as the host walks give"""
    for n_conns, health_at in ((3, None), (200, None), (6, 4)):
        lim, twin, ring = _pair((9, 10), row_capacity=4096, max_conns=256)
        conns, per = shared_key_conns(n_conns, 200, health_at)
        ref = copy_conns(conns)
        got = mixed.process_connections(conns, lim, NOW, ring)
        want = mixed.process_connections(ref, twin, NOW, None)
        assert got == want
        flags = allowed_flags(conns, got)
        assert flags == allowed_flags(ref, want)
        assert sum(not a for f in flags for a in f) == 100


# ---- 6. denied keys ---------------------------------------------------------------------------------------------------
def test_denied_counts_add_up_over_the_three_transports():
    lim, _, ring = _pair(SIP, row_capacity=4096, max_conns=256)
    lim.store.track_denied(1 << 10)
    conns, per = shared_key_conns(9, 300)
    got = mixed.process_connections(conns, lim, NOW, ring)
    flags = allowed_flags(conns, got)
    by_proto = {}
    for (p, _), f in zip(conns, flags):
        by_proto[p] = by_proto.get(p, 0) + sum(not a for a in f)
    assert all(by_proto[p] > 0 for p in P) and sum(by_proto.values()) == 200
    lim.store.sync()
    top, dropped = lim.store.top_denied(8)
    assert dropped == 0 and top == [(lim.store.hash_key(b"shared_test_key"), 200)]
