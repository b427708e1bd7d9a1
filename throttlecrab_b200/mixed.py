"""RESP, HTTP and gRPC connections served together, against one engine's table.

The reference server is one process that serves its Redis, HTTP and gRPC transports at once against one store, so a
key's limit is shared by all three.  process_connections serves connections of all three protocols in rounds, with
their plain requests parsed, decided as one batch and answered on the GPU through a MixedRing; what the GPU cannot
take goes to each protocol's own general path (resp.general, http.general, grpc_transport.Connection.general).
"""
import ctypes as C

import numpy as np

from . import REQ_DTYPE, RES_DTYPE, RESP_MAX_CONN_BYTES, RESP_REPLY_MAX, HTTP_REPLY_MAX, PROTO_RESP, PROTO_HTTP, \
    PROTO_GRPC, _native
from . import grpc_transport as _gt
from . import http as _http
from . import resp as _resp
from .metrics import Metrics

PROTOCOLS = {"resp": PROTO_RESP, "http": PROTO_HTTP, "grpc": PROTO_GRPC}
# the smallest plain frame of RESP and HTTP (gcra_resp.cuh, gcra_http.cuh MIN_FRAME_BYTES): room for a walk's rows
_MIN_FRAME = {"resp": 45, "http": 133}


def host_walk(protocol, data, limiter, now):
    """A RESP or HTTP connection's plain prefix by its host walk (gcra_resp_parse_throttle, gcra_http_parse_throttle),
    decided by limiter.rate_limit_batch, with keys hashed as limiter.store.hash_key hashes them -> (reply bytes,
    bytes consumed, rows, stop)"""
    L = _native.lib()
    resp = protocol == "resp"
    parse = L.gcra_resp_parse_throttle if resp else L.gcra_http_parse_throttle
    fmt = L.gcra_resp_format_replies if resp else L.gcra_http_format_replies
    req = np.zeros(len(data) // _MIN_FRAME[protocol] + 1, REQ_DTYPE)
    used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
    h = getattr(limiter.store, "_h", None)
    rc = parse(h, data, len(data), now, len(req), req.ctypes.data, C.byref(used), C.byref(cnt), C.byref(stop))
    assert rc == 0
    n = cnt.value
    if not n:
        return b"", used.value, 0, stop.value
    res = np.ascontiguousarray(limiter.rate_limit_batch(req[:n]), RES_DTYPE)
    out = C.create_string_buffer(n * (RESP_REPLY_MAX if resp else HTTP_REPLY_MAX))
    w = fmt(req.ctypes.data, res.ctypes.data, n, out, len(out))
    return out.raw[:w], used.value, n, stop.value


def process_connections(conns, limiter, now_ns, ring, slot=0, metrics=None):
    """Serve connections of all three protocols against `limiter`'s one table.  `conns` is a list of (protocol, conn):
    for "resp" and "http", conn is the connection's received bytes (at most 65,536); for "grpc", a
    grpc_transport.Connection whose `buf` holds at most 65,536 bytes.  `ring` is a MixedRing of `limiter`'s engine, or
    None: the same rounds with each connection's host walk decided by limiter.rate_limit_batch, one connection at a time
    in list order.  Returns per connection what its protocol's own driver returns: (reply_bytes, bytes_consumed,
    n_throttle, close) for RESP (resp.process_connections) and HTTP (http.process_connections, `metrics` serving GET
    /metrics), and the Throttle decisions made for gRPC (grpc_transport.process_connections, which updates the
    Connection).

    The decision order: rounds run until every connection has ended at the end of its bytes, at an incomplete frame,
    or closed.  In a round, the GPU takes every ready connection's plain prefix, whatever its protocol: one batch per
    submit, rows in list order of the connections and request order within each (a full slot leaves the rest to the
    next round, or to the next submit of the same round when the connections do not fit one).  A gRPC connection is
    ready when its preface is done and no stream is open.  Then, in list order, each connection that stopped at a
    request that is not plain takes its own protocol's general path: a RESP or HTTP connection for that one request,
    a gRPC connection (also one that was not ready) until no stream is open.  A Throttle request there is decided there
    and then, on its own.  Connections that share keys see each other's requests in that order, whatever their
    transports.

    A metrics.Metrics as `metrics` is GET /metrics for the HTTP connections, and records every request the general
    paths decide as the reference's transports do (the GPU counts the ring's rows).  It needs a ring: the host walks
    have no key positions to name denied keys from (ValueError)."""
    if ring is None and isinstance(metrics, Metrics):
        raise ValueError("metrics need a ring: the host walks do not name denied keys")
    now = int(now_ns)
    room = RESP_MAX_CONN_BYTES if ring is None else min(RESP_MAX_CONN_BYTES, ring.in_capacity)
    for p, cn in conns:
        if p not in PROTOCOLS:
            raise ValueError("protocol must be 'resp', 'http' or 'grpc', not %r" % (p,))
        size = len(cn.buf) if p == "grpc" else len(cn)
        if size > room:
            raise ValueError("a connection buffer of %d bytes: at most %d" % (size, room))
    n = len(conns)
    grpc = [p == "grpc" for p, _ in conns]
    datas = [None if grpc[c] else bytes(conns[c][1]) for c in range(n)]
    before = [conns[c][1].n_throttle if grpc[c] else 0 for c in range(n)]
    pos, n_thr, close = [0] * n, [0] * n, [None] * n
    out = [[] for _ in range(n)]

    def rest(c):
        return bytes(conns[c][1].buf) if grpc[c] else datas[c][pos[c]:]

    def took(c, reply, consumed, n_frames, go=None):
        """apply a walk's outcome to connection c (go: a gRPC connection's outcome row)"""
        if grpc[c]:
            cn = conns[c][1]
            cn.out += reply
            cn.take_outcome(go)
            del cn.buf[:consumed]
            cn.n_throttle += n_frames
        else:
            out[c].append(reply)
            pos[c] += consumed
            n_thr[c] += n_frames

    live = [c for c in range(n) if (conns[c][1].buf and not conns[c][1].closed if grpc[c] else datas[c])]
    while live:
        stops = {}
        ready = [c for c in live if not grpc[c] or conns[c][1].plain_ready]
        if ring is None:
            for c in ready:
                if grpc[c]:
                    o, reply, _, _, _ = _gt.host_walk(conns[c][1], limiter, now)
                    took(c, reply, int(o["consumed"]), int(o["n_frames"]), o)
                    stops[c] = int(o["stop"])
                else:
                    reply, consumed, k, stops[c] = host_walk(conns[c][0], rest(c), limiter, now)
                    took(c, reply, consumed, k)
            ready = []
        i = 0
        while i < len(ready):                              # as many submits as the ring's capacity needs
            group, used, k = [], 0, 0
            while i < len(ready) and len(group) < ring.max_conns:
                c = ready[i]
                b = rest(c)
                if used + len(b) > ring.in_capacity:
                    break
                ring.input[slot][used:used + len(b)] = np.frombuffer(b, np.uint8)
                row = ring.conns[slot][len(group)]
                row["off"], row["len"], row["protocol"] = used, len(b), PROTOCOLS[conns[c][0]]
                row["grpc_state"] = k if grpc[c] else 0
                if grpc[c]:
                    conns[c][1].state(ring.grpc_conns[slot][k])
                    k += 1
                group.append(c)
                used += len(b)
                i += 1
            ring.submit(slot, len(group), now)
            ring.wait(slot)
            k = 0
            for j, c in enumerate(group):
                o = ring.outcome[slot][j]
                off, ln = int(o["reply_off"]), int(o["reply_len"])
                go = None
                if grpc[c]:
                    go = ring.grpc_outcome[slot][k]
                    k += 1
                took(c, ring.replies[slot][off:off + ln].tobytes(), int(o["consumed"]), int(o["n_frames"]), go)
                stops[c] = int(o["stop"])
        nxt = []
        for c in live:
            st = stops.get(c, 2)                           # (a gRPC connection that was not ready: the general path)
            if st == 3:
                nxt.append(c)
                continue
            if st != 2:
                continue                                   # the end of its bytes, or an incomplete request
            p, cn = conns[c]
            if p == "grpc":
                had = len(cn.buf)
                cn.general(limiter, now, metrics)
                if not cn.closed and cn.buf and len(cn.buf) < had and cn.plain_ready:
                    nxt.append(c)
                continue
            data = datas[c][pos[c]:]
            g = _resp.general(data, limiter, now, metrics) if p == "resp" else _http.general(data, limiter, now, metrics)
            if g is None:
                continue
            used, reply, k, close[c] = g
            pos[c] += used
            out[c].append(reply)
            n_thr[c] += k
            if close[c] is None and pos[c] < len(datas[c]):
                nxt.append(c)
        live = nxt
    return [conns[c][1].n_throttle - before[c] if grpc[c] else (b"".join(out[c]), pos[c], n_thr[c], close[c])
            for c in range(n)]
