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
from .metrics import Metrics, ShardedMetrics

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
    _check_conns(conns, RESP_MAX_CONN_BYTES if ring is None else min(RESP_MAX_CONN_BYTES, ring.in_capacity))

    def gpu(rounds, ready):
        if ring is None:
            for c in ready:
                if rounds.grpc[c]:
                    o, reply, _, _, _ = _gt.host_walk(conns[c][1], limiter, now)
                    rounds.took(c, reply, int(o["consumed"]), int(o["n_frames"]), o)
                    rounds.stops[c] = int(o["stop"])
                else:
                    reply, consumed, k, rounds.stops[c] = host_walk(conns[c][0], rounds.rest(c), limiter, now)
                    rounds.took(c, reply, consumed, k)
            return
        i = 0
        while i < len(ready):                              # as many submits as the ring's capacity needs
            group, i = rounds.fill(ring, slot, ready, i)
            ring.submit(slot, len(group), now)
            ring.wait(slot)
            rounds.take(ring, slot, group)

    return _Rounds(conns).run(limiter, now, metrics, gpu)


def process_connections_sharded(ranks, now_ns, slot=0, metrics=None):
    """Serve the connections of several engines of ONE process against their one hash-sharded table.  `ranks` is a
    list of (conns, limiter, ring), one per engine, rank r = its place in the list: the engines connected with
    sharded.connect_local (on one GPU or several), each ring a MixedRing of its engine; the rings are switched to
    peer-memory ticks (RespRing.peer_memory).  Returns, per rank, what process_connections returns for its conns.

    The rounds are process_connections's over the ranks' lists joined in rank order.  In a round every rank submits
    ring ticks together: every rank's submit_route, then every rank's submit_finish, ranks with no ready connection
    included (a tick of 0 rows), one tick or more until every rank's ready connections are through.  A rank whose ready
    connections do not all fit its slot (max_conns, in_capacity) leaves the ranks after it empty in that tick, so the
    connections go through the ticks in the joined order.  So a tick's rows are decided in rank order, then table
    order, each on its key's owner.  Then the general paths run in rank order, then list order; a Throttle they decide
    goes to its key's owner engine (OwnerRouter).  When no slot's row capacity fills (stop 3), every connection gets
    the bytes process_connections(ring=None) gives on ONE engine over the joined list.

    `metrics` may be a metrics.ShardedMetrics over the ranks' limiters in rank order: it is GET /metrics for the HTTP
    connections, and records every request the general paths decide as process_connections does (each rank's GPU
    counts its ring's rows and names their denied keys).  Anything else is refused (ValueError)."""
    check_sharded_metrics(metrics, [lim for _, lim, _ in ranks])
    now = int(now_ns)
    conns, rank_of = [], []
    for r, (cs, _, ring) in enumerate(ranks):
        _check_conns(cs, min(RESP_MAX_CONN_BYTES, ring.in_capacity))
        conns += cs
        rank_of += [r] * len(cs)
    rings = [ring for _, _, ring in ranks]
    for ring in rings:
        ring.peer_memory(True)
    router = OwnerRouter([lim for _, lim, _ in ranks])

    def gpu(rounds, ready):
        mine = [[c for c in ready if rank_of[c] == r] for r in range(len(ranks))]
        at = [0] * len(ranks)
        while True:
            groups, behind = [], False
            for r, ring in enumerate(rings):
                group = []
                if not behind:                             # (an earlier rank still has connections for a later tick)
                    group, at[r] = rounds.fill(ring, slot, mine[r], at[r])
                    behind = at[r] < len(mine[r])
                groups.append(group)
            for ring, group in zip(rings, groups):         # every route of the tick before the first finish
                ring.submit_route(slot, len(group), now)
            for ring in rings:
                ring.submit_finish(slot)
            for ring, group in zip(rings, groups):
                ring.wait(slot)
                rounds.take(ring, slot, group)
            if all(a == len(m) for a, m in zip(at, mine)):
                break

    got = _Rounds(conns).run(router, now, metrics, gpu)
    out, a = [], 0
    for cs, _, _ in ranks:
        out.append(got[a:a + len(cs)])
        a += len(cs)
    return out


def check_sharded_metrics(metrics, limiters):
    """ValueError unless `metrics` is None or a metrics.ShardedMetrics over exactly `limiters`, in their order"""
    if metrics is not None and not (isinstance(metrics, ShardedMetrics) and len(metrics.limiters) == len(limiters) and
                                    all(m is lim for m, lim in zip(metrics.limiters, limiters))):
        raise ValueError("the sharded driver serves metrics only from a ShardedMetrics of its ranks' limiters")


class OwnerRouter:
    """The limiter that process_connections_sharded's general paths decide on: store.hash_key is the ranks' shared
    seed's hash, and rate_limit_batch decides each row on its key's owner, limiters[gcra_owner_of(key_hash, world)]
    (rows of one owner in their order; rows of different owners have different keys)."""

    def __init__(self, limiters):
        self.limiters = list(limiters)
        self.store = _Hasher(self.limiters[0].store.hash_key)

    def rate_limit_batch(self, requests):
        req = np.ascontiguousarray(requests, REQ_DTYPE)
        res = np.zeros(len(req), RES_DTYPE)
        L, world = _native.lib(), len(self.limiters)
        own = np.array([L.gcra_owner_of(int(k), world) for k in req["key_hash"]], np.int64)
        for r in np.unique(own):
            m = own == r
            res[m] = self.limiters[int(r)].rate_limit_batch(req[m])
        return res


class _Hasher:
    def __init__(self, hash_key):
        self.hash_key = hash_key


def _check_conns(conns, room):
    for p, cn in conns:
        if p not in PROTOCOLS:
            raise ValueError("protocol must be 'resp', 'http' or 'grpc', not %r" % (p,))
        size = len(cn.buf) if p == "grpc" else len(cn)
        if size > room:
            raise ValueError("a connection buffer of %d bytes: at most %d" % (size, room))


class _Rounds:
    """The state of process_connections's rounds over `conns`: what every connection took, where it stopped."""

    def __init__(self, conns):
        self.conns = conns
        n = len(conns)
        self.grpc = [p == "grpc" for p, _ in conns]
        self.datas = [None if self.grpc[c] else bytes(conns[c][1]) for c in range(n)]
        self.before = [conns[c][1].n_throttle if self.grpc[c] else 0 for c in range(n)]
        self.pos, self.n_thr, self.close = [0] * n, [0] * n, [None] * n
        self.out = [[] for _ in range(n)]
        self.stops = {}

    def rest(self, c):
        return bytes(self.conns[c][1].buf) if self.grpc[c] else self.datas[c][self.pos[c]:]

    def took(self, c, reply, consumed, n_frames, go=None):
        """apply a walk's outcome to connection c (go: a gRPC connection's outcome row)"""
        if self.grpc[c]:
            cn = self.conns[c][1]
            cn.out += reply
            cn.take_outcome(go)
            del cn.buf[:consumed]
            cn.n_throttle += n_frames
        else:
            self.out[c].append(reply)
            self.pos[c] += consumed
            self.n_thr[c] += n_frames

    def fill(self, ring, slot, ready, i):
        """ready[i:] into the ring's slot, as many as fit -> (the connections placed, the next i)"""
        group, used, k = [], 0, 0
        while i < len(ready) and len(group) < ring.max_conns:
            c = ready[i]
            b = self.rest(c)
            if used + len(b) > ring.in_capacity:
                break
            ring.input[slot][used:used + len(b)] = np.frombuffer(b, np.uint8)
            row = ring.conns[slot][len(group)]
            row["off"], row["len"], row["protocol"] = used, len(b), PROTOCOLS[self.conns[c][0]]
            row["grpc_state"] = k if self.grpc[c] else 0
            if self.grpc[c]:
                self.conns[c][1].state(ring.grpc_conns[slot][k])
                k += 1
            group.append(c)
            used += len(b)
            i += 1
        return group, i

    def take(self, ring, slot, group):
        """after the slot's wait: its outcomes and replies to the connections placed in it"""
        k = 0
        for j, c in enumerate(group):
            o = ring.outcome[slot][j]
            off, ln = int(o["reply_off"]), int(o["reply_len"])
            go = None
            if self.grpc[c]:
                go = ring.grpc_outcome[slot][k]
                k += 1
            self.took(c, ring.replies[slot][off:off + ln].tobytes(), int(o["consumed"]), int(o["n_frames"]), go)
            self.stops[c] = int(o["stop"])

    def run(self, limiter, now, metrics, gpu):
        """the rounds: gpu(self, ready) takes the ready connections' plain prefixes (and sets their stops), then the
        general paths decide on `limiter` -> per connection, what process_connections returns"""
        conns, grpc, datas, pos = self.conns, self.grpc, self.datas, self.pos
        n = len(conns)
        live = [c for c in range(n) if (conns[c][1].buf and not conns[c][1].closed if grpc[c] else datas[c])]
        while live:
            self.stops = {}
            gpu(self, [c for c in live if not grpc[c] or conns[c][1].plain_ready])
            nxt = []
            for c in live:
                st = self.stops.get(c, 2)                  # (a gRPC connection that was not ready: the general path)
                if st == 3:
                    nxt.append(c)
                    continue
                if st != 2:
                    continue                               # the end of its bytes, or an incomplete request
                p, cn = conns[c]
                if p == "grpc":
                    had = len(cn.buf)
                    cn.general(limiter, now, metrics)
                    if not cn.closed and cn.buf and len(cn.buf) < had and cn.plain_ready:
                        nxt.append(c)
                    continue
                data = datas[c][pos[c]:]
                g = _resp.general(data, limiter, now, metrics) if p == "resp" else \
                    _http.general(data, limiter, now, metrics)
                if g is None:
                    continue
                used, reply, k, self.close[c] = g
                pos[c] += used
                self.out[c].append(reply)
                self.n_thr[c] += k
                if self.close[c] is None and pos[c] < len(datas[c]):
                    nxt.append(c)
            live = nxt
        return [conns[c][1].n_throttle - self.before[c] if grpc[c] else
                (b"".join(self.out[c]), pos[c], self.n_thr[c], self.close[c]) for c in range(n)]
