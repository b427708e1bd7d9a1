"""Requests/s of a server that serves RESP, HTTP and gRPC against one table: (a) every connection walked on one host
core by its protocol's host walk (gcra_resp_parse_throttle, gcra_http_parse_throttle, gcra_grpc_parse_throttle) into
one plain ring slot, replies formatted on the host, against (b) the mixed ring (parse and replies on the GPU, one
batch).  (c) is three single-protocol rings on three engines: three tables, so not a valid server, only a reference for
what mixing the protocols in one slot costs the kernels.  Connections are split evenly over the three protocols, keys
Zipf(1.1).  Shapes: 3 x C connections with R requests each; R = 0 fills one connection of each protocol to 64 KiB.
The variants alternate in one run, (a) and (b) must give the same reply bytes in every repetition, and medians are
reported.  The ring kernels are timed with torch.profiler in a run of their own.  Prints one JSON line per shape, plus
the card and its power limit.

    python tools/mixed_ring_e2e.py [--reps 7] [--shapes 1x0,16x1,16x8,256x1,256x8,4096x1,4096x8] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
import grpc_streams  # noqa: E402
from resp_ring_e2e import card  # noqa: E402

NOW = 1_700_000_000 * 10**9
ROW_CAP = 1 << 17
PROTOS = ("resp", "http", "grpc")
P = {"resp": tc.PROTO_RESP, "http": tc.PROTO_HTTP, "grpc": tc.PROTO_GRPC}


def resp_frame(key):
    a = [b"THROTTLE", key, b"10", b"100", b"60"]
    return b"*5\r\n" + b"".join(b"$%d\r\n%s\r\n" % (len(x), x) for x in a)


def http_request(key):
    body = b'{"key":"%s","max_burst":10,"count_per_period":100,"period":60}' % key
    return (b"POST /throttle HTTP/1.1\r\nHost: localhost:8080\r\nContent-Type: application/json\r\n"
            b"Content-Length: %d\r\n\r\n" % len(body)) + body


def connections(n_per, per_conn, rng):
    """(protocol, bytes, gRPC state row or None), the protocols interleaved in table order"""
    out = []
    for c in range(n_per):
        for p in PROTOS:
            n = per_conn or 65536
            keys = [b"user:%d" % int(i) for i in np.minimum(rng.zipf(1.1, n), 1_000_000)]
            b, row = bytearray(), None
            if p == "grpc":
                cn = grpc_streams.established()
                block, row = grpc_streams.steady_block(cn.hpack), cn.conn_row()
            for k, key in enumerate(keys):
                if p == "resp":
                    f = resp_frame(key)
                elif p == "http":
                    f = http_request(key)
                else:
                    f = grpc_streams.call(3 + 2 * k, block, grpc_streams.request_bytes(key, 10, 100, 60, 1),
                                          ping=k == 3)
                if len(b) + len(f) > 65536:
                    break
                b += f
            out.append((p, bytes(b), row))
    return out


def _engine():
    return tc.RateLimiter(tc.ManualStore(capacity=1 << 21, created_ns=NOW, max_batch=ROW_CAP))


class HostPath:
    """(a): each connection's host walk on this thread into one plain ring slot, replies formatted on this thread"""

    def __init__(self):
        self.lim = _engine()
        self.ring = tc.Ring(self.lim, 1, ROW_CAP)
        self.out = C.create_string_buffer(ROW_CAP * tc.HTTP_REPLY_MAX)
        self.sids = np.zeros(ROW_CAP, np.uint32)
        self.o = np.zeros((), tc.GRPC_OUTCOME_DTYPE)

    def run(self, conns):
        L, h, ring = self.lim._L, self.lim._h, self.ring
        req = ring.req[0]
        n, spans = 0, []
        used, cnt, stop, sent = C.c_uint64(), C.c_uint32(), C.c_int32(), C.c_uint32()
        for p, b, row in conns:
            if p == "grpc":
                L.gcra_grpc_parse_throttle(h, b, len(b), NOW, ROW_CAP - n, row.ctypes.data, req.ctypes.data + n * 48,
                                           self.sids.ctypes.data + n * 4, self.o.ctypes.data)
                k = int(self.o["n_frames"])
            else:
                walk = L.gcra_resp_parse_throttle if p == "resp" else L.gcra_http_parse_throttle
                walk(h, b, len(b), NOW, ROW_CAP - n, req.ctypes.data + n * 48, C.byref(used), C.byref(cnt),
                     C.byref(stop))
                k = cnt.value
            spans.append((p, n, k))
            n += k
        ring.submit(0, n, NOW)
        ring.wait(0)
        res = ring.res[0]
        replies = []
        for p, first, k in spans:
            q, r = req.ctypes.data + first * 48, res.ctypes.data + first * 32
            if p == "grpc":
                w = L.gcra_grpc_format_replies(q, r, self.sids.ctypes.data + first * 4, k, self.out, len(self.out),
                                               C.byref(sent))
            elif p == "resp":
                w = L.gcra_resp_format_replies(q, r, k, self.out, len(self.out))
            else:
                w = L.gcra_http_format_replies(q, r, k, self.out, len(self.out))
            replies.append(C.string_at(self.out, w))
        return n, replies


def _fill(ring, conns, mixed):
    at, g = 0, 0
    for c, (p, b, row) in enumerate(conns):
        ring.input[0][at:at + len(b)] = np.frombuffer(b, np.uint8)
        if mixed:
            ring.conns[0][c] = (at, len(b), P[p], g if p == "grpc" else 0)
            if p == "grpc":
                ring.grpc_conns[0][g] = row
                g += 1
        else:
            if p == "grpc":
                ring.conns[0][c] = row
            ring.conns[0][c]["off"], ring.conns[0][c]["len"] = at, len(b)
        at += len(b)


def _replies(ring, n):
    o = ring.outcome[0][:n]
    rep = ring.replies[0]
    return [rep[int(x["reply_off"]):int(x["reply_off"]) + int(x["reply_len"])].tobytes() for x in o]


class MixedPath:
    """(b): the mixed ring"""

    def __init__(self, conns):
        self.lim = _engine()
        self.ring = tc.MixedRing(self.lim, 1, len(conns), sum(len(b) for _, b, _ in conns), ROW_CAP)

    def run(self, conns):
        _fill(self.ring, conns, True)
        self.ring.submit(0, len(conns), NOW)
        self.ring.wait(0)
        return int(self.ring.outcome[0][:len(conns)]["n_frames"].sum()), _replies(self.ring, len(conns))


class SplitPath:
    """(c): one single-protocol ring per protocol, each on its own engine (three tables: a kernel-time reference)"""

    def __init__(self, conns):
        self.parts = {}
        for p in PROTOS:
            mine = [x for x in conns if x[0] == p]
            lim = _engine()
            self.parts[p] = (lim, tc.RespRing(lim, 1, len(mine), sum(len(b) for _, b, _ in mine), ROW_CAP,
                                              protocol=p), mine)

    def run(self, conns):
        for p, (_, ring, mine) in self.parts.items():
            _fill(ring, mine, False)
            ring.submit(0, len(mine), NOW)
        n = 0
        for p, (_, ring, mine) in self.parts.items():
            ring.wait(0)
            n += int(ring.outcome[0][:len(mine)]["n_frames"].sum())
        return n, None


def kernel_ms(path, conns, names, iters=5):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            path.run(conns)
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for name in names:
            if name in e.name:
                tot[name] = tot.get(name, 0.0) + e.device_time / 1000.0
    return {k: round(v / iters, 4) for k, v in tot.items()}


# (with the template argument: variant (c)'s single-protocol rings must not count the mixed instantiation's time)
RING_KERNELS = tuple("%s<gcra::%s>" % (k, t) for t in ("MixedTraits", "RespTraits", "HttpTraits", "GrpcTraits")
                     for k in ("ring_parse_kernel", "ring_reply_kernel", "ring_outcome_kernel"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--shapes", default="1x0,16x1,16x8,256x1,256x8,4096x1,4096x8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    rng = np.random.default_rng(1)
    lines = []
    for shape in a.shapes.split(","):
        n_per, per = (int(x) for x in shape.split("x"))
        conns = connections(n_per, per, rng)
        paths = {"a": HostPath(), "b": MixedPath(conns), "c": SplitPath(conns)}
        t = {v: [] for v in paths}
        reqs = 0
        for rep in range(a.reps + 1):                     # rep 0 warms up
            got = {}
            order = ("a", "b", "c") if rep % 2 == 0 else ("c", "b", "a")
            for v in order:
                t0 = time.perf_counter()
                got[v] = paths[v].run(conns)
                dt = time.perf_counter() - t0
                if rep:
                    t[v].append(dt)
            reqs = got["a"][0]
            if got["a"] != got["b"] or got["c"][0] != reqs:
                raise SystemExit("reply bytes of the mixed ring differ from the host path (%s)" % shape)
        kb = kernel_ms(paths["b"], conns, RING_KERNELS)
        kc = kernel_ms(paths["c"], conns, RING_KERNELS)
        line = {"shape": "3x" + shape, "conns": len(conns), "requests": reqs,
                "in_bytes": sum(len(b) for _, b, _ in conns), "reply_bytes": sum(len(x) for x in got["b"][1]),
                "a_host_walk_ring_mrps": round(reqs / np.median(t["a"]) / 1e6, 3),
                "b_mixed_ring_mrps": round(reqs / np.median(t["b"]) / 1e6, 3),
                "c_three_rings_mrps": round(reqs / np.median(t["c"]) / 1e6, 3),
                "a_ms": round(1e3 * np.median(t["a"]), 3), "b_ms": round(1e3 * np.median(t["b"]), 3),
                "c_ms": round(1e3 * np.median(t["c"]), 3),
                "b_kernel_ms": kb, "c_kernel_ms": kc,
                "b_ring_kernels_ms": round(sum(kb.values()), 4), "c_ring_kernels_ms": round(sum(kc.values()), 4),
                "replies_equal": True}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del paths
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps({"card": card()}) + "\n")
            for x in lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
