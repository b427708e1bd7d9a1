"""Throttle calls/s of the gRPC transport end to end: (a) gcra_grpc_parse_throttle on one host core into a plain ring
slot, then the responses formatted on the host (gcra_grpc_format_replies), against (b) the gRPC ring (parse and
responses on the GPU).  Connections are in the steady state grpcio reaches after its first call (an indexed-only
header block, a stream WINDOW_UPDATE, DATA(END_STREAM), a connection WINDOW_UPDATE per call, one BDP PING) over
Zipf(1.1) keys.  Shapes: one 64 KiB connection; 16 to 16,384 connections with one call each; 4,096 connections with
8 calls each.  Each variant has a fresh engine, the variants alternate in one run and must give the same response
bytes; medians are reported.  The gRPC kernels are timed with torch.profiler in a run of their own.  Prints one JSON
line per shape, plus the card and its power limit.

    python tools/grpc_ring_e2e.py [--reps 7] [--shapes 1x0,16x1,256x1,4096x1,16384x1,4096x8] [--out FILE]

(a shape CxR is C connections with R calls each; R = 0 fills each connection to 64 KiB)
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
from throttlecrab_b200 import grpc_transport as gt  # noqa: E402
import grpc_streams  # noqa: E402
from resp_ring_e2e import card  # noqa: E402

NOW = 1_700_000_000 * 10**9
ROW_CAP = 1 << 16


def connections(n_conns, per_conn, rng):
    """(state row, bytes) per connection"""
    out = []
    for _ in range(n_conns):
        cn = grpc_streams.established()
        block = grpc_streams.steady_block(cn.hpack)
        b, sid = bytearray(), 3
        n = per_conn or 65536
        for k, i in enumerate(np.minimum(rng.zipf(1.1, n), 1_000_000)):
            msg = grpc_streams.request_bytes(b"user:%d" % int(i), 10, 100, 60, 1)
            c = grpc_streams.call(sid, block, msg, ping=k == 3)
            if len(b) + len(c) > 65536:
                break
            b += c
            sid += 2
        out.append((cn.conn_row(), bytes(b)))
    return out


class HostPath:
    """(a): the host walk on this thread into a plain ring slot, responses formatted on this thread"""

    def __init__(self):
        self.lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 21, created_ns=NOW, max_batch=ROW_CAP))
        self.ring = tc.Ring(self.lim, 1, ROW_CAP)
        self.out = C.create_string_buffer(ROW_CAP * tc.GRPC_REPLY_MAX)
        self.sids = np.zeros(ROW_CAP, np.uint32)
        self.o = np.zeros((), tc.GRPC_OUTCOME_DTYPE)

    def run(self, conns):
        L, h, ring = self.lim._L, self.lim._h, self.ring
        req = ring.req[0]
        n, spans = 0, []
        sent = C.c_uint32()
        for row, b in conns:
            L.gcra_grpc_parse_throttle(h, b, len(b), NOW, ROW_CAP - n, row.ctypes.data, req.ctypes.data + n * 48,
                                       self.sids.ctypes.data + n * 4, self.o.ctypes.data)
            k = int(self.o["n_frames"])
            spans.append((n, k))
            n += k
        ring.submit(0, n, NOW)
        ring.wait(0)
        res = ring.res[0]
        replies = []
        for first, k in spans:
            w = L.gcra_grpc_format_replies(req.ctypes.data + first * 48, res.ctypes.data + first * 32,
                                           self.sids.ctypes.data + first * 4, k, self.out, len(self.out),
                                           C.byref(sent))
            replies.append(C.string_at(self.out, w))
        return n, replies


class GpuPath:
    """(b): the gRPC ring"""

    def __init__(self, n_conns, in_bytes):
        self.lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 21, created_ns=NOW, max_batch=ROW_CAP))
        self.ring = tc.GrpcRing(self.lim, 1, max(n_conns, 1), max(in_bytes, 1), ROW_CAP)

    def run(self, conns):
        ring = self.ring
        at = 0
        for c, (row, b) in enumerate(conns):
            ring.input[0][at:at + len(b)] = np.frombuffer(b, np.uint8)
            ring.conns[0][c] = row
            ring.conns[0][c]["off"], ring.conns[0][c]["len"] = at, len(b)
            at += len(b)
        ring.submit(0, len(conns), NOW)
        ring.wait(0)
        o = ring.outcome[0][:len(conns)]
        rep = ring.replies[0]
        return int(o["n_frames"].sum()), [rep[int(x["reply_off"]):int(x["reply_off"]) + int(x["reply_len"])].tobytes()
                                          for x in o]


KERNELS = tuple("%s<gcra::GrpcTraits>" % k for k in ("ring_parse_kernel", "ring_reply_kernel", "ring_outcome_kernel"))


def kernel_ms(gpu, conns, iters=5):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            gpu.run(conns)
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        for name in KERNELS:
            if name in e.name and e.device_type.name == "CUDA":
                tot[name] = tot.get(name, 0.0) + e.device_time / 1000.0
    return {k: v / iters for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--shapes", default="1x0,16x1,256x1,4096x1,16384x1,4096x8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    rng = np.random.default_rng(1)
    lines = []
    for shape in a.shapes.split(","):
        n_conns, per = (int(x) for x in shape.split("x"))
        conns = connections(n_conns, per, rng)
        host, gpu = HostPath(), GpuPath(n_conns, sum(len(b) for _, b in conns))
        t = {"a": [], "b": []}
        calls = 0
        for rep in range(a.reps + 1):                     # rep 0 warms up
            ra = rb = None
            for v in ("a", "b") if rep % 2 == 0 else ("b", "a"):
                t0 = time.perf_counter()
                if v == "a":
                    calls, ra = host.run(conns)
                else:
                    fb, rb = gpu.run(conns)
                dt = time.perf_counter() - t0
                if rep:
                    t[v].append(dt)
            if ra != rb or fb != calls:
                raise SystemExit("response bytes of the gRPC ring differ from the host path (%s)" % shape)
        k = kernel_ms(gpu, conns)
        line = {"shape": shape, "conns": n_conns, "calls": calls, "in_bytes": sum(len(b) for _, b in conns),
                "reply_bytes": sum(len(x) for x in rb),
                "a_host_parse_ring_mcps": round(calls / np.median(t["a"]) / 1e6, 3),
                "b_grpc_ring_mcps": round(calls / np.median(t["b"]) / 1e6, 3),
                "a_ms": round(1e3 * np.median(t["a"]), 3), "b_ms": round(1e3 * np.median(t["b"]), 3),
                "kernel_ms": {x: round(y, 4) for x, y in k.items()}, "replies_equal": True}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del host, gpu
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps({"card": card()}) + "\n")
            for x in lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
