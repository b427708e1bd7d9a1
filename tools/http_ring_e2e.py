"""Requests/s of POST /throttle end to end: (a) gcra_http_parse_throttle on one host core into a plain ring slot,
then the responses formatted on the host (gcra_http_format_replies), against (b) the HTTP ring (parse and responses
on the GPU).  Requests are in curl's header layout over Zipf(1.1) keys.  Shapes: one connection with a 64 KiB
pipeline; 16 to 65,536 connections with one request each (HTTP's usual keep-alive shape); 4,096 connections with 8
pipelined requests each.  Each variant has a fresh engine, the variants alternate in one run and must give the same
response bytes; medians are reported.  The parse and reply kernels are timed with torch.profiler in a run of their
own.  Prints one JSON line per shape, plus the card and its power limit.

    python tools/http_ring_e2e.py [--reps 7] [--shapes 1x0,16x1,256x1,4096x1,16384x1,65536x1,4096x8] [--out FILE]

(a shape CxR is C connections with R requests each; R = 0 fills each connection to 64 KiB)
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import throttlecrab_b200 as tc  # noqa: E402
from resp_ring_e2e import card  # noqa: E402

NOW = 1_700_000_000 * 10**9
ROW_CAP = 1 << 16


def one_request(key):
    body = b'{"key":"%s","max_burst":10,"count_per_period":100,"period":60}' % key
    return (b"POST /throttle HTTP/1.1\r\nHost: localhost:8080\r\nUser-Agent: curl/8.5.0\r\nAccept: */*\r\n"
            b"Content-Type: application/json\r\nContent-Length: %d\r\n\r\n" % len(body)) + body


def buffers(n_conns, per_conn, rng):
    out = []
    for _ in range(n_conns):
        n = per_conn or 65536 // 150
        b = bytearray()
        for i in np.minimum(rng.zipf(1.1, n), 1_000_000):
            r = one_request(b"user:%d" % int(i))
            if len(b) + len(r) > 65536:
                break
            b += r
        out.append(bytes(b))
    return out


class HostPath:
    """(a): the host walk on this thread into a plain ring slot, responses formatted on this thread"""

    def __init__(self):
        self.lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 21, created_ns=NOW, max_batch=ROW_CAP))
        self.ring = tc.Ring(self.lim, 1, ROW_CAP)
        self.out = C.create_string_buffer(ROW_CAP * tc.HTTP_REPLY_MAX)

    def run(self, bufs):
        L, h, ring = self.lim._L, self.lim._h, self.ring
        req = ring.req[0]
        n, spans = 0, []
        used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
        for b in bufs:
            L.gcra_http_parse_throttle(h, b, len(b), NOW, ROW_CAP - n, req.ctypes.data + n * 48, C.byref(used),
                                       C.byref(cnt), C.byref(stop))
            spans.append((n, cnt.value))
            n += cnt.value
        ring.submit(0, n, NOW)
        ring.wait(0)
        res = ring.res[0]
        replies = []
        for first, k in spans:
            w = L.gcra_http_format_replies(req.ctypes.data + first * 48, res.ctypes.data + first * 32, k, self.out,
                                           len(self.out))
            replies.append(C.string_at(self.out, w))
        return n, replies


class GpuPath:
    """(b): the HTTP ring"""

    def __init__(self, n_conns, in_bytes):
        self.lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 21, created_ns=NOW, max_batch=ROW_CAP))
        self.ring = tc.HttpRing(self.lim, 1, max(n_conns, 1), max(in_bytes, 1), ROW_CAP)

    def run(self, bufs):
        ring = self.ring
        at = 0
        for c, b in enumerate(bufs):
            ring.input[0][at:at + len(b)] = np.frombuffer(b, np.uint8)
            ring.conns[0][c] = (at, len(b))
            at += len(b)
        ring.submit(0, len(bufs), NOW)
        ring.wait(0)
        o = ring.outcome[0][:len(bufs)]
        rep = ring.replies[0]
        return int(o["n_frames"].sum()), [rep[int(x["reply_off"]):int(x["reply_off"]) + int(x["reply_len"])].tobytes()
                                          for x in o]


KERNELS = tuple("%s<gcra::HttpTraits>" % k for k in ("ring_parse_kernel", "ring_reply_kernel", "ring_outcome_kernel"))


def kernel_ms(gpu, bufs, iters=5):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            gpu.run(bufs)
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
    ap.add_argument("--shapes", default="1x0,16x1,256x1,4096x1,16384x1,65536x1,4096x8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    rng = np.random.default_rng(1)
    lines = []
    for shape in a.shapes.split(","):
        n_conns, per = (int(x) for x in shape.split("x"))
        bufs = buffers(n_conns, per, rng)
        host, gpu = HostPath(), GpuPath(n_conns, sum(len(b) for b in bufs))     # fresh engines: the same history
        t = {"a": [], "b": []}
        frames = 0
        for rep in range(a.reps + 1):                     # rep 0 warms up
            ra = rb = None
            for v in ("a", "b") if rep % 2 == 0 else ("b", "a"):
                t0 = time.perf_counter()
                if v == "a":
                    frames, ra = host.run(bufs)
                else:
                    fb, rb = gpu.run(bufs)
                dt = time.perf_counter() - t0
                if rep:
                    t[v].append(dt)
            if ra != rb or fb != frames:
                raise SystemExit("response bytes of the HTTP ring differ from the host path (%s)" % shape)
        in_bytes = sum(len(b) for b in bufs)
        out_bytes = sum(len(x) for x in rb)
        k = kernel_ms(gpu, bufs)
        line = {"shape": shape, "conns": n_conns, "requests": frames, "in_bytes": in_bytes, "reply_bytes": out_bytes,
                "a_host_parse_ring_mrps": round(frames / np.median(t["a"]) / 1e6, 3),
                "b_http_ring_mrps": round(frames / np.median(t["b"]) / 1e6, 3),
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
