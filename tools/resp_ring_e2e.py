"""Frames/s of RESP THROTTLE pipelines end to end: (a) the keyed parse on one host core into a keyed ring, then the
replies formatted on the host, against (b) the RESP ring (parse and replies on the GPU).  Each connection holds up to
64 KiB of THROTTLE frames over the bench's Zipf keys; 1, 16, 256 and 4096 connections; the variants alternate in one
run and must give the same reply bytes.  The parse and reply kernels are timed with torch.profiler in a run of their
own.  Prints one JSON line per case, plus the card and its power limit.

    python tools/resp_ring_e2e.py [--reps 7] [--conns 1,16,256,4096] [--out FILE.jsonl]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import throttlecrab_b200 as tc  # noqa: E402

NOW = 1_700_000_000 * 10**9
ROW_CAP = 1 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def buffers(n_conns, rng):
    """per connection: frames up to 64 KiB, at most ~ROW_CAP frames in all; Zipf(1.1) keys over 1 M ids"""
    per = min(65536, (ROW_CAP * 40) // n_conns)
    out = []
    for _ in range(n_conns):
        ids = np.minimum(rng.zipf(1.1, per // 40 + 1), 1_000_000)
        b, fr = bytearray(), None
        for i in ids:
            k = b"user:%d" % int(i)
            fr = b"*5\r\n$8\r\nTHROTTLE\r\n$%d\r\n%s\r\n$2\r\n10\r\n$3\r\n100\r\n$2\r\n60\r\n" % (len(k), k)
            if len(b) + len(fr) > per:
                break
            b += fr
        out.append(bytes(b))
    return out


class HostPath:
    """(a): keyed parse on this thread, keyed ring, replies formatted on this thread"""

    def __init__(self):
        self.lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 21, created_ns=NOW, max_batch=ROW_CAP))
        self.ring = tc.Ring(self.lim, 1, ROW_CAP, key_capacity=64 << 20)
        self.out = C.create_string_buffer(ROW_CAP * tc.RESP_REPLY_MAX)

    def run(self, bufs):
        L, h, ring = self.lim._L, self.lim._h, self.ring
        req, arena = ring.req[0], ring.keys[0]
        kused, n, spans = C.c_uint64(0), 0, []
        used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
        for b in bufs:
            L.gcra_resp_parse_throttle_keyed(h, b, len(b), NOW, ROW_CAP - n, req.ctypes.data + n * 48, arena.ctypes.data,
                                             len(arena), C.byref(kused), C.byref(used), C.byref(cnt), C.byref(stop))
            spans.append((n, cnt.value))
            n += cnt.value
        ring.submit(0, n, NOW, keys_len=kused.value)
        ring.wait(0)
        res = ring.res[0]
        replies = []
        for first, k in spans:
            w = L.gcra_resp_format_replies(req.ctypes.data + first * 48, res.ctypes.data + first * 32, k, self.out,
                                           len(self.out))
            replies.append(C.string_at(self.out, w))
        return n, replies


class GpuPath:
    """(b): the RESP ring"""

    def __init__(self, n_conns, in_bytes):
        self.lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 21, created_ns=NOW, max_batch=ROW_CAP))
        self.ring = tc.RespRing(self.lim, 1, max(n_conns, 1), max(in_bytes, 1), ROW_CAP)

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


KERNELS = tuple("%s<gcra::RespTraits>" % k for k in ("ring_parse_kernel", "ring_reply_kernel", "ring_outcome_kernel"))


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
    ap.add_argument("--conns", default="1,16,256,4096")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    rng = np.random.default_rng(1)
    lines = []
    for n_conns in [int(x) for x in a.conns.split(",")]:
        bufs = buffers(n_conns, rng)
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
                raise SystemExit("reply bytes of the RESP ring differ from the host path (%d connections)" % n_conns)
        in_bytes = sum(len(b) for b in bufs)
        out_bytes = sum(len(x) for x in rb)
        k = kernel_ms(gpu, bufs)
        line = {"conns": n_conns, "frames": frames, "in_bytes": in_bytes, "reply_bytes": out_bytes,
                "d2h_bytes_per_frame": round((out_bytes + 32 * n_conns) / max(frames, 1), 2),
                "a_host_parse_keyed_ring_mfps": round(frames / np.median(t["a"]) / 1e6, 2),
                "b_resp_ring_mfps": round(frames / np.median(t["b"]) / 1e6, 2),
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
