"""What the server's snapshot directory (--snapshot-dir, persist.SnapshotDir) costs, on tables of --keys entries
(traces.warm_pass): one JSON line per key count.

  save_s          the shutdown save (SnapshotDir.save: every engine's file, the manifest), from 1 and from 2 engines
  restore_s       the start-up restore (SnapshotDir.restore) 1 -> 1, 1 -> 2 and 2 -> 1 engines, all on cuda:0
  serve           ms per serve round on the 1-engine table: 3 x --conns connections (RESP, HTTP, gRPC), --depth
                  THROTTLE requests each, decided by mixed.process_connections on a MixedRing (the rounds the server's
                  serve runs, here driven from Python, so the host's share is larger than in the native server).  Rounds
                  alternate: without a save, and with a background save begun at the round's start (as the server
                  begins one between serves); median and maximum of each
  capture_ms      snapshot_capture_kernel's device time from torch.profiler, in a separate pass
  gpu             name, power limit and max SM clock, read in the same run

    python tools/server_snapshot_e2e.py [--keys 1000000 --keys 10000000] [--conns 4096] [--depth 8] [--rounds 10]

The snapshot directories go to a temporary directory that is removed afterwards.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

import throttlecrab_b200 as tc  # noqa: E402
from throttlecrab_b200 import grpc_transport as gt  # noqa: E402
from throttlecrab_b200 import mixed  # noqa: E402
from throttlecrab_b200.persist import SnapshotDir  # noqa: E402
import traces  # noqa: E402
from server_e2e import GrpcCalls, http_req, resp_req  # noqa: E402

BATCH = 1 << 20


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else None


def store(capacity):
    return tc.PeriodicStore(capacity=capacity, created_ns=traces.T0, max_batch=BATCH)


def filled(keys):
    st = store(keys)
    lim = tc.RateLimiter(st)
    warm = traces.warm_pass(keys)
    req = np.empty(BATCH, tc.REQ_DTYPE)
    for a in range(0, keys, BATCH):
        w = warm[a:a + BATCH]
        r = req[:len(w)]
        r["key_hash"] = tc.hash_key_ids(w["key"])
        for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
            r[f] = w[f]
        lim.rate_limit_batch(r)
    st.sync()
    return st, lim


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def restore_into(path, stores):
    sd = SnapshotDir(path, "periodic")
    try:
        s, _ = timed(lambda: sd.restore(stores))
        assert sd.generation >= 1
        return s
    finally:
        sd.close()


def save_from(path, stores):
    sd = SnapshotDir(path, "periodic")
    try:
        sd.restore(stores)
        s, _ = timed(sd.save)
        return s
    finally:
        sd.close()


def serve_rounds(lim, keys, conns, depth, rounds, path):
    rng = np.random.default_rng(1)
    ring = tc.MixedRing(lim, 1, 3 * conns, 16 << 20, 3 * conns * depth)
    grpc = [GrpcCalls("k:%d" % k) for k in rng.integers(0, keys, conns)]
    gconns = [gt.Connection() for _ in grpc]
    sd = SnapshotDir(path, "periodic")
    sd.restore([lim.store])

    def one(now, opening=False):
        ids = rng.integers(0, keys, (2, conns, depth))
        cs = [("resp", b"".join(resp_req("k:%d" % k) for k in row)) for row in ids[0]]
        cs += [("http", b"".join(http_req("k:%d" % k) for k in row)) for row in ids[1]]
        for g, cn in zip(grpc, gconns):
            cn.buf += g.opening if opening else b"".join(g.next() for _ in range(depth))
            cn.out.clear()
        cs += [("grpc", cn) for cn in gconns]
        t0 = time.perf_counter()
        mixed.process_connections(cs, lim, now, ring)
        return 1e3 * (time.perf_counter() - t0)
    now = traces.T0 + 3600 * 10**9
    one(now, opening=True)                             # the gRPC openings, and every launch shape
    one(now)
    plain, saving = [], []
    try:
        for i in range(2 * rounds):
            now += 10**8
            if i % 2:
                assert sd.begin()
                saving.append(one(now))
                while sd.in_flight():                  # (the round's save committed; not timed)
                    sd.poll()
                    time.sleep(0.001)
            else:
                plain.append(one(now))
    finally:
        sd.close()
    return {"connections": 3 * conns, "depth": depth, "rounds": rounds,
            "without_save_ms": {"median": float(np.median(plain)), "max": float(np.max(plain))},
            "with_save_ms": {"median": float(np.median(saving)), "max": float(np.max(saving))}}


def capture_ms(st, path, reps=3):
    from torch.profiler import ProfilerActivity, profile
    times = []
    for _ in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            st.save_begin(path)
            st.save_wait()
            torch.cuda.synchronize()
        ks = [e for e in prof.events() if "snapshot_capture_kernel" in e.name]
        assert len(ks) == 1, [e.name for e in prof.events()][:20]
        times.append(ks[0].device_time / 1e3)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, action="append")
    ap.add_argument("--conns", type=int, default=4096)
    ap.add_argument("--depth", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("server_snapshot_e2e.py measures on a GPU; there is none here")
    gpu = gpu_info()
    for keys in a.keys or [1_000_000, 10_000_000]:
        tmp = tempfile.mkdtemp(prefix="gcra_server_snapshot_")
        out = {"gpu": gpu, "keys": keys}
        try:
            one, lim = filled(keys)
            d1, d2 = os.path.join(tmp, "one"), os.path.join(tmp, "two")
            out["save_s"] = {"1": save_from(d1, [one])}
            st = store(keys)
            out["restore_s"] = {"1->1": restore_into(d1, [st])}
            out["len"] = {"saved": one.len(), "1->1": st.len()}
            st.close()
            two = [store(-(-keys // 2)) for _ in range(2)]
            out["restore_s"]["1->2"] = restore_into(d1, two)
            out["len"]["1->2"] = sum(s.len() for s in two)
            out["save_s"]["2"] = save_from(d2, two)
            for s in reversed(two):
                s.close()
            st = store(keys)
            out["restore_s"]["2->1"] = restore_into(d2, [st])
            out["len"]["2->1"] = st.len()
            st.close()
            out["serve"] = serve_rounds(lim, keys, a.conns, a.depth, a.rounds, os.path.join(tmp, "serve"))
            out["capture_ms"] = capture_ms(one, os.path.join(tmp, "capture.gcra"))
            one.close()
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
