"""What sharded ring metrics (gcra_ring_metrics_sharded, metrics.ShardedMetrics) cost rings over peer memory.

Per world (1, 2 and 4 loop-back engines on ONE GPU, sharded.connect_local, every mixed ring on peer-memory ticks) two
sets of engines serve the same connections, split in order over the ranks: one with metrics off, one with a
ShardedMetrics (denied tracking of 100 keys and sharded ring metrics on every rank).  The two alternate in one run and
must give the same reply bytes in every repetition.  Connections are tools/mixed_ring_e2e.py's (3 x C of R requests,
RESP, HTTP and gRPC interleaved, Zipf(1.1) keys, so the hot keys are denied and named).  Reported per world: medians
of ms per submit round of both, and ring_metrics_kernel's device time per round summed over the ranks (torch.profiler,
CUDA activities, in a pass of its own).

Then the scrape's two calls on one engine whose name table holds 3 x k names (k = 100 and 10,000): the lookup
(gcra_denied_names on the name table) of those 3 x k hashes, and the keep (gcra_ring_names_keep) of k of them.  Each
is timed with a host clock around the call, which ends in a device synchronise (median of --reps), and its kernel by
torch.profiler.  Prints the card and its power limit, then one JSON line per world and per k.

    python tools/sharded_ring_metrics_e2e.py [--reps 7] [--shape 4096x8] [--worlds 1,2,4] [--ks 100,10000] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

# engines of one process wait for each other in kernels: one hardware queue per stream (as bench.py)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, "tests"))
sys.path.insert(0, os.path.join(_ROOT, "tools"))
import throttlecrab_b200 as tc  # noqa: E402
from throttlecrab_b200.metrics import ShardedMetrics  # noqa: E402
from mixed_ring_e2e import NOW, ROW_CAP, _engine, _fill, connections, kernel_ms  # noqa: E402
from resp_ring_e2e import card  # noqa: E402
from sharded_ring_e2e import ShardedPath  # noqa: E402


def denied_frame(key):
    """a THROTTLE that is denied: quantity 5 over a burst of 1"""
    a = [b"THROTTLE", key, b"1", b"1", b"60", b"5"]
    return b"*6\r\n" + b"".join(b"$%d\r\n%s\r\n" % (len(x), x) for x in a)


def median_ms(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return round(1e3 * float(np.median(t)), 4)


def scrape_calls(k, reps):
    """the lookup of 3 x k hashes and the keep of k, on a name table of max_keys k holding 3 x k names"""
    lim = _engine()
    lim.store.ring_metrics_sharded(True, k)
    keys = [b"n:%d" % i for i in range(3 * k)]
    conns, b = [], bytearray()
    for key in keys:
        f = denied_frame(key)
        if len(b) + len(f) > 65536:
            conns.append(("resp", bytes(b), None))
            b = bytearray()
        b += f
    conns.append(("resp", bytes(b), None))
    ring = tc.MixedRing(lim, 1, len(conns), sum(len(x) for _, x, _ in conns), ROW_CAP)
    _fill(ring, conns, True)
    ring.submit(0, len(conns), NOW)
    ring.wait(0)
    hs = [lim.store.hash_key(x) for x in keys]
    names = lim.store.denied_names(hs)
    named = sum(isinstance(x, bytes) for x in names)
    lookup = median_ms(lambda: lim.store.denied_names(hs), reps)
    keep = median_ms(lambda: lim.store.ring_names_keep(hs[:k]), reps)      # (the same k survive every time)
    ks = _kernels(lambda: (lim.store.denied_names(hs), lim.store.ring_names_keep(hs[:k])))
    return {"k": k, "table_entries": 1 << max(10, (16 * k - 1).bit_length()), "names_in_table": named,
            "lookup_hashes": len(hs), "lookup_ms": lookup, "keep_hashes": k, "keep_ms": keep,
            "lookup_kernel_ms": ks.get("ring_names_lookup_kernel", 0.0),
            "keep_kernel_ms": ks.get("ring_names_keep_kernel", 0.0)}


def _kernels(fn, iters=5):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            for name in ("ring_names_lookup_kernel", "ring_names_keep_kernel"):
                if name in e.name:
                    tot[name] = tot.get(name, 0.0) + e.device_time / 1000.0
    return {n: round(v / iters, 4) for n, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--shape", default="4096x8")
    ap.add_argument("--worlds", default="1,2,4")
    ap.add_argument("--ks", default="100,10000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    head = {"card": card(), "note": "loop-back on one GPU: no NVLink traffic is measured"}
    print(json.dumps(head), flush=True)
    lines = []
    n_per, per = (int(x) for x in a.shape.split("x"))
    conns = connections(n_per, per, np.random.default_rng(1))
    for w in (int(x) for x in a.worlds.split(",")):
        paths = {"off": ShardedPath(conns, w), "on": ShardedPath(conns, w)}
        m = ShardedMetrics(paths["on"].lims, 100)
        t = {v: [] for v in paths}
        reqs = 0
        for rep in range(a.reps + 1):                      # rep 0 warms up
            got = {}
            for v in (("off", "on") if rep % 2 == 0 else ("on", "off")):
                t0 = time.perf_counter()
                got[v] = paths[v].run(conns)
                if rep:
                    t[v].append(time.perf_counter() - t0)
            reqs = got["off"][0]
            if got["off"] != got["on"]:
                raise SystemExit("reply bytes with sharded metrics differ from those without (world %d)" % w)
        k_on = kernel_ms(paths["on"], conns, ("ring_metrics_kernel",))
        off, on = float(np.median(t["off"])), float(np.median(t["on"]))
        counts = m.counts()
        line = {"world": w, "shape": "3x" + a.shape, "conns": len(conns), "requests": reqs,
                "off_ms": round(1e3 * off, 3), "on_ms": round(1e3 * on, 3),
                "off_ms_min_max": [round(1e3 * min(t["off"]), 3), round(1e3 * max(t["off"]), 3)],
                "on_ms_min_max": [round(1e3 * min(t["on"]), 3), round(1e3 * max(t["on"]), 3)],
                "ring_metrics_kernel_ms_per_round": k_on.get("ring_metrics_kernel", 0.0),
                "counted": sum(sum(c) for c in counts), "denied": sum(c[1] for c in counts),
                "named_top_keys": len(m.top_denied_keys()), "replies_equal": True}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del paths, m
    for k in (int(x) for x in a.ks.split(",")):
        line = scrape_calls(k, a.reps)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            for x in [head] + lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
