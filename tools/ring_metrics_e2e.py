"""What ring metrics cost a mixed ring: the same connections through two mixed rings on two engines, one with metrics
off (as before) and one with a metrics.Metrics (denied tracking of 100 keys and ring metrics on), alternated in one
run.  Both must give the same reply bytes in every repetition.  Connections are split evenly over RESP, HTTP and gRPC
with Zipf(1.1) keys (tools/mixed_ring_e2e.py's), so the hot keys are denied and named.  Shapes: 3 x C connections with
R requests each.  Reported per shape: medians of the submit-to-wait time of both, the throughput lost, and
ring_metrics_kernel's and the denied count's device time per submit (torch.profiler, CUDA activities, in a run of
their own).  Prints one JSON line per shape, plus the card and its power limit.

    python tools/ring_metrics_e2e.py [--reps 9] [--shapes 16x8,256x8,4096x1,4096x8] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, "tests"))
sys.path.insert(0, os.path.join(_ROOT, "tools"))
from throttlecrab_b200.metrics import Metrics  # noqa: E402
from mixed_ring_e2e import MixedPath, connections, kernel_ms  # noqa: E402
from resp_ring_e2e import card  # noqa: E402

KERNELS = ("ring_metrics_kernel", "denied_count_seg_kernel", "ring_parse_kernel<gcra::MixedTraits>",
           "ring_reply_kernel<gcra::MixedTraits>", "ring_outcome_kernel<gcra::MixedTraits>")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--shapes", default="16x8,256x8,4096x1,4096x8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    rng = np.random.default_rng(1)
    lines = []
    for shape in a.shapes.split(","):
        n_per, per = (int(x) for x in shape.split("x"))
        conns = connections(n_per, per, rng)
        paths = {"off": MixedPath(conns), "on": MixedPath(conns)}
        m = Metrics(paths["on"].lim, 100)
        t = {v: [] for v in paths}
        reqs = 0
        for rep in range(a.reps + 1):                     # rep 0 warms up
            got = {}
            for v in (("off", "on") if rep % 2 == 0 else ("on", "off")):
                t0 = time.perf_counter()
                got[v] = paths[v].run(conns)
                if rep:
                    t[v].append(time.perf_counter() - t0)
            reqs = got["off"][0]
            if got["off"] != got["on"]:
                raise SystemExit("reply bytes with ring metrics differ from those without (%s)" % shape)
        counts = m.counts()
        k_on = kernel_ms(paths["on"], conns, KERNELS)
        k_off = kernel_ms(paths["off"], conns, KERNELS)
        off, on = np.median(t["off"]), np.median(t["on"])
        line = {"shape": "3x" + shape, "conns": len(conns), "requests": reqs,
                "off_ms": round(1e3 * off, 3), "on_ms": round(1e3 * on, 3),
                "off_mrps": round(reqs / off / 1e6, 3), "on_mrps": round(reqs / on / 1e6, 3),
                "throughput_lost_pct": round(100 * (1 - off / on), 2),
                "ring_metrics_kernel_ms": k_on.get("ring_metrics_kernel", 0.0),
                "denied_count_ms": k_on.get("denied_count_seg_kernel", 0.0),
                "kernel_ms_on": k_on, "kernel_ms_off": k_off,
                "counted": {"redis": sum(counts[0]), "http": sum(counts[1]), "grpc": sum(counts[2]),
                            "denied": sum(c[1] for c in counts)},
                "named_top_keys": len(m.top_denied_keys()), "replies_equal": True}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del paths, m
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps({"card": card()}) + "\n")
            for x in lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
