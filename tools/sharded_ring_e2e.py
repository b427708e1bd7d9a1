"""What serving the mixed ring over peer memory (gcra_ring_p2p) adds to a submit round.  Shapes and connections are
tools/mixed_ring_e2e.py's (3 x C connections with R requests each, keys Zipf(1.1)); the variants:
  (a) one engine's plain mixed ring (mixed_ring_e2e's (b));
  (b) the same ring with ring p2p on, world 1: the slot's rows go through the peer-memory tick to the one owner;
  (c) 2 and 4 engines on ONE GPU (loop-back, sharded.connect_local), the connections split in order over them, every
      round all routes then all finishes then all waits.
The variants alternate in one run, every variant must give (a)'s reply bytes in every repetition (the rows are decided
in the same order against one table), and medians of ms per submit round are reported, with rank 0's p2p stage times
(gcra_p2p_set_timing, one round at a time, in a pass of their own).  The loop-back runs every engine on one GPU: it
measures the launches and flag waits a tick adds, not NVLink.  Every round is also split into its host-side parts
(fill, submit calls, waits, replies read back), and the spread of the round times is printed.  Prints the card and
its power limit, then one JSON line per shape.

    python tools/sharded_ring_e2e.py [--reps 7] [--shapes 16x8,256x8,4096x1,4096x8] [--worlds 2,4] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

# engines of one process wait for each other in kernels: one hardware queue per stream (as bench.py)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, "tools"))
import throttlecrab_b200 as tc  # noqa: E402
from throttlecrab_b200.sharded import connect_local  # noqa: E402
from mixed_ring_e2e import NOW, ROW_CAP, MixedPath, _engine, _fill, _replies, connections  # noqa: E402
from resp_ring_e2e import card  # noqa: E402


class PlainPath(MixedPath):
    """(a), with the round's parts timed as ShardedPath times them"""

    def run(self, conns):
        t0 = time.perf_counter()
        _fill(self.ring, conns, True)
        t1 = time.perf_counter()
        self.ring.submit(0, len(conns), NOW)
        t2 = time.perf_counter()
        self.ring.wait(0)
        t3 = time.perf_counter()
        out = (int(self.ring.outcome[0][:len(conns)]["n_frames"].sum()), _replies(self.ring, len(conns)))
        self.parts_ms = (t1 - t0, t2 - t1, t3 - t2, time.perf_counter() - t3)
        return out


class ShardedPath:
    """`world` engines on one GPU, each a mixed ring with ring p2p on; connections split in order over the ranks"""

    def __init__(self, conns, world):
        self.world = world
        self.lims = [_engine() for _ in range(world)]
        cut = np.linspace(0, len(conns), world + 1).astype(int)
        self.parts = [(int(cut[r]), int(cut[r + 1])) for r in range(world)]
        self.rings = []
        for lim, (a, b) in zip(self.lims, self.parts):
            mine = conns[a:b]
            self.rings.append(tc.MixedRing(lim, 1, max(len(mine), 1), max(sum(len(x) for _, x, _ in mine), 1),
                                           ROW_CAP))
        connect_local(self.lims, ROW_CAP)
        for ring in self.rings:
            ring.peer_memory(True)

    def run(self, conns):
        t0 = time.perf_counter()
        for ring, (a, b) in zip(self.rings, self.parts):
            _fill(ring, conns[a:b], True)
        t1 = time.perf_counter()
        for ring, (a, b) in zip(self.rings, self.parts):
            ring.submit_route(0, b - a, NOW)
        for ring in self.rings:
            ring.submit_finish(0)
        t2 = time.perf_counter()
        for ring in self.rings:
            ring.wait(0)
        t3 = time.perf_counter()
        n, out = 0, []
        for ring, (a, b) in zip(self.rings, self.parts):
            n += int(ring.outcome[0][:b - a]["n_frames"].sum())
            out += _replies(ring, b - a)
        self.parts_ms = (t1 - t0, t2 - t1, t3 - t2, time.perf_counter() - t3)
        return n, out

    def stage_ms(self, conns, iters=5):
        """rank 0's p2p stage times, rounds one at a time: [route, wait for senders, owner batch, wait for owners,
        unpermute]"""
        L = self.lims[0]._L
        for lim in self.lims:
            lim.store._check(L.gcra_p2p_set_timing(lim._h, 1))
        acc = np.zeros(5)
        for _ in range(iters):
            self.run(conns)
            out = (C.c_float * 5)()
            self.lims[0].store._check(L.gcra_p2p_last_tick_ms(self.lims[0]._h, C.byref(out)))
            acc += np.array(out[:])
        for lim in self.lims:
            lim.store._check(L.gcra_p2p_set_timing(lim._h, 0))
        return [round(x, 4) for x in acc / iters]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--shapes", default="16x8,256x8,4096x1,4096x8")
    ap.add_argument("--worlds", default="2,4")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print(json.dumps({"card": card(), "note": "loop-back on one GPU: no NVLink traffic is measured"}), flush=True)
    rng = np.random.default_rng(1)
    worlds = [int(w) for w in a.worlds.split(",")]
    lines = []
    for shape in a.shapes.split(","):
        n_per, per = (int(x) for x in shape.split("x"))
        conns = connections(n_per, per, rng)
        paths = {"a": PlainPath(conns), "b": ShardedPath(conns, 1)}
        for w in worlds:
            paths["c%d" % w] = ShardedPath(conns, w)
        t = {v: [] for v in paths}
        parts = {v: [] for v in paths}
        reqs = 0
        for rep in range(a.reps + 1):                     # rep 0 warms up
            got = {}
            order = list(paths) if rep % 2 == 0 else list(reversed(list(paths)))
            for v in order:
                t0 = time.perf_counter()
                got[v] = paths[v].run(conns)
                dt = time.perf_counter() - t0
                if rep:
                    t[v].append(dt)
                    parts[v].append(paths[v].parts_ms)
            reqs = got["a"][0]
            for v in paths:
                if got[v] != got["a"]:
                    raise SystemExit("reply bytes of %s differ from the plain mixed ring (%s)" % (v, shape))
        line = {"shape": "3x" + shape, "conns": len(conns), "requests": reqs, "replies_equal": True}
        for v in paths:
            line["%s_ms" % v] = round(1e3 * np.median(t[v]), 3)
            line["%s_ms_min_max" % v] = [round(1e3 * min(t[v]), 3), round(1e3 * max(t[v]), 3)]
            # medians of the round's parts: fill the slots, the submit calls, the waits, the replies read back
            line["%s_parts_ms" % v] = [round(1e3 * x, 3) for x in np.median(np.array(parts[v]), axis=0)]
        for v in paths:
            if v != "a":
                line["%s_stage_ms" % v] = paths[v].stage_ms(conns)
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
