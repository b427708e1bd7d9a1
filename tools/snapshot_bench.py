"""Background snapshot (gcra_snapshot_begin) against the blocking gcra_snapshot_save, on the bench's table: 10 M keys
after a warm pass, Zipf-1.0 ticks of 2^20 requests (tests/traces.py config2).  One JSON line:

  capture        snapshot_capture_kernel's device time (torch.profiler), and its achieved bandwidth in algorithmic
                 bytes (32 B read per slot + 32 B written per entry) against the H100 SXM data sheet's 3.35 TB/s
  ticks          device time of every pipelined tick submitted back to back (the interval between the completion events
                 of consecutive ticks), with a background save begun after tick `cut`, and in a run without a save:
                 median, maximum and the ticks around the cut
  save_v2_s      wall time of the blocking gcra_snapshot_save of the same table
  background_s   wall time from gcra_snapshot_begin, called between ticks, until the file is complete
                 (gcra_snapshot_wait); background_quiescent_s the same on an idle engine
  file_bytes     both files' sizes
  gpu            name, power limit and max SM clock, read in the same run

    python tools/snapshot_bench.py [--keys N] [--ticks T] [--cut C]

The files go to a temporary directory that is removed afterwards.
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
import torch  # noqa: E402

import throttlecrab_b200 as tc  # noqa: E402
import traces  # noqa: E402

TICK = 1 << 20
PEAK_HBM_GBS = 3350.0          # NVIDIA's data sheet for the H100 SXM: a bound, not a reached figure


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else None


def device_rows(tr, dev):
    out = []
    for a in range(0, len(tr), TICK):
        t = tr[a:a + TICK]
        r = np.empty(len(t), tc.REQ_DTYPE)
        r["key_hash"] = tc.hash_key_ids(t["key"])
        for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
            r[f] = t[f]
        out.append(torch.from_numpy(r.view(np.uint8)).to(dev))
    return out


def timed_ticks(lim, qs, res, dev, cut=None, path=None):
    """submit every tick pipelined, back to back; after each, a side stream joins the engine and records an event.
    Returns the per-tick device times (ms) and, with `cut`, when begin was called (time.perf_counter) and how long
    the call took (ms)."""
    side = torch.cuda.Stream(dev)
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(len(qs) + 1)]
    cur = torch.cuda.current_stream(dev)
    evs[0].record(side)
    begin_at = begin_ms = None
    for i, q in enumerate(qs):
        lim.submit_device(TICK, q.data_ptr(), res.data_ptr(), cur.cuda_stream)
        lim.join(side.cuda_stream)
        evs[i + 1].record(side)
        if i == cut:
            begin_at = time.perf_counter()
            lim.store.save_begin(path)
            begin_ms = 1e3 * (time.perf_counter() - begin_at)
    torch.cuda.synchronize()
    return [evs[i].elapsed_time(evs[i + 1]) for i in range(len(qs))], (begin_at, begin_ms)


def summary(ms, cut):
    return {"median_ms": float(np.median(ms)), "max_ms": float(np.max(ms)),
            "around_cut_ms": [round(x, 4) for x in ms[max(cut - 2, 0):cut + 4]]}


def capture_ms(lim, path, reps=3):
    """snapshot_capture_kernel's device time from torch.profiler, median over `reps` quiescent saves"""
    from torch.profiler import ProfilerActivity, profile
    times = []
    for _ in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            lim.store.save_begin(path)
            lim.store.save_wait()
            torch.cuda.synchronize()
        ks = [e for e in prof.events() if "snapshot_capture_kernel" in e.name]
        assert len(ks) == 1, [e.name for e in prof.events()][:20]
        times.append(ks[0].device_time / 1e3)
    return float(np.median(times)), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=10_000_000)
    ap.add_argument("--ticks", type=int, default=24)
    ap.add_argument("--cut", type=int, default=12)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("snapshot_bench.py measures on a GPU; there is none here")
    dev = torch.device("cuda", 0)
    out = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(0), "keys": args.keys, "tick": TICK}
    lim = tc.RateLimiter(tc.ManualStore(capacity=args.keys, created_ns=traces.T0, max_batch=TICK))
    warm = traces.warm_pass(args.keys)
    req = np.empty(TICK, tc.REQ_DTYPE)
    for a in range(0, args.keys, TICK):
        w = warm[a:a + TICK]
        r = req[:len(w)]
        r["key_hash"] = tc.hash_key_ids(w["key"])
        for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
            r[f] = w[f]
        lim.rate_limit_batch(r)
    n_ticks = 2 * args.ticks + 4
    qs = device_rows(traces.config2(n_keys=args.keys, n_ticks=n_ticks, tick_size=TICK), dev)
    res = torch.empty(TICK * 32, dtype=torch.uint8, device=dev)
    tmp = tempfile.mkdtemp(prefix="gcra_snapshot_bench_")
    try:
        bg = os.path.join(tmp, "bg.gcra")
        timed_ticks(lim, qs[:4], res, dev)                                  # warm-up: every launch shape
        # the first save makes the staging (pinned chunks, device sections) that later saves reuse: timed on its own
        t0 = time.perf_counter()
        lim.store.save_begin(bg)
        out["first_begin_call_ms"] = 1e3 * (time.perf_counter() - t0)
        lim.store.save_wait()
        plain, _ = timed_ticks(lim, qs[4:4 + args.ticks], res, dev)
        saving, (begin_at, begin_ms) = timed_ticks(lim, qs[4 + args.ticks:], res, dev, args.cut, bg)
        lim.store.save_wait()
        out["background_s"] = time.perf_counter() - begin_at
        out["begin_call_ms"] = begin_ms
        out["ticks"] = {"without_save": summary(plain, args.cut), "with_save": summary(saving, args.cut),
                        "cut_after_tick": args.cut, "n": args.ticks}
        s = lim.store.stats()
        slots = s["table_slots"]
        t0 = time.perf_counter()
        lim.store.save_begin(bg)
        lim.store.save_wait()
        out["background_quiescent_s"] = time.perf_counter() - t0
        v2 = os.path.join(tmp, "v2.gcra")
        t0 = time.perf_counter()
        lim.store.save(v2)
        out["save_v2_s"] = time.perf_counter() - t0
        out["file_bytes"] = {"v2": os.path.getsize(v2), "v3": os.path.getsize(bg)}
        ms, runs = capture_ms(lim, bg)
        entries = lim.store.len()
        alg = 32.0 * slots + 32.0 * entries
        out["capture"] = {"kernel": "snapshot_capture_kernel", "table_slots": slots, "entries": entries,
                          "ms": ms, "runs_ms": runs, "algorithmic_bytes": alg, "achieved_GBps": alg / ms / 1e6,
                          "frac_of_datasheet": alg / ms / 1e6 / PEAK_HBM_GBS}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    lim.store.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
