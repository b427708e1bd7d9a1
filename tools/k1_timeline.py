"""Kernel timeline of the pipelined N=1 ticks (the bench.py workload): where stage 2 of the sort pipeline, "decide
+ hot runs", spends its time, and what runs beside it.

The workload is bench.py's: 10 M resident keys (warm pass), then Zipf-1.0 ticks of 2^20 requests (tests/traces.py
config2) submitted with submit_device.  After the warm-up ticks, one window of --ticks pipelined ticks runs under
torch.profiler (CUDA activities); every kernel's start, end and stream go to OUT/k1_timeline.json.  Per tick it prints
  decide_ms    the decide_kernel launch that decides the batch (the last one of the tick)
  list_ms      the list_runs_kernel launch before it that lists the hot runs (if there is one)
  runs1_ms / runsC_ms   the one-CTA and the cluster hot-run kernel
  tail_ms      from the end of that decide_kernel to the end of the last hot-run kernel: the time in which
               only hot-run kernels of the tick are left (0 when they end first)
  front_in_tail  whether a kernel of the next tick's front stage (ingest, sort) ran during the tail
and the pipelined tick (window / ticks).  It also prints the card, its power limit, and the occupancy of the decide
kernels (tools/k1_occupancy.cu, built with the library's flags into a temporary directory).
  python tools/k1_timeline.py --out DIR [--defines="-DGCRA_CLUSTER=16 ..."]   (DIR: a temporary directory by default)
The profiler slows the host: take throughput from bench.py, not from this run."""
import argparse
import json
import os
import re
import shlex
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
from throttlecrab_b200 import _native  # noqa: E402
import traces  # noqa: E402

TICK = 1 << 20
FRONT = ("ingest_kernel", "sort_digits_kernel", "sort_sweep_kernel", "probe_kernel")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": q}


def occupancy(defines):
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "k1_occupancy")
        flags, nf = [], _native.NVCC_FLAGS            # the library's flags, less the shared-library ones
        for i, f in enumerate(nf):
            if f in ("--shared", "-ldl", "-fPIC") or (f == "-Xcompiler" and nf[i + 1] == "-fPIC"):
                continue
            flags.append(f)
        subprocess.check_call(["nvcc"] + flags + shlex.split(defines) + ["-o", exe, os.path.join(ROOT, "tools", "k1_occupancy.cu")])
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    return [json.loads(line) for line in out.splitlines() if line.strip()]


def requests(trace, kh):
    req = np.empty(len(trace), tc.REQ_DTYPE)
    req["key_hash"] = kh[trace["key"].astype(np.int64)]
    for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
        req[f] = trace[f]
    return req


def short(name):
    m = re.search(r"(\w+_kernel)(<[^()]*>)?", name)
    return (m.group(1) + (m.group(2) or "")) if m else name


def per_tick(kernels):
    """kernels in launch order; a tick starts at its front stage's first kernel"""
    ticks, cur = [], None
    for k in kernels:
        if k["name"].split("<")[0] in ("ingest_kernel", "probe_kernel"):
            cur = []
            ticks.append(cur)
        if cur is not None:
            cur.append(k)
    rows = []
    for i, t in enumerate(ticks):
        dec = [k for k in t if k["name"].startswith(("list_runs_kernel", "decide_kernel"))]
        runs = [k for k in t if k["name"].startswith("decide_runs_kernel")]
        if not dec:
            continue
        d = dec[-1]
        r1 = [k for k in runs if k["name"].startswith("decide_runs_kernel<1,")]
        rc = [k for k in runs if not k["name"].startswith("decide_runs_kernel<1,")]
        hot_end = max([k["end"] for k in runs], default=d["end"])
        tail = max(0.0, hot_end - d["end"])
        nxt = ticks[i + 1] if i + 1 < len(ticks) else []
        front_in_tail = any(k["name"].split("<")[0] in FRONT and k["start"] < hot_end and k["end"] > d["end"] for k in nxt)
        hot_overlaps_decide = any(k["start"] < d["end"] and k["end"] > d["start"] for k in runs)
        rows.append({"tick": i, "decide_ms": (d["end"] - d["start"]) / 1e3,
                     "list_ms": (dec[0]["end"] - dec[0]["start"]) / 1e3 if len(dec) > 1 else None,
                     "runs1_ms": sum(k["end"] - k["start"] for k in r1) / 1e3,
                     "runsC_ms": sum(k["end"] - k["start"] for k in rc) / 1e3,
                     "tail_ms": tail / 1e3, "front_in_tail": front_in_tail,
                     "hot_runs_overlap_decide": hot_overlaps_decide})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "k1_timeline"))
    ap.add_argument("--ticks", type=int, default=8, help="pipelined ticks in the profiled window")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--keys", type=int, default=10_000_000)
    ap.add_argument("--defines", default="", help="preprocessor defines the library was built with (occupancy probe)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("k1_timeline.py needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    info = card()
    info["occupancy"] = occupancy(args.defines)
    print(json.dumps(info), flush=True)

    n_keys, W, K = args.keys, args.warmup, args.ticks
    kh = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64))
    st = tc.ManualStore(capacity=n_keys, created_ns=traces.T0, max_batch=TICK)
    lim = tc.RateLimiter(st)
    warm = requests(traces.warm_pass(n_keys), kh)
    for a in range(0, n_keys, TICK):
        lim.rate_limit_batch(warm[a:a + TICK])
    del warm
    tr = traces.config2(n_keys=n_keys, n_ticks=W + K, tick_size=TICK)
    dev = torch.device("cuda", 0)
    d_req = torch.from_numpy(requests(tr, kh).view(np.uint8).reshape(W + K, TICK * 48)).to(dev)
    d_res = torch.empty((W + K, TICK * 32), dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    for i in range(W):
        lim.submit_device(TICK, d_req[i].data_ptr(), d_res[i].data_ptr(), stream.cuda_stream)
    lim.join(stream.cuda_stream)
    torch.cuda.synchronize()

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(W, W + K):
            lim.submit_device(TICK, d_req[i].data_ptr(), d_res[i].data_ptr(), stream.cuda_stream)
        lim.join(stream.cuda_stream)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    kernels = []
    for e in ev:
        if e.get("cat") != "kernel" or "dur" not in e:
            continue
        a = e.get("args", {})
        kernels.append({"name": short(e["name"]), "start": float(e["ts"]), "end": float(e["ts"]) + float(e["dur"]),
                        "stream": a.get("stream"), "correlation": a.get("correlation", 0)})
    kernels.sort(key=lambda k: (k["correlation"], k["start"]))
    t0 = min(k["start"] for k in kernels)
    window_us = max(k["end"] for k in kernels) - t0
    rows = per_tick(kernels)
    path = os.path.join(args.out, "k1_timeline.json")
    print("kernel timeline: %s" % path, flush=True)
    with open(path, "w") as f:
        json.dump({**info, "t0_us": t0, "kernels": [{**k, "start": k["start"] - t0, "end": k["end"] - t0} for k in kernels],
                   "ticks": rows}, f)
    for r in rows:
        print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}))
    tick_ms = window_us / 1e3 / K
    full = rows[1:-1] or rows     # ticks with both neighbours inside the window
    mean = lambda key: float(np.mean([r[key] for r in full]))  # noqa: E731
    print(json.dumps({"summary": True, "ticks": K, "pipelined_tick_ms": round(tick_ms, 4),
                      "decide_ms": round(mean("decide_ms"), 4), "runs1_ms": round(mean("runs1_ms"), 4),
                      "runsC_ms": round(mean("runsC_ms"), 4), "tail_ms": round(mean("tail_ms"), 4),
                      "tail_share_of_tick": round(mean("tail_ms") / tick_ms, 4),
                      "list_ms": round(float(np.mean([r["list_ms"] for r in full])), 4) if full[0]["list_ms"] is not None else None,
                      "front_in_tail_ticks": sum(r["front_in_tail"] for r in full), "of": len(full)}), flush=True)
    st.close()


if __name__ == "__main__":
    main()
