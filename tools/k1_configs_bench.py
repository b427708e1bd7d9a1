"""Kernel-only K1 throughput on the other BASELINE.json configs (device-resident ticks, CUDA events on
the launching stream, same harness as bench.py's `value`):
  configs[1]  10 M keys, Zipf-1.0           (the bench.py headline, repeated here for comparison)
  configs[3]  10 M keys, top-100 keys = 50 % of the traffic
  configs[2]  100 M keys, uniform           (every probe and state access misses L2)
One JSON line per config."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
import traces  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--configs", default="zipf,hot100,uniform100m")
ap.add_argument("--steps", type=int, default=12)
args = ap.parse_args()
TICK, W, K = 1 << 20, 3, args.steps
peak = 3350.0        # GB/s, NVIDIA's data sheet for the H100 SXM (HBM3): a bound, not a reached figure
dev = torch.device("cuda", 0)
stream = torch.cuda.Stream(dev)
torch.cuda.set_stream(stream)


def rows(trace, kh=None):
    req = np.empty(len(trace), tc.REQ_DTYPE)
    req["key_hash"] = kh[trace["key"].astype(np.int64)] if kh is not None else tc.hash_key_ids(trace["key"])
    for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
        req[f] = trace[f]
    return req


for name in args.configs.split(","):
    n_keys = 100_000_000 if name == "uniform100m" else 10_000_000
    st = tc.ManualStore(capacity=n_keys, created_ns=traces.T0, max_batch=TICK)
    lim = tc.RateLimiter(st)
    kh = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64)) if n_keys <= 10_000_000 else None
    for a in range(0, n_keys, TICK):          # warm pass: every key resident
        ids = np.arange(a, min(a + TICK, n_keys), dtype=np.uint64)
        w = np.zeros(len(ids), traces.REQ_DTYPE)
        w["key"] = ids
        traces.fill_policy(w, (ids % 8).astype(np.int64))
        w["quantity"] = 1
        w["now_ns"] = traces.T0
        lim.rate_limit_batch(rows(w, kh))
    if name == "zipf":
        tr = traces.config2(n_keys=n_keys, n_ticks=W + K, tick_size=TICK)
    elif name == "hot100":
        tr = traces.config4(n_keys=n_keys, n_ticks=W + K, tick_size=TICK)
    else:
        tr = traces.config3(n_keys=n_keys, n_ticks=W + K, tick_size=TICK)
    d_req = torch.from_numpy(rows(tr, kh).view(np.uint8).reshape(W + K, TICK * 48)).to(dev)
    d_res = torch.empty((W + K, TICK * 32), dtype=torch.uint8, device=dev)
    for i in range(W):
        lim.rate_limit_batch_device(TICK, d_req[i].data_ptr(), d_res[i].data_ptr(), stream.cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(W, W + K):
        lim.rate_limit_batch_device(TICK, d_req[i].data_ptr(), d_res[i].data_ptr(), stream.cuda_stream)
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    res = d_res[W:].cpu().numpy().view(tc.RES_DTYPE)
    n_allowed = int(res["allowed"].sum())
    alg = 112.0 * n_allowed + 96.0 * (K * TICK - n_allowed)
    ph = st.last_kernel_ms()
    print(json.dumps({"config": name, "keys": n_keys, "tick": TICK, "ms_per_tick": ms,
                      "decisions_per_s": TICK / ms * 1e3, "allowed_fraction": n_allowed / (K * TICK),
                      "k1_algorithmic_GBps": alg / (ms * K) / 1e6, "frac_of_datasheet_peak": alg / (ms * K) / 1e6 / peak,
                      "last_tick_phase_ms": {"ingest": ph[1], "order": ph[2], "decide": ph[3]},
                      "table_slots": st.stats()["table_slots"], "stash_entries": st.stats()["stash_entries"]}),
          flush=True)
    st.close()
    del d_req, d_res
    torch.cuda.empty_cache()
