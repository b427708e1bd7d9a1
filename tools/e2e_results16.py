"""End-to-end rate through the pinned ring with 16-byte requests: 32-byte results (ring mode 1) against 16-byte
results (ring mode 2), plus what explains the difference.

One run prints one JSON line with:
  gpu           name and power limit (read-only nvidia-smi query)
  link          pinned H2D, D2H and duplex GB/s (as tools/pcie_probe.py measures them)
  ring          decisions/s of mode 1 and mode 2, alternated over --reps repetitions (median, min, max of each)
  kernel_ms     device time of one 2^20-row tick, gcra_rate_limit_batch16_device against the _r16_device variant
                (CUDA events, median of --reps alternated calls)
  expand_cpu    rows/s of gcra_expand_results16 on ONE CPU core (host work, not GPU): what a server pays per row to
                get the full 32-byte result back
The workload is bench.py's e2e leg: seeded Zipf ticks of 2^20 requests over 10 M keys (traces.config2), the 8-entry
policy table, keys inserted by a warm pass.  Two engines run the same ticks, one per mode; every timed tick's mode-2
results, expanded on the host, must equal mode 1's results byte for byte, else the script exits with status 1.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import throttlecrab_b200 as tc  # noqa: E402
import traces  # noqa: E402

TICK = 1 << 20


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as ex:
        out = "nvidia-smi unavailable: %r" % ex
    return {"nvidia_smi": out, "torch_name": torch.cuda.get_device_name(0)}


def link_bandwidth(n=256 << 20, reps=5):
    h = torch.empty(n, dtype=torch.uint8).pin_memory()
    d = torch.empty(n, dtype=torch.uint8, device="cuda")
    h2 = torch.empty(n, dtype=torch.uint8).pin_memory()
    d2 = torch.empty(n, dtype=torch.uint8, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def best_ms(fn):
        best = 1e9
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            best = min(best, a.elapsed_time(b))
        return best

    def both():
        with torch.cuda.stream(s1):
            d.copy_(h, non_blocking=True)
        with torch.cuda.stream(s2):
            h2.copy_(d2, non_blocking=True)
        torch.cuda.current_stream().wait_stream(s1)
        torch.cuda.current_stream().wait_stream(s2)

    out = {"h2d_GBps": n / best_ms(lambda: d.copy_(h, non_blocking=True)) / 1e6,
           "d2h_GBps": n / best_ms(lambda: h.copy_(d, non_blocking=True)) / 1e6,
           "duplex_each_GBps": n / best_ms(both) / 1e6}
    del h, d, h2, d2
    return out


def policy_table():
    pol = np.zeros(len(traces.POLICIES), tc.POLICY_DTYPE)
    pol["max_burst"], pol["count_per_period"], pol["period"] = traces.POLICIES.T
    return pol


def compact_ticks(n_keys, n_ticks):
    key_hash_of = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64))
    tr = traces.config2(n_keys=n_keys, n_ticks=n_ticks, tick_size=TICK)
    req = np.zeros(len(tr), tc.REQ16_DTYPE)
    req["key_hash"] = key_hash_of[tr["key"].astype(np.int64)]
    req["quantity"] = tr["quantity"]
    req["policy"] = (tr["key"] % np.uint64(8)).astype(np.uint32)     # config2: policy = key & 7
    nows = [int(tr["now_ns"][t * TICK]) for t in range(n_ticks)]
    warm = np.zeros(n_keys, tc.REQ16_DTYPE)
    warm["key_hash"] = key_hash_of
    warm["quantity"] = 1
    warm["policy"] = (np.arange(n_keys) % 8).astype(np.uint32)
    return req.reshape(n_ticks, TICK), nows, warm


def make_engine(n_keys, warm, mode, slots):
    st = tc.ManualStore(capacity=n_keys, created_ns=traces.T0, max_batch=TICK)
    lim = tc.RateLimiter(st)
    lim.set_policies(policy_table())
    for a in range(0, n_keys, TICK):
        lim.rate_limit_batch16(warm[a:a + TICK], traces.T0)
    ring = tc.Ring(lim, slots=slots, slot_capacity=TICK, compact=mode)
    return st, lim, ring


def run_ring(ring, st, ticks, nows, W, K, shift):
    for i in range(W + K):
        ring.req[i][:] = ticks[i]
    for i in range(W):
        ring.submit(i, TICK, nows[i] + shift)
    for i in range(W):
        ring.wait(i)
    st.sync()
    t_a = time.perf_counter()
    for i in range(W, W + K):
        ring.submit(i, TICK, nows[i] + shift)
    for i in range(W, W + K):
        ring.wait(i)
    t_b = time.perf_counter()
    return K * TICK / (t_b - t_a), [ring.res[i].copy() for i in range(W, W + K)]


def spread(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "runs": [float(x) for x in v]}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--keys", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=16, help="timed ticks per repetition")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    W, K = args.warmup, args.steps
    out = {"gpu": gpu_info(), "workload": "config2 Zipf ticks of 2^20 compact requests over %d keys, 8 policies, "
                                          "%d warm-up + %d timed ticks per repetition" % (args.keys, W, K)}
    out["link"] = link_bandwidth()

    ticks, nows, warm = compact_ticks(args.keys, W + K)
    eng = {m: make_engine(args.keys, warm, m, W + K) for m in (1, 2)}
    pol = policy_table()
    rates = {1: [], 2: []}
    mismatches = 0
    for r in range(args.reps):
        shift = r * (W + K + 1) * 1_000_000          # every repetition decides later ticks on both engines
        res = {}
        for m in ((1, 2) if r % 2 == 0 else (2, 1)):
            st, _, ring = eng[m]
            rate, res[m] = run_ring(ring, st, ticks, nows, W, K, shift)
            rates[m].append(rate)
        for j in range(K):
            full = tc.expand_results16(ticks[W + j], nows[W + j] + shift, pol, res[2][j])
            if full.tobytes() != res[1][j].tobytes():
                mismatches += 1
    out["ring"] = {"mode1_16B_req_32B_res": spread(rates[1]), "mode2_16B_req_16B_res": spread(rates[2]),
                   "unit": "decisions/s", "d2h_bytes_per_tick": {"mode1": TICK * 32, "mode2": TICK * 16},
                   "h2d_bytes_per_tick": TICK * 16, "timed_ticks_compared": args.reps * K,
                   "expanded_mode2_equals_mode1": mismatches == 0}

    # kernel-only: one device-resident tick per call, both result formats, alternated
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    d_req = torch.from_numpy(ticks[W].view(np.uint8)).to(dev)
    d_res = torch.empty(TICK * 32, dtype=torch.uint8, device=dev)
    ms = {False: [], True: []}
    for r in range(2 * args.reps + 2):
        r16 = r % 2 == 1
        _, lim, _ = eng[2 if r16 else 1]
        now = nows[W] + (args.reps + 2 + r) * (W + K + 1) * 1_000_000
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record(stream)
        lim.rate_limit_batch16_device(TICK, d_req.data_ptr(), now, d_res.data_ptr(), stream.cuda_stream,
                                      compact_results=r16)
        b.record(stream)
        torch.cuda.synchronize()
        if r >= 2:
            ms[r16].append(a.elapsed_time(b))
    out["kernel_ms"] = {"batch16_device_32B_res": spread(ms[False]), "batch16_r16_device_16B_res": spread(ms[True]),
                        "rows": TICK}

    # host expansion, one thread
    best = 1e9
    for _ in range(5):
        t0 = time.perf_counter()
        tc.expand_results16(ticks[W], nows[W], pol, res[2][0])
        best = min(best, time.perf_counter() - t0)
    out["expand_cpu"] = {"rows_per_s": TICK / best, "rows": TICK, "note": "CPU work, one core, best of 5"}
    for m in eng:
        eng[m][0].close()
    print(json.dumps(out), flush=True)
    if mismatches:
        raise SystemExit("%d timed ticks: expanded mode-2 results differ from mode 1" % mismatches)


if __name__ == "__main__":
    main()
