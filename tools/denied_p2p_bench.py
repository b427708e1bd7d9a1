"""What top-denied tracking (gcra_track_denied) costs a peer-memory multi-GPU tick (gcra_p2p_*).  Bench workload:
Zipf-1.0 ticks of 2^20 requests per rank over 10 M keys per rank (tests/traces.py config2), after a warm pass that
inserts every key.  Rounds of back-to-back pipelined ticks alternate tracking off and on in one run.  One JSON line:

  tick_ms_off / tick_ms_on   pipelined tick time (all ticks of a round between two CUDA events, / ticks), median
                             over the rounds of each kind
  count_ms                   denied_count_seg_kernel's device time per tick and engine (torch.profiler, one round)
  denied_fraction            denied rows / decided rows of every tick after the warm pass
  gpu                        name, power limit and max SM clock, read in the same run
  remote                     "nvlink" with two GPUs (one process per GPU); "loopback" otherwise: two engines on one
                             GPU, whose "remote" reads never cross NVLink -- that cost is then not measured

    python tools/denied_p2p_bench.py [--keys-per-rank N] [--ticks T] [--rounds R]
"""
import argparse
import json
import os
import socket
import subprocess
import sys

# the loop-back's engines wait for each other's kernels: each needs its own hardware queues (read at CUDA init)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
import traces  # noqa: E402

TICK = 1 << 20
WORLD = 2
MAX_KEYS = 1 << 20


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else None


def device_ticks(tr, dev):
    out = []
    for a in range(0, len(tr), TICK):
        t = tr[a:a + TICK]
        r = np.empty(len(t), tc.REQ_DTYPE)
        r["key_hash"] = tc.hash_key_ids(t["key"])
        for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
            r[f] = t[f]
        out.append(torch.from_numpy(r.view(np.uint8)).to(dev))
    return out


class Engines:
    """the ranks this process drives: both engines (loop-back) or its own (one process per GPU)"""

    def __init__(self, ranks, dev, n_keys, dist=None):
        from throttlecrab_b200.sharded import PeerShardedLimiter, connect_local
        self.ranks, self.dev = ranks, dev
        # room for every key of a rank without growing (a growth waits for the device: in the loop-back, for the
        # other engine's tick too)
        self.lims = [tc.RateLimiter(tc.ManualStore(capacity=2 * n_keys // WORLD, device=dev.index, created_ns=traces.T0,
                                                   max_batch=2 * TICK)) for _ in ranks]
        if dist is None:
            connect_local(self.lims, TICK)
        else:
            self.sh = PeerShardedLimiter(self.lims[0], dist, dev, TICK)
        self.stream = torch.cuda.Stream(dev)
        torch.cuda.set_stream(self.stream)
        self.res = [torch.empty(TICK * 32, dtype=torch.uint8, device=dev) for _ in ranks]

    def submit(self, qs):
        """one tick: qs[i] = the requests of self.ranks[i]"""
        for lim, q in zip(self.lims, qs):
            lim.store._check(lim._L.gcra_p2p_submit_route(lim._h, TICK, q.data_ptr(), self.stream.cuda_stream))
        for lim, r in zip(self.lims, self.res):
            lim.store._check(lim._L.gcra_p2p_submit_finish(lim._h, r.data_ptr()))

    def join(self):
        for lim in self.lims:
            lim.store._check(lim._L.gcra_p2p_join(lim._h, self.stream.cuda_stream))
        torch.cuda.synchronize(self.dev)

    def track(self, on):
        for lim in self.lims:
            lim.store.track_denied(MAX_KEYS if on else 0)


def measure(eng, n_keys, n_ticks, rounds):
    """(report fields) -- every process drives its ranks through the same ticks"""
    # warm pass: every key once (the last tick repeats the first keys), ticks of 2^20 rows per rank
    per_tick = WORLD * TICK
    warm = np.resize(traces.warm_pass(n_keys), -(-n_keys // per_tick) * per_tick)
    for a in range(0, len(warm), per_tick):
        eng.submit([device_ticks(warm[a + r * TICK:a + (r + 1) * TICK], eng.dev)[0] for r in eng.ranks])
        eng.join()
    ticks = [[device_ticks(traces.config2_rank_slice(n_keys, TICK, 1 + i * n_ticks, n_ticks, r, WORLD), eng.dev)
              for r in eng.ranks] for i in range(2 * rounds + 2)]
    ms = {False: [], True: []}
    s0 = [lim.store.stats() for lim in eng.lims]
    for i in range(2 * rounds + 1):
        on = i % 2 == 1
        eng.track(on)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(eng.stream)
        for t in range(n_ticks):
            eng.submit([ticks[i][j][t] for j in range(len(eng.ranks))])
        for lim in eng.lims:
            lim.store._check(lim._L.gcra_p2p_join(lim._h, eng.stream.cuda_stream))
        e1.record(eng.stream)
        eng.join()
        if i > 0:                                   # (round 0: warm-up)
            ms[on].append(e0.elapsed_time(e1) / n_ticks)
    # the count kernel's device time, one more round with tracking on, under the profiler
    eng.track(True)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t in range(n_ticks):
            eng.submit([ticks[-1][j][t] for j in range(len(eng.ranks))])
        eng.join()
    count_us = [e.device_time for e in prof.events() if "denied_count_seg_kernel" in e.name]
    s1 = [lim.store.stats() for lim in eng.lims]
    denied = sum(b["denied"] - a["denied"] for a, b in zip(s0, s1))
    rows = denied + sum(b["allowed"] - a["allowed"] for a, b in zip(s0, s1))
    return {"tick_ms_off": float(np.median(ms[False])), "tick_ms_on": float(np.median(ms[True])),
            "tick_ms_off_all": [round(x, 4) for x in ms[False]], "tick_ms_on_all": [round(x, 4) for x in ms[True]],
            "count_ms": float(np.mean(count_us)) / 1000.0 if count_us else None, "count_launches": len(count_us),
            "denied_fraction": denied / max(rows, 1)}


def _rank_main(rank, port, n_keys, n_ticks, rounds, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=WORLD, device_id=dev)
    eng = Engines([rank], dev, n_keys, dist)
    rep = measure(eng, n_keys, n_ticks, rounds)
    out[rank] = rep
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys-per-rank", type=int, default=10_000_000)
    ap.add_argument("--ticks", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    n_keys = a.keys_per_rank * WORLD
    rep = {"workload": "config2 Zipf-1.0, %d M keys per rank, ticks of 2^20 rows per rank, %d ranks"
                       % (a.keys_per_rank // 1_000_000, WORLD), "ticks_per_round": a.ticks, "gpu": gpu_info()}
    if torch.cuda.device_count() >= WORLD:
        import torch.multiprocessing as mp
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        out = mp.Manager().dict()
        mp.spawn(_rank_main, args=(port, n_keys, a.ticks, a.rounds, out), nprocs=WORLD, join=True)
        rep.update(remote="nvlink", per_rank={r: out[r] for r in range(WORLD)}, **out[0])
    else:
        eng = Engines(list(range(WORLD)), torch.device("cuda", 0), n_keys)
        rep.update(remote="loopback: %d engines on one GPU, remote reads do not cross NVLink (not measured)" % WORLD,
                   **measure(eng, n_keys, a.ticks, a.rounds))
    print(json.dumps(rep))


if __name__ == "__main__":
    main()
