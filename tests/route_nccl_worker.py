"""Child processes of tests/test_gpu_route_nccl.py: the two host-driven sharded ticks on ONE GPU.

    route_nccl_worker.py gloo  WORLD RANK PORT OUT_DIR PARENT_PID
        one rank of a `ShardedLimiter` over gloo (CUDA tensors, world 2-4, every rank's engine on cuda:0) with the
        real route kernels (the default CudaOps) and max_rows = the engine's max_batch = GLOO_MAX_ROWS
    route_nccl_worker.py nccl1 PORT OUT_DIR PARENT_PID
        the native NCCL tick (gcra_shard_*, through make_sharded with GCRA_SHARD=nccl) over a single-rank NCCL group,
        then the same ticks through a ShardedLimiter over that group

Every rank submits the 9 ticks of `gloo_ticks` / `nccl1_ticks` back to back with denied-key tracking on, joins, and
writes what the test checks into OUT_DIR: its results (`<run>_rank<r>.npy`, the ticks' result rows in order) and a
JSON report (`<run>_rank<r>.json`: the collective top_denied, its own engine's list, the engine's counters).  The
checks against the oracle are the test's; this file only drives the pipelines and asserts the refusals it provokes.
The trace builders are shared with the test, which replays the same ticks through ONE oracle store.

The process gets SIGKILL when its parent (PARENT_PID, the test) dies, so that a rank waiting for a peer in a
collective never outlives the test that started it."""
import ctypes
import json
import os
import signal
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
import traces  # noqa: E402

N_KEYS, HOT = 20_000, 20
N_TICKS = 9                     # more than twice the pipelines' 4 buffer slots: every slot is reused
GLOO_MAX_ROWS = 3000            # not a multiple of 256: every full slice ends in a partial tile
FLOOD_TICK = 5                  # the gloo tick in which one owner receives 1.25 x max_rows rows
NCCL1_MAX_ROWS = 6000
TOP_ALL = 1 << 15               # > N_KEYS: every denied key


def mix64(x):
    """gcra_device.cuh mix64 (the splitmix64 finaliser), in numpy uint64"""
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(30))
        x = x * np.uint64(0xBF58476D1CE4E5B9)
        x = x ^ (x >> np.uint64(27))
        x = x * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return x


def owner_of(key_hash, n_shards):
    """gcra_owner_of restated: the high word of mix64(h ^ 0xA24BAED4963EE407), scaled to n_shards"""
    m = mix64(np.asarray(key_hash, np.uint64) ^ np.uint64(0xA24BAED4963EE407))
    return (((m >> np.uint64(32)) * np.uint64(n_shards)) >> np.uint64(32)).astype(np.int64)


def hot_keys():
    return traces.rank_to_key(np.arange(HOT, dtype=np.uint64), N_KEYS)


def _ticks(sizes, flood_owner=None, world=1):
    """config4 rows cut into ticks of sizes[t][r] rows (rank r's slice of tick t; 1 ms per tick).  In FLOOD_TICK every
    row is moved onto the hot keys that `flood_owner` owns among `world` shards."""
    width = max(sum(s) for s in sizes)
    g = traces.config4(n_keys=N_KEYS, n_ticks=len(sizes), tick_size=width, hot=HOT)
    out = []
    for t, s in enumerate(sizes):
        tick = g[t * width:t * width + sum(s)].copy()
        if flood_owner is not None and t == FLOOD_TICK:
            hot = hot_keys()
            mine = hot[owner_of(tc.hash_key_ids(hot), world) == flood_owner]
            tick["key"] = mine[(traces.stream(9, t, len(tick)) % np.uint64(len(mine))).astype(np.int64)]
            traces.fill_policy(tick, (tick["key"] % np.uint64(8)).astype(np.int64))
        out.append(np.split(tick, np.cumsum(s)[:-1]))
    return out


def gloo_sizes(world, m=GLOO_MAX_ROWS):
    """ragged slices: rank world-1 empty in tick 2, rank 0 at exactly max_rows in tick 3 and rank world-1 in tick 7;
    in FLOOD_TICK the ranks together send 1.25 x max_rows rows (no rank more than max_rows)"""
    sizes = [[(m // 3 + 977 * (t + 1) * (r + 1)) % m + 1 for r in range(world)] for t in range(N_TICKS)]
    sizes[2][world - 1] = 0
    sizes[3][0] = m
    sizes[7][world - 1] = m
    total = m + m // 4
    sizes[FLOOD_TICK] = [total // world + (total % world if r == 0 else 0) for r in range(world)]
    return sizes


def gloo_ticks(world):
    """the gloo trace: ticks[t][r] = trace rows (key ids) of rank r in tick t.  The hot keys span every rank, and
    FLOOD_TICK sends every row to the hot keys of the last rank."""
    own = owner_of(tc.hash_key_ids(hot_keys()), world)
    assert set(own.tolist()) == set(range(world)), "the hot keys do not span every rank"
    return _ticks(gloo_sizes(world), flood_owner=world - 1, world=world)


# the 0-row tick is the fifth: its buffer slot still holds the counts of the first tick
NCCL1_SIZES = [4097, NCCL1_MAX_ROWS, 255, 1, 0, 256, NCCL1_MAX_ROWS, 1, 4097]


def nccl1_ticks():
    return _ticks([[n] for n in NCCL1_SIZES])


def engine_rows(sl):
    e = np.zeros(len(sl), tc.REQ_DTYPE)
    if len(sl):
        e["key_hash"] = tc.hash_key_ids(sl["key"])
        for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
            e[f] = sl[f]
    return e


def _expect_internal(fn, what):
    try:
        fn()
    except tc.Internal:
        return
    raise AssertionError("%s was not refused" % what)


def drive(sh, lim, mine, dev, out_dir, name, on_first=None, before_finish=None):
    """Submit rank `sh.rank`'s slices `mine` back to back (one tick each), join, and write the results and report."""
    sh.track_denied(1 << 20)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    reqs = [torch.from_numpy(engine_rows(sl).view(np.uint8)).to(dev) for sl in mine]
    ress = [torch.full((len(sl) * 32,), 0xA5, dtype=torch.uint8, device=dev) for sl in mine]
    report = {}
    for t in range(len(mine)):
        sh.submit(reqs[t], ress[t])
        if t == 0 and on_first is not None:
            on_first()
    if before_finish is not None:
        report.update(before_finish(ress))
    sh.finish()
    torch.cuda.synchronize()
    out = np.concatenate([r.cpu().numpy() for r in ress])
    top, dropped = sh.top_denied(TOP_ALL)                 # collective
    own, own_dropped = lim.store.top_denied(TOP_ALL)
    st = lim.store.stats()
    report.update(top=top, dropped=dropped, own=own, own_dropped=own_dropped,
                  allowed=st["allowed"], denied=st["denied"], errors=st["errors"])
    np.save(os.path.join(out_dir, "%s_rank%d.npy" % (name, sh.rank)), out)
    with open(os.path.join(out_dir, "%s_rank%d.json" % (name, sh.rank)), "w") as f:
        json.dump(report, f)


def run_gloo(world, rank, port, out_dir):
    import torch.distributed as dist
    from throttlecrab_b200.sharded import CudaOps, ShardedLimiter
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ticks = gloo_ticks(world)
    lim = tc.RateLimiter(tc.ManualStore(capacity=N_KEYS, device=0, created_ns=traces.T0, max_batch=GLOO_MAX_ROWS))
    sh = ShardedLimiter(lim, dist, dev)
    assert type(sh.ops) is CudaOps and sh.max_rows == GLOO_MAX_ROWS and sh.cuda
    drive(sh, lim, [t[rank] for t in ticks], dev, out_dir, "gloo")
    dist.barrier()
    dist.destroy_process_group()
    lim.store.close()


def run_nccl1(port, out_dir):
    import torch.distributed as dist
    from throttlecrab_b200.sharded import NativeShardedLimiter, ShardedLimiter, make_sharded
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), GCRA_SHARD="nccl")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev)
    mine = [t[0] for t in nccl1_ticks()]

    lim = tc.RateLimiter(tc.ManualStore(capacity=N_KEYS, device=0, created_ns=traces.T0, max_batch=NCCL1_MAX_ROWS))
    sh = make_sharded(lim, dist, dev)
    assert isinstance(sh, NativeShardedLimiter), type(sh)
    assert sh.max_rows == NCCL1_MAX_ROWS
    L, h = lim._L, lim._h
    _expect_internal(lambda: lim.store._check(L.gcra_shard_init(h, 0, 1, bytes(384), NCCL1_MAX_ROWS)),
                     "a second gcra_shard_init")
    reader = torch.cuda.Stream(dev)
    _expect_internal(lambda: sh.wait_tick(0, reader), "wait_tick(0) before any tick")

    def on_first():
        _expect_internal(lambda: sh.wait_tick(1, reader), "wait_tick(1) after one tick")

    def before_finish(ress):
        """every tick is submitted: wait for the last three on `reader`, one at a time, and read each there"""
        _expect_internal(lambda: sh.wait_tick(3, reader), "wait_tick(3)")
        _expect_internal(lambda: sh.wait_tick(N_TICKS, reader), "wait_tick past the submitted ticks")
        early = {}
        for back in (0, 1, 2):
            t = N_TICKS - 1 - back
            sh.wait_tick(back, reader)
            with torch.cuda.stream(reader):
                early[t] = ress[t].cpu().numpy().tobytes().hex()
        return {"early": early}
    drive(sh, lim, mine, dev, out_dir, "native", on_first, before_finish)
    lim.store.close()

    lim2 = tc.RateLimiter(tc.ManualStore(capacity=N_KEYS, device=0, created_ns=traces.T0, max_batch=NCCL1_MAX_ROWS))
    drive(ShardedLimiter(lim2, dist, dev), lim2, mine, dev, out_dir, "torch_nccl")
    lim2.store.close()
    dist.destroy_process_group()


def die_with_parent(parent_pid):
    """PR_SET_PDEATHSIG: SIGKILL this process once the parent that started it exits"""
    libc = ctypes.CDLL(None, use_errno=True)
    if libc.prctl(1, signal.SIGKILL, 0, 0, 0) != 0:
        raise OSError(ctypes.get_errno(), "prctl(PR_SET_PDEATHSIG)")
    if os.getppid() != parent_pid:            # the parent exited before the signal was armed
        raise SystemExit("the test that started this process is gone")


def main():
    a = sys.argv[1:]
    die_with_parent(int(a[-1]))
    if a[0] == "gloo":
        run_gloo(int(a[1]), int(a[2]), int(a[3]), a[4])
    elif a[0] == "nccl1":
        run_nccl1(int(a[1]), a[2])
    else:
        raise SystemExit("unknown run %r" % a[0])
    print("route worker ok")


if __name__ == "__main__":
    main()
