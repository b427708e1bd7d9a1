"""Top denied keys on the multi-GPU pipelines: every pipeline counts a denied request on the engine that owns its key,
so the ranks' lists are disjoint and the global top k is the top k of their concatenated lists.

The peer-memory scenarios run tests/p2p_denied_worker.py in a child process with CUDA_DEVICE_MAX_CONNECTIONS=32 (see
test_gpu_sharded.test_peer_memory_pipeline_loopback_on_one_gpu): `world` engines in one process on one GPU.  A
segmented tick always takes the index-order pipeline, so the K1 pipeline is pinned to the engine's own choice.  The
last test runs the three sharded pipelines on two GPUs."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu


def run_worker(*args, timeout=1500):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "p2p_denied_worker.py")] + [str(a) for a in args],
                         capture_output=True, text=True, timeout=timeout, env=env)
    assert out.returncode == 0 and "denied ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    report = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])
    print(report)
    return report


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("world", [2, 3, 4])
def test_counts_on_the_owner_are_exact(world, k1_path):
    """config4 (hot keys on every rank), ragged ticks, one empty rank in one tick: each rank's whole list equals the
    host count of the union results' denied rows it owns, the lists are disjoint, nothing is dropped, a rank's
    counts add up to its denied total, and merge_top_denied gives the host's global top k (k through ties too)."""
    rep = run_worker("exact", world)
    assert all(k > 0 for k in rep["keys"]) and all(d > 0 for d in rep["denied"])
    assert len(rep["rows"]) == 6 and len(set(rep["rows"])) > 1


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_flood_counts_on_the_keys_owner(k1_path):
    """2 x 2^22 rows on one key per tick (fresh, saturated, 1 s later): the whole count lands on the owner."""
    rep = run_worker("flood", 2)
    assert rep["rows"] == [2 << 22] * 3
    assert rep["denied"] > 2 << 22         # (the saturated tick alone is almost all denied)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("scenario", ["residue", "table_full"])
def test_refused_rows_are_not_counted(scenario, k1_path):
    """Rows answered GCRA_INTERNAL (a residue beyond max_batch, a table full inside a tick) are in no count, while
    the denied rows around them are counted exactly."""
    rep = run_worker(scenario, 4)
    assert rep["refused"] > 0 and rep["denied"] > 0 and rep["allowed"] > 0


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_off_launches_nothing_and_on_changes_no_result(k1_path):
    """The same ticks three times: tracking off, on, and switched on after tick 3.  Results are byte-identical (in the
    worker); tracking adds exactly one launch per tick and engine, and only while it is on."""
    rep = run_worker("off_on", 3)
    off, on, later = (np.array(rep["launches"][m]) for m in ("off", "on", "later"))
    assert (off > 0).all()
    assert (on == off + 1).all()
    assert (later[:3] == off[:3]).all() and (later[3:] == off[3:] + 1).all()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_pruning_is_per_rank(k1_path):
    """max_keys 64: the rank holding 320 denied keys is pruned to its top 64 by its query, the one holding 128 is not;
    a later tick adds to the pruned table as the host model predicts."""
    rep = run_worker("prune", 2)
    assert rep["keys_before"] == [320, 128]
    assert rep["keys_after"][0] == 64 and rep["keys_after"][1] == 128


# ---------------------------------------------------------------------------------------------- two GPUs
def _worker(rank, world, port, kind, n_keys, n_ticks, tick, ks, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import throttlecrab_b200 as tc
    import traces
    from throttlecrab_b200.sharded import NativeShardedLimiter, PeerShardedLimiter, ShardedLimiter
    key_hash_of = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64))
    lim = tc.RateLimiter(tc.ManualStore(capacity=n_keys, device=rank, created_ns=traces.T0, max_batch=2 * tick))
    sh = {"native": NativeShardedLimiter, "torch": ShardedLimiter, "p2p": PeerShardedLimiter}[kind](lim, dist, dev)
    sh.track_denied(1 << 20)
    glob = traces.config4(n_keys=n_keys, n_ticks=n_ticks, tick_size=tick * world, hot=20)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    reqs, ress = [], []
    for t in range(n_ticks):
        sl = glob[t * tick * world:(t + 1) * tick * world][rank * tick:(rank + 1) * tick]
        e = np.empty(tick, tc.REQ_DTYPE)
        e["key_hash"] = key_hash_of[sl["key"].astype(np.int64)]
        for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
            e[f] = sl[f]
        reqs.append(torch.from_numpy(e.view(np.uint8)).to(dev))
        ress.append(torch.empty(tick * 32, dtype=torch.uint8, device=dev))
    for t in range(n_ticks):
        sh.submit(reqs[t], ress[t])
    got = {str(k): sh.top_denied(k) for k in ks}          # collective: joins every tick first
    with open(os.path.join(out_dir, "%s_rank%d.json" % (kind, rank)), "w") as f:
        json.dump(got, f)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(900)
def test_two_gpu_pipelines_agree_on_the_global_top_k(tmp_path):
    """PeerShardedLimiter, NativeShardedLimiter and ShardedLimiter on the same config4 union trace: their collective
    top_denied(k) lists are identical on every rank and equal the host's global top k of the oracle's results."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import collections

    import oracle
    import throttlecrab_b200 as tc
    import traces
    from test_gpu_sharded import _free_port
    world, n_keys, n_ticks, tick = 2, 50_000, 6, 1 << 16
    glob = traces.config4(n_keys=n_keys, n_ticks=n_ticks, tick_size=tick * world, hot=20)
    want = oracle.OracleStore(oracle.PERIODIC, capacity=n_keys, created_ns=traces.T0, p0=10**9).replay(glob)
    d = (want["status"] == tc.OK) & (want["allowed"] == 0)
    cnt = collections.Counter(tc.hash_key_ids(glob["key"][d]).tolist())
    host = sorted(((int(h), int(c)) for h, c in cnt.items()), key=lambda hc: (-hc[1], hc[0]))
    counts = [c for _, c in host]
    tie = next(i for i in range(1, len(counts)) if counts[i] == counts[i - 1])
    ks = sorted({1, 10, tie, 1000, len(host) + 3})
    for kind in ("p2p", "native", "torch"):
        mp.spawn(_worker, args=(world, _free_port(), kind, n_keys, n_ticks, tick, ks, str(tmp_path)), nprocs=world, join=True)
    for kind in ("p2p", "native", "torch"):
        for r in range(world):
            got = json.load(open(str(tmp_path / ("%s_rank%d.json" % (kind, r)))))
            for k in ks:
                lst, dropped = got[str(k)]
                assert dropped == 0
                assert [tuple(x) for x in lst] == host[:k], (kind, r, k)
