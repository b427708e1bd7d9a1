"""Two real GPUs: the hash-sharded engine (partition kernel -> NCCL all-to-all -> decide -> all-to-all
-> unpermute, pipelined) must give exactly the answers of ONE oracle store fed the union trace in global
index order.  Skipped on boxes with fewer than 2 GPUs (run with `gpurun --gpus 2`)."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, n_keys, n_ticks, tick, ret, native=False):
    return _worker_impl(rank, world, port, n_keys, n_ticks, tick, ret, "native" if native else "torch")


def _worker_p2p(rank, world, port, n_keys, n_ticks, tick, ret, trace="config4"):
    return _worker_impl(rank, world, port, n_keys, n_ticks, tick, ret, "p2p", trace)


def _global_trace(trace, n_keys, n_ticks, tick, world):
    """the union trace of all ranks, tick by tick (rank r's rows of tick t: [(t world + r) tick, +tick))"""
    import traces
    if trace == "config4":
        return traces.config4(n_keys=n_keys, n_ticks=n_ticks, tick_size=tick * world, hot=20)
    # flood: every row on one key, ticks at T0, +1 ms, +1 s (tests/test_gpu_p2p_skew.py)
    import p2p_loopback_worker as w
    return np.concatenate([w.flood(tick * world, traces.T0 + ms * 1_000_000) for ms in (0, 1, 1000)[:n_ticks]])


def _worker_impl(rank, world, port, n_keys, n_ticks, tick, ret, kind, trace="config4"):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import throttlecrab_b200 as tc
    import traces
    from throttlecrab_b200.sharded import NativeShardedLimiter, PeerShardedLimiter, ShardedLimiter
    key_hash_of = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64))
    # (flood: table room for the 1.25 x tick rows an engine reserves per tick, so that no tick grows the table)
    lim = tc.RateLimiter(tc.ManualStore(capacity=n_keys if trace == "config4" else 6_000_000, device=rank,
                                        created_ns=traces.T0, max_batch=2 * tick))
    sh = {"native": NativeShardedLimiter, "torch": ShardedLimiter, "p2p": PeerShardedLimiter}[kind](lim, dist, dev)
    glob = _global_trace(trace, n_keys, n_ticks, tick, world)
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
        sh.submit(reqs[t], ress[t])            # pipelined across ticks
    sh.finish()
    torch.cuda.synchronize()
    if kind == "p2p":
        assert sh.error() == 0, "a peer-memory wait gave up"
    out = np.concatenate([r.cpu().numpy() for r in ress])
    if isinstance(ret, str):                  # large runs: through a file, not the manager's pipe
        np.save(os.path.join(ret, "rank%d.npy" % rank), out)
    else:
        ret[rank] = out.tobytes()
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("native", [False, True], ids=["torch_distributed", "native_nccl"])
def test_two_gpu_sharded_matches_single_oracle(native):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import oracle
    import traces
    world, n_keys, n_ticks, tick = 2, 50_000, 6, 1 << 16
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), n_keys, n_ticks, tick, ret, native), nprocs=world, join=True)
    glob = traces.config4(n_keys=n_keys, n_ticks=n_ticks, tick_size=tick * world, hot=20)
    want = oracle.OracleStore(oracle.PERIODIC, capacity=n_keys, created_ns=traces.T0, p0=10**9).replay(glob)
    got = np.empty(len(glob), oracle.RES_DTYPE)
    for r in range(world):
        pr = np.frombuffer(ret[r], oracle.RES_DTYPE).reshape(n_ticks, tick)
        for t in range(n_ticks):
            a = t * tick * world + r * tick
            got[a:a + tick] = pr[t]
    assert got.tobytes() == want.tobytes()


def _union_trace_check(ret, world, n_keys, n_ticks, tick, glob=None):
    import oracle
    import traces
    if glob is None:
        glob = _global_trace("config4", n_keys, n_ticks, tick, world)
    want = oracle.OracleStore(oracle.PERIODIC, capacity=n_keys, created_ns=traces.T0, p0=10**9).replay(glob)
    got = np.empty(len(glob), oracle.RES_DTYPE)
    for r in range(world):
        pr = np.frombuffer(ret[r], oracle.RES_DTYPE).reshape(n_ticks, tick)
        for t in range(n_ticks):
            a = t * tick * world + r * tick
            got[a:a + tick] = pr[t]
    bad = np.nonzero((got.view(np.uint8).reshape(len(got), -1) != want.view(np.uint8).reshape(len(want), -1)).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), int(bad[0]), want[bad[0]], got[bad[0]], glob[bad[0]])
    assert want["allowed"].sum() > 0 and (want["allowed"] == 0).sum() > 0


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("trace", ["config4", "flood"])
def test_two_gpu_peer_memory_matches_single_oracle(trace, tmp_path, k1_path):
    """gcra_p2p_*: rows stored straight into the owner's inbox over NVLink, results straight into the sender's
    outbox; two processes, CUDA IPC windows.  `flood`: 3 ticks of 2 x 2^22 rows on ONE key (fresh, saturated, 1 s
    later), so the owner's batch spans 32768 tiles, each holding the key 256 times (tests/test_gpu_p2p_skew.py)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    if trace == "flood" and k1_path != "auto":
        pytest.skip("a segmented tick takes the index-order pipeline whatever K1 path is forced")
    world, n_keys, n_ticks, tick = 2, 50_000, 6, 1 << 16
    if trace == "flood":
        n_keys, n_ticks, tick = 1, 3, 1 << 22
    mp.spawn(_worker_p2p, args=(world, _free_port(), n_keys, n_ticks, tick, str(tmp_path), trace), nprocs=world, join=True)
    ret = {r: np.load(str(tmp_path / ("rank%d.npy" % r))).tobytes() for r in range(world)}
    _union_trace_check(ret, world, n_keys, n_ticks, tick, _global_trace(trace, n_keys, n_ticks, tick, world))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("world,tick,hot", [(2, 1 << 15, 20), (4, 1 << 14, 3), (3, 5000, 50)])
def test_peer_memory_pipeline_loopback_on_one_gpu(world, tick, hot):
    """The same pipeline with `world` engines in ONE process on ONE GPU (windows exchanged as plain pointers): every
    kernel, flag and segment computation of gcra_p2p_* runs, only the stores do not cross NVLink.  Runs on the
    1-GPU boxes too.  Checked against ONE oracle store fed the union trace in global order (hot keys span all
    ranks; ragged tick sizes exercise partial tiles and empty segments).

    Runs in a child process with CUDA_DEVICE_MAX_CONNECTIONS=32: the engines' kernels wait for each other, so two
    engines of one process must not share a hardware work queue (a launch queued behind another engine's blocked
    stream would never start); one engine per process -- the product's configuration -- has no such coupling."""
    import subprocess
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "p2p_loopback_worker.py"), str(world), str(tick), str(hot)],
                         capture_output=True, text=True, timeout=500, env=env)
    assert out.returncode == 0 and "loopback ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
