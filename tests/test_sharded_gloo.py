"""World-size-2 (gloo, CPU) test of the multi-GPU host logic in throttlecrab_b200/sharded.py:
count exchange, variable-size all-to-all, result return and inverse permutation, and the global
ordering rule.  The three DEVICE steps (partition / decide / unpermute) are CUDA-only in the
product; here they are replaced by numpy stand-ins defined in THIS test (the decide stand-in is the
CPU oracle, used as the checker's engine), so only the routing logic around them is under test.  The real kernels
under the same host logic (ShardedLimiter over gloo with CUDA tensors, worlds 2-4 on one GPU) are tested in
test_gpu_route_nccl.py."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class NumpyOps:
    """CPU stand-ins with the contracts of gcra_route_partition / _batch_device / _unpermute."""

    def __init__(self, world, oracle_store, owner_fn):
        self.world, self.store, self.owner_fn = world, oracle_store, owner_fn

    def partition(self, n, req, world, routed, src_index, counts, stream):
        import throttlecrab_b200 as tc
        rows = req.numpy()[:n * 48].view(tc.REQ_DTYPE)
        own = self.owner_fn(rows["key_hash"])
        order = np.argsort(own, kind="stable")
        routed.numpy()[:n * 48] = rows[order].view(np.uint8)
        src_index.numpy()[:n] = order.astype(np.int32)
        counts.numpy()[:world] = np.bincount(own, minlength=world).astype(np.int32)

    def decide(self, n, req, res, stream):
        import oracle
        rows = req.numpy()[:n * 48].view(oracle.REQ_DTYPE)      # key column = key id in this test
        res.numpy()[:n * 32] = self.store.replay(rows).view(np.uint8)

    def unpermute(self, n, routed_res, src_index, res, stream):
        import oracle
        r = routed_res.numpy()[:n * 32].view(oracle.RES_DTYPE)
        out = np.empty(n, oracle.RES_DTYPE)
        out[src_index.numpy()[:n]] = r
        res.numpy()[:n * 32] = out.view(np.uint8)


def _worker(rank, world, port, n_ticks, tick, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import oracle
    import traces
    from throttlecrab_b200.sharded import ShardedLimiter

    class _Lim:           # ShardedLimiter only needs .store.max_batch when ops are injected
        class store:
            max_batch = 4 * tick

    def owner(key):       # any deterministic key -> shard map; the product uses gcra_owner_of
        return (traces.splitmix64(key) % np.uint64(world)).astype(np.int64)

    st = oracle.OracleStore(oracle.PERIODIC, capacity=10_000, created_ns=traces.T0, p0=10**9)
    sh = ShardedLimiter(_Lim, dist, torch.device("cpu"), ops=NumpyOps(world, st, owner))
    glob = traces.config4(n_keys=5_000, n_ticks=n_ticks, tick_size=tick * world, hot=20)
    out = []
    for t in range(n_ticks):
        sl = glob[t * tick * world:(t + 1) * tick * world][rank * tick:(rank + 1) * tick]
        req = torch.from_numpy(np.ascontiguousarray(sl).view(np.uint8).copy())
        res = torch.empty(tick * 32, dtype=torch.uint8)
        sh.step(req, res)
        out.append(res.numpy().view(oracle.RES_DTYPE).copy())
    ret[rank] = np.concatenate(out).tobytes()
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_routing_preserves_global_order():
    import oracle
    import traces
    world, n_ticks, tick = 2, 5, 3000
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), n_ticks, tick, ret), nprocs=world, join=True)
    # single-store replay of the union trace in global index order
    glob = traces.config4(n_keys=5_000, n_ticks=n_ticks, tick_size=tick * world, hot=20)
    want = oracle.OracleStore(oracle.PERIODIC, capacity=10_000, created_ns=traces.T0, p0=10**9).replay(glob)
    got = np.empty(len(glob), oracle.RES_DTYPE)
    per_rank = {r: np.frombuffer(ret[r], oracle.RES_DTYPE).reshape(n_ticks, tick) for r in range(world)}
    for t in range(n_ticks):
        for r in range(world):
            a = t * tick * world + r * tick
            got[a:a + tick] = per_rank[r][t]
    assert got.tobytes() == want.tobytes()
    assert want["allowed"].sum() > 0 and (want["allowed"] == 0).sum() > 0
