"""Child process of tests/test_gpu_failed_calls.py for the scenarios with a peer-memory loop-back (several engines in
one process on cuda:0: run with CUDA_DEVICE_MAX_CONNECTIONS=32, see p2p_loopback_worker.py).

    failed_calls_worker.py p2p        a peer-memory window no H100 can hold, then the same engine: index-order batches
                                      and a 2-engine loop-back tick
    failed_calls_worker.py lifecycle  20 rounds of engines that use every feature, then destroyed

Every result is checked against the oracle; prints "<scenario> ok" at the end."""
import ctypes as C
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
import throttlecrab_b200 as tc  # noqa: E402
import traces  # noqa: E402
from gpu_util import engine_requests, first_mismatch  # noqa: E402
from p2p_loopback_worker import rows  # noqa: E402
from throttlecrab_b200.sharded import connect_local  # noqa: E402

DEV = torch.device("cuda", 0)
NOW = traces.T0 + 1_000_000


def oracle_store(capacity=1000):
    return oracle.OracleStore(oracle.PERIODIC, capacity=capacity, created_ns=traces.T0, p0=10**9)


def exact(want, got, req, what):
    bad = first_mismatch(want, got, req)
    assert bad is None, what + ": " + bad


def engine(capacity, max_batch, flags=0):
    return tc.RateLimiter(tc.ManualStore(capacity=capacity, created_ns=traces.T0, max_batch=max_batch, flags=flags))


def loopback_tick(lims, per_rank, stream):
    """one peer-memory tick: rank r submits per_rank[r] (trace rows); its results, in its input order"""
    keep, outs = [], []
    for lim, r in zip(lims, per_rank):
        q = torch.from_numpy(engine_requests(r).view(np.uint8)).to(DEV)
        outs.append(torch.zeros(len(r) * 32, dtype=torch.uint8, device=DEV))
        keep.append(q)
        lim.store._check(lim._L.gcra_p2p_submit_route(lim._h, len(r), q.data_ptr(), stream.cuda_stream))
    for lim, out in zip(lims, outs):
        lim.store._check(lim._L.gcra_p2p_submit_finish(lim._h, out.data_ptr()))
    for lim in lims:
        lim.store._check(lim._L.gcra_p2p_join(lim._h, stream.cuda_stream))
        e = C.c_uint32()
        lim.store._check(lim._L.gcra_p2p_error(lim._h, C.byref(e)))
        assert e.value == 0, "a wait gave up"
    torch.cuda.synchronize()
    return [o.cpu().numpy().view(tc.RES_DTYPE) for o in outs]


def check_tick(lims, key0, n, stream):
    """a loop-back tick of n fresh keys per rank (ids from key0), bit-identical to one oracle over the union trace"""
    per_rank = [rows(np.uint64(key0) + (np.arange(n, dtype=np.uint64) * np.uint64(7) + np.uint64(r)) % np.uint64(3000), NOW)
                for r in range(len(lims))]
    got = loopback_tick(lims, per_rank, stream)
    glob = np.concatenate(per_rank)
    exact(oracle_store().replay(glob), np.concatenate(got), glob, "loop-back tick")


def p2p():
    stream = torch.cuda.Stream(DEV)
    torch.cuda.set_stream(stream)
    B = 1 << 15
    lim = engine(200_000, B)
    L, h = lim._L, lim._h
    # 4 inbox slots x 16 senders x 2^24 rows x 80 bytes = 80 GiB of window: more than an 80 GB H100 has
    total = torch.cuda.get_device_properties(DEV).total_memory
    world, cap = 16, 1 << 24
    assert 4 * world * cap * 80 > total, "a card this large needs a larger request"
    w = C.c_void_p()
    assert L.gcra_p2p_prepare(h, 0, world, cap, None, C.byref(w)) != tc.OK
    assert "out of memory" in L.gcra_last_error(h).decode()
    # the same engine: index-order batches (in the engine's own choice of pipeline: batches of 2^15 rows)
    req = traces.config4(n_keys=40_000, n_ticks=4, tick_size=B, hot=50)
    ereq = engine_requests(req)
    res = np.empty(len(req), tc.RES_DTYPE)
    for a in range(0, len(req), B):
        lim.rate_limit_batch(ereq[a:a + B], out=res[a:a + B])
    exact(oracle_store(40_000).replay(req), res, req, "batches after the failed prepare")
    if os.environ.get("GCRA_INDEX_MIN") != "0":
        assert lim.store.stats()["index_batches"] >= 1
    # ... and a loop-back tick with a second engine: 2 x 2^15 row ids per inbox slot, more than max_batch, so the
    # engines' index-order buffers are made anew
    lims = [lim, engine(200_000, B)]
    connect_local(lims, B)
    check_tick(lims, 1_000_000, 1 << 14, stream)
    for x in lims:
        x.store.close()


def compact(trace_rows):
    r16 = np.zeros(len(trace_rows), tc.REQ16_DTYPE)
    r16["key_hash"] = tc.hash_key_ids(trace_rows["key"])
    r16["quantity"] = trace_rows["quantity"]
    r16["policy"] = trace_rows["key"] % np.uint64(8)
    return r16


def lifecycle(rounds=20):
    stream = torch.cuda.Stream(DEV)
    torch.cuda.set_stream(stream)
    pol = np.zeros(len(traces.POLICIES), tc.POLICY_DTYPE)
    pol["max_burst"], pol["count_per_period"], pol["period"] = traces.POLICIES.T
    T = 4096
    path = os.path.join(tempfile.mkdtemp(), "snap.bin")
    for i in range(rounds):
        # engine 0 starts with a table of 64 slots and grows; every engine gets its own keys
        lims = [engine(64, T, tc._native.FLAG_TIGHT_TABLE), engine(1000, T), engine(1000, T)]
        stores = [oracle_store() for _ in lims]
        for m, lim in enumerate(lims):
            lim.set_policies(pol)
            lim.store.track_denied(50)
            ring = tc.Ring(lim, slots=2, slot_capacity=T, compact=[False, True, 2][m])
            r = rows(np.uint64(m * 100_000) + np.arange(T, dtype=np.uint64) % np.uint64(300), NOW)
            ring.req[0][:] = engine_requests(r) if m == 0 else compact(r)
            ring.submit(0, T, NOW)
            ring.wait(0)
            got = ring.res[0] if m < 2 else tc.expand_results16(ring.req[0], NOW, pol, ring.res[0])
            exact(stores[m].replay(r), got, r, "round %d, ring mode %d" % (i, m))
            top, dropped = lim.store.top_denied(50)
            assert top and dropped == 0
        # a peer-memory tick between engines 0 and 1 (keys of their own)
        connect_local(lims[:2], T)
        check_tick(lims[:2], 1_000_000, 2048, stream)
        # growth of the tight table: new keys on engine 0
        r = rows(np.arange(20_000, 20_000 + T, dtype=np.uint64), NOW)
        exact(stores[0].replay(r), lims[0].rate_limit_batch(engine_requests(r)), r, "round %d, growth" % i)
        assert lims[0].store.stats()["grows"] >= 1
        # snapshot of engine 0 into engine 2
        lims[0].store.save(path)
        restored, conflicts = lims[2].store.restore(path)
        assert restored == lims[0].store.len() and conflicts == 0
        for lim in lims:
            lim.store.close()
    os.remove(path)


if __name__ == "__main__":
    {"p2p": p2p, "lifecycle": lifecycle}[sys.argv[1]]()
    print(sys.argv[1] + " ok")
