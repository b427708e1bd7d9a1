"""Child process of the loop-back tests (tests/test_gpu_sharded.py, tests/test_gpu_p2p_skew.py): `world` engines in
one process on cuda:0, the peer-memory pipeline (gcra_p2p_*) between them, results against ONE oracle store fed the
union trace in global order (tick by tick, rank 0's rows first).

    p2p_loopback_worker.py WORLD TICK HOT [options]

WORLD TICK HOT alone is the original run: 6 pipelined ticks of config4 (40 K keys, `hot` hot keys), TICK rows per
rank.  The options pick a skewed scenario:
    --trace config4 | flood | flood_mix | fresh_to_owner
        flood           every row on key 0 (policy --flood-policy, quantity 1)
        flood_mix       half the rows on key 0, the other half uniform over the cold keys (1 .. n_keys-1) that have
                        key 0's owner: that owner receives the whole tick, with key 0 in every 256-row tile
        fresh_to_owner  tick 1: distinct new keys (policy P0, quantity 1), all owned by rank 0; every later tick:
                        the keys of tick 1 the engines did not refuse, each sent again by the same rank
    --ticks A,B,../C,D,..  rows per rank of each tick ('/' separates ticks, the last group repeats; 0 allowed)
    --n-ticks N   --tick-ms T1,T2,..  (tick clocks in ms after traces.T0; default t + 1)
    --max-batch N[,..]   --capacity N[,..]   (per engine, the last value repeats)
    --refusable   rows answered GCRA_INTERNAL are allowed (they must leave no trace: the oracle replays only the
                  others); without it every row must be bit-identical
Prints one JSON line with what the test checks beyond exactness (refused rows, error counters, table sizes, device
memory in use), then "loopback ok"."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
import throttlecrab_b200 as tc  # noqa: E402
import traces  # noqa: E402
from gpu_util import replay_skipping_refused  # noqa: E402
from throttlecrab_b200.sharded import connect_local  # noqa: E402

P0 = tuple(int(x) for x in traces.POLICIES[0])


def owners(key_ids, world):
    """gcra_owner_of of the engine key hash of every key id"""
    L = tc._native.lib()
    h = tc.hash_key_ids(np.asarray(key_ids, dtype=np.uint64))
    return np.fromiter((L.gcra_owner_of(int(x), world) for x in h), np.uint32, len(h))


def rows(key, now_ns, policy=None, quantity=1):
    """trace rows (key ids) with one clock, a fixed policy (default: traces' per-key policy) and quantity"""
    r = np.zeros(len(key), traces.REQ_DTYPE)
    r["key"] = key
    if policy is None:
        traces.fill_policy(r, (r["key"] % np.uint64(8)).astype(np.int64))
    else:
        r["max_burst"], r["count_per_period"], r["period"] = policy
    r["quantity"] = quantity
    r["now_ns"] = now_ns
    return r


def flood(n, now_ns, policy=P0):
    return rows(np.zeros(n, np.uint64), now_ns, policy)


def flood_mix(n, now_ns, cold_keys, tick_index, policy=P0):
    """half the rows (chosen at random) on key 0, the rest uniform over `cold_keys`"""
    u0, u1 = traces.stream(5, 0, n, tick_index * n), traces.stream(5, 1, n, tick_index * n)
    hot = traces.unit(u1) < 0.5
    r = rows(np.where(hot, np.uint64(0), cold_keys[(u0 % np.uint64(len(cold_keys))).astype(np.int64)]), now_ns)
    r["max_burst"][hot], r["count_per_period"][hot], r["period"][hot] = policy
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("world", type=int)
    ap.add_argument("tick", type=int)
    ap.add_argument("hot", type=int)
    ap.add_argument("--trace", default="config4", choices=["config4", "flood", "flood_mix", "fresh_to_owner"])
    ap.add_argument("--ticks", default=None)
    ap.add_argument("--n-ticks", type=int, default=6)
    ap.add_argument("--tick-ms", default=None)
    ap.add_argument("--n-keys", type=int, default=40_000)
    ap.add_argument("--max-batch", default=None)
    ap.add_argument("--capacity", default="4000000")
    ap.add_argument("--flood-policy", default="%d,%d,%d" % P0)
    ap.add_argument("--refusable", action="store_true")
    a = ap.parse_args()
    world, n_ticks = a.world, a.n_ticks

    def per_engine(s, default):
        v = [int(x) for x in s.split(",")] if s else [default]
        return [v[min(r, len(v) - 1)] for r in range(world)]
    groups = [[int(x) for x in g.split(",")] for g in a.ticks.split("/")] if a.ticks else [[a.tick]]
    sizes = [[g[min(r, len(g) - 1)] for r in range(world)] for g in
             (groups[min(t, len(groups) - 1)] for t in range(n_ticks))]
    cap = max(max(s) for s in sizes)
    max_batch = per_engine(a.max_batch, 4 * cap)
    capacity = per_engine(a.capacity, 4_000_000)
    tick_ms = [int(x) for x in a.tick_ms.split(",")] if a.tick_ms else [t + 1 for t in range(n_ticks)]
    assert len(tick_ms) == n_ticks
    policy = tuple(int(x) for x in a.flood_policy.split(","))

    dev = torch.device("cuda", 0)
    free0, total = torch.cuda.mem_get_info(dev)
    lims = [tc.RateLimiter(tc.ManualStore(capacity=capacity[r], device=0, created_ns=traces.T0, max_batch=max_batch[r]))
            for r in range(world)]
    connect_local(lims, cap)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)

    # the global trace of every tick: a list (one array per rank), None = built once the previous tick is known
    if a.trace == "config4":
        assert all(len(set(s)) == 1 for s in sizes), "config4 takes one tick size for every rank"
        g = traces.config4(n_keys=a.n_keys, n_ticks=n_ticks, tick_size=sizes[0][0] * world, hot=a.hot)
        per_tick = [np.split(g[t * sizes[0][0] * world:(t + 1) * sizes[0][0] * world], world) for t in range(n_ticks)]
    elif a.trace == "flood":
        per_tick = [[flood(n, traces.T0 + ms * 1_000_000, policy) for n in s] for s, ms in zip(sizes, tick_ms)]
    elif a.trace == "flood_mix":
        ids = np.arange(1, a.n_keys, dtype=np.uint64)
        cold = ids[owners(ids, world) == owners([0], world)[0]]
        per_tick = [[flood_mix(n, traces.T0 + ms * 1_000_000, cold, t * world + r, policy) for r, n in enumerate(s)]
                    for t, (s, ms) in enumerate(zip(sizes, tick_ms))]
    else:
        n_new = sum(sizes[0])
        ids = np.arange(1, 8 * n_new + 1, dtype=np.uint64)
        ids = ids[owners(ids, world) == 0][:n_new]
        assert len(ids) == n_new
        ofs = np.cumsum([0] + sizes[0])
        per_tick = [[rows(ids[ofs[r]:ofs[r + 1]], traces.T0 + tick_ms[0] * 1_000_000, P0) for r in range(world)]]
        per_tick += [None] * (n_ticks - 1)

    def device_rows(sl):
        e = np.empty(len(sl), tc.REQ_DTYPE)
        u, inv = np.unique(sl["key"], return_inverse=True)
        e["key_hash"] = tc.hash_key_ids(u)[inv]
        for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
            e[f] = sl[f]
        return torch.from_numpy(e.view(np.uint8)).to(dev)

    ress = [[None] * world for _ in range(n_ticks)]
    keep = []
    # config4 enqueues every tick at once (pipelined across ticks).  The other traces run tick by tick: every tick's
    # error count is known on its own, and every engine's host-side table-room bound starts each tick from the
    # real occupancy.  (Were it stale, an engine would synchronize the device before growing its table -- which,
    # with several engines in ONE process, waits for the ranks whose tick has not been submitted yet.)
    sync_each = a.trace != "config4"
    errors = []                      # engines' error counters before every tick (sync_each) and at the end
    peak_used = 0

    def join_all():
        for lim in lims:
            lim.store._check(lim._L.gcra_p2p_join(lim._h, stream.cuda_stream))
        torch.cuda.synchronize()

    for t in range(n_ticks):
        if per_tick[t] is None:
            # fresh_to_owner: every rank sends again the rows of tick 1 that were not refused
            join_all()
            per_tick[t] = []
            for r in range(world):
                sl = per_tick[0][r]
                got0 = ress[0][r].cpu().numpy().view(oracle.RES_DTYPE)[:len(sl)]
                sl = sl[got0["status"] != tc.INTERNAL].copy()
                sl["now_ns"] = traces.T0 + tick_ms[t] * 1_000_000
                per_tick[t].append(sl)
        if sync_each or t == 0:
            errors.append([lim.store.stats()["errors"] for lim in lims])
        for r in range(world):
            n = len(per_tick[t][r])
            q = device_rows(per_tick[t][r]) if n else torch.zeros(48, dtype=torch.uint8, device=dev)
            ress[t][r] = torch.zeros(max(n, 1) * 32, dtype=torch.uint8, device=dev)
            keep.append(q)
            lims[r].store._check(lims[r]._L.gcra_p2p_submit_route(lims[r]._h, n, q.data_ptr(), stream.cuda_stream))
        for r in range(world):        # every engine's route is enqueued before the first kernel that waits for it
            lims[r].store._check(lims[r]._L.gcra_p2p_submit_finish(lims[r]._h, ress[t][r].data_ptr()))
        if sync_each:
            join_all()
        peak_used = max(peak_used, total - torch.cuda.mem_get_info(dev)[0])
    join_all()
    peak_used = max(peak_used, total - torch.cuda.mem_get_info(dev)[0])
    for lim in lims:
        e = C.c_uint32()
        lim.store._check(lim._L.gcra_p2p_error(lim._h, C.byref(e)))
        assert e.value == 0, "a wait gave up"
    errors.append([lim.store.stats()["errors"] for lim in lims])

    st_o = oracle.OracleStore(oracle.PERIODIC, capacity=max(a.n_keys, 1000), created_ns=traces.T0, p0=10**9)
    report = {"rows": [], "refused": [], "refused_first": [], "refused_last": [],
              # per tick (sync_each) or for the whole run: how much each engine's error counter rose
              "errors_delta": [[e1 - e0 for e0, e1 in zip(errors[i], errors[i + 1])] for i in range(len(errors) - 1)]}
    n_allowed = n_denied = 0
    for t in range(n_ticks):
        glob = np.concatenate(per_tick[t])
        got = np.concatenate([ress[t][r].cpu().numpy().view(oracle.RES_DTYPE)[:len(per_tick[t][r])]
                              for r in range(world)])
        refused = replay_skipping_refused(st_o, glob, got, "tick %d: " % t)
        assert a.refusable or len(refused) == 0, "tick %d: %d rows refused, first %d: %s" % (
            t, len(refused), refused[0], glob[refused[0]])
        n_allowed += int(got["allowed"].sum())
        n_denied += int(((got["allowed"] == 0) & (got["status"] == tc.OK)).sum())
        report["rows"].append(len(glob))
        report["refused"].append(len(refused))
        report["refused_first"].append(int(refused[0]) if len(refused) else -1)
        report["refused_last"].append(int(refused[-1]) if len(refused) else -1)
    if a.trace == "config4":
        assert n_allowed > 0 and n_denied > 0
    report["len"] = [lim.store.len() for lim in lims]
    report["oracle_len"] = st_o.len()
    report["device_mem_used_gb"] = round(peak_used / 2**30, 2)
    report["device_mem_used_before_gb"] = round((total - free0) / 2**30, 2)
    print(json.dumps(report))
    for lim in lims:
        lim.store.close()
    print("loopback ok: %d rows, %d engines" % (sum(report["rows"]), world))


if __name__ == "__main__":
    main()
