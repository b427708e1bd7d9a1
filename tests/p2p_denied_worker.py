"""Child process of tests/test_gpu_sharded_denied.py: `world` engines in one process on cuda:0, the peer-memory
pipeline (gcra_p2p_*) between them, top-denied tracking (gcra_track_denied / gcra_top_denied) on the engines.  Every
rank's list is checked against a host count of the denied rows (status GCRA_OK, allowed 0) of the union trace's
results, restricted to the keys that rank owns (gcra_owner_of).

    p2p_denied_worker.py SCENARIO WORLD

    exact       config4 (hot keys span every rank), ragged tick sizes, one rank empty in one tick, ticks pipelined:
                per-rank lists exact and disjoint, nothing dropped, a rank's counts sum to its denied total, and
                merge_top_denied of the ranks' lists is the host's global top k
    flood       3 ticks of world x 2^22 rows on one key (fresh, saturated, 1 s later): every count on the owner
    residue     4 ranks x 2^16 rows on one fresh key, max_batch 2^16: the residue beyond max_batch is refused
                (GCRA_INTERNAL), the rows before it are allowed up to the burst, then denied
    table_full  rank 0 empty with room for about 1 K keys, ranks 1-3 send 2^13 new keys of rank 0, 6 rows each
                (burst 3): rows of keys that found no slot are refused, the others allowed or denied
    off_on      the same seeded ticks with tracking never on, on from the start, and switched on after tick 3
    prune       small max_keys: a query prunes the rank that holds more than 3 x max_keys keys to its top max_keys
Prints one JSON report line, then "denied ok"."""
import argparse
import collections
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
from p2p_loopback_worker import flood, owners, rows  # noqa: E402
from throttlecrab_b200.sharded import connect_local, merge_top_denied  # noqa: E402

P4 = tuple(int(x) for x in traces.POLICIES[4])          # burst 3
ALL = 1 << 17                                            # "every key" for top_denied


def owner_of_hash(hashes, world):
    L = tc._native.lib()
    return {int(h): int(L.gcra_owner_of(int(h), world)) for h in np.unique(np.asarray(hashes, np.uint64))}


class Run:
    """`world` engines, connected, and the ticks submitted to them so far (trace rows and results, per tick and rank)"""

    def __init__(self, world, cap, max_batch=None, capacity=4_000_000):
        def per_engine(v):
            return v if isinstance(v, (list, tuple)) else [v] * world
        self.world, self.dev = world, torch.device("cuda", 0)
        max_batch, capacity = per_engine(max_batch or 4 * cap), per_engine(capacity)
        self.lims = [tc.RateLimiter(tc.ManualStore(capacity=capacity[r], device=0, created_ns=traces.T0,
                                                   max_batch=max_batch[r])) for r in range(world)]
        connect_local(self.lims, cap)
        self.stream = torch.cuda.Stream(self.dev)
        torch.cuda.set_stream(self.stream)
        self.ticks, self.ress, self.launches, self.keep = [], [], [], []

    def join(self):
        for lim in self.lims:
            lim.store._check(lim._L.gcra_p2p_join(lim._h, self.stream.cuda_stream))
        torch.cuda.synchronize()

    def submit(self, per_rank):
        """one tick: per_rank[r] = trace rows (key ids) rank r submits.  Only enqueues."""
        before = [lim.store.launch_count() for lim in self.lims]
        ress = []
        for r, lim in enumerate(self.lims):
            sl = per_rank[r]
            n = len(sl)
            e = np.zeros(max(n, 1), tc.REQ_DTYPE)
            if n:
                e["key_hash"] = tc.hash_key_ids(sl["key"])
                for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
                    e[f] = sl[f]
            q = torch.from_numpy(e.view(np.uint8)).to(self.dev)
            ress.append(torch.zeros(max(n, 1) * 32, dtype=torch.uint8, device=self.dev))
            self.keep.append(q)
            lim.store._check(lim._L.gcra_p2p_submit_route(lim._h, n, q.data_ptr(), self.stream.cuda_stream))
        for r, lim in enumerate(self.lims):     # every route is enqueued before the first kernel that waits for it
            lim.store._check(lim._L.gcra_p2p_submit_finish(lim._h, ress[r].data_ptr()))
        self.launches.append([lim.store.launch_count() - b for lim, b in zip(self.lims, before)])
        self.ticks.append(per_rank)
        self.ress.append(ress)

    def finish(self):
        """join, check no wait gave up, and the union results of every tick submitted since the last finish (global
        order: rank 0's rows first)"""
        self.join()
        for lim in self.lims:
            e = C.c_uint32()
            lim.store._check(lim._L.gcra_p2p_error(lim._h, C.byref(e)))
            assert e.value == 0, "a wait gave up"
        out = []
        for per_rank, ress in zip(self.ticks, self.ress):
            glob = np.concatenate(per_rank)
            got = np.concatenate([ress[r].cpu().numpy().view(oracle.RES_DTYPE)[:len(per_rank[r])]
                                  for r in range(self.world)])
            out.append((glob, got))
        self.ticks, self.ress, self.keep = [], [], []
        return out

    def close(self):
        for lim in self.lims:
            lim.store.close()


def host_counts(ticks, world):
    """{rank: {key_hash: denied rows}} over (trace rows, results) pairs; denied = status OK and allowed 0"""
    per = {r: collections.Counter() for r in range(world)}
    for glob, got in ticks:
        d = (got["status"] == tc.OK) & (got["allowed"] == 0)
        if not d.any():
            continue
        u, c = np.unique(tc.hash_key_ids(glob["key"][d]), return_counts=True)
        own = owner_of_hash(u, world)
        for h, n in zip(u.tolist(), c.tolist()):
            per[own[h]][h] += n
    return per


def ordered(counter):
    return sorted(((int(h), int(c)) for h, c in counter.items()), key=lambda hc: (-hc[1], hc[0]))


def check_exact(run, ticks, what, stats0=None):
    """every rank's whole list against the host count of `ticks`; returns the host counts"""
    host = host_counts(ticks, run.world)
    seen = set()
    for r, lim in enumerate(run.lims):
        got, dropped = lim.store.top_denied(ALL)
        want = ordered(host[r])
        assert dropped == 0, "%s: rank %d dropped %d" % (what, r, dropped)
        assert got == want, "%s: rank %d: %d keys counted, host %d; first difference %s" % (
            what, r, len(got), len(want), next(((a, b) for a, b in zip(got, want) if a != b), None))
        keys = {h for h, _ in got}
        assert not keys & seen, "%s: rank %d shares keys with another rank" % (what, r)
        seen |= keys
        if stats0 is not None:
            assert sum(c for _, c in got) == lim.store.stats()["denied"] - stats0[r], "%s: rank %d: counts vs stats" % (what, r)
    return host


def ragged_config4(world, n_ticks, hot, n_keys=40_000):
    """config4 ticks split raggedly between the ranks; in tick 2 rank world-1 submits nothing"""
    sizes = [[1000 + 3 * (t + 1) * (r + 1) * 517 % 9000 for r in range(world)] for t in range(n_ticks)]
    sizes[2][world - 1] = 0
    g = traces.config4(n_keys=n_keys, n_ticks=n_ticks, tick_size=max(sum(s) for s in sizes), hot=hot)
    per_tick = []
    for t, s in enumerate(sizes):
        tick = g[t * (len(g) // n_ticks):][:sum(s)]
        per_tick.append(np.split(tick, np.cumsum(s)[:-1]))
    return per_tick, max(max(s) for s in sizes)


def scenario_exact(world, report):
    per_tick, cap = ragged_config4(world, 6, hot=20)
    run = Run(world, cap)
    for lim in run.lims:
        lim.store.track_denied(1 << 20)
    stats0 = [lim.store.stats()["denied"] for lim in run.lims]
    for t in per_tick:
        run.submit(t)                                   # pipelined across ticks
    ticks = run.finish()
    assert not any((got["status"] == tc.INTERNAL).any() for _, got in ticks), "a row was refused"
    host = check_exact(run, ticks, "exact", stats0)
    glob = ordered(sum(host.values(), collections.Counter()))
    assert len(glob) > 100, "too few denied keys to test anything"
    cnt = [c for _, c in glob]
    tie = next(i for i in range(1, len(cnt)) if cnt[i] == cnt[i - 1])      # k that cuts through a group of ties
    ks = sorted({1, 5, 10, tie, tie + 1, len(glob) // 2, len(glob), len(glob) + 7})
    for k in ks:
        lists = [lim.store.top_denied(k)[0] for lim in run.lims]
        assert merge_top_denied(lists, k) == glob[:k], "merge_top_denied, k = %d" % k
    report.update(keys=[len(host[r]) for r in range(world)], denied=[sum(host[r].values()) for r in range(world)],
                  ks=ks, rows=[sum(len(x) for x in t) for t in per_tick])
    run.close()


def scenario_flood(world, report):
    tick = 1 << 22
    run = Run(world, tick, max_batch=world * tick, capacity=6_000_000)
    for lim in run.lims:
        lim.store.track_denied(1024)
    for ms in (0, 1, 1000):
        run.submit([flood(tick, traces.T0 + ms * 1_000_000) for _ in range(world)])
        run.join()
    ticks = run.finish()
    host = check_exact(run, ticks, "flood")
    owner = owners([0], world)[0]
    assert [len(host[r]) for r in range(world)] == [1 if r == owner else 0 for r in range(world)]
    report.update(owner=int(owner), denied=sum(host[owner].values()), rows=[len(g) for g, _ in ticks])
    run.close()


def refused_report(ticks, report):
    got = np.concatenate([g for _, g in ticks])
    report.update(refused=int((got["status"] == tc.INTERNAL).sum()),
                  denied=int(((got["status"] == tc.OK) & (got["allowed"] == 0)).sum()),
                  allowed=int(got["allowed"].sum()))


def scenario_residue(world, report):
    tick, mb = 1 << 16, 1 << 16
    run = Run(world, tick, max_batch=mb)
    for lim in run.lims:
        lim.store.track_denied(1024)
    # burst 2^15: of the rows before the refused residue, about 2^15 are allowed and the rest denied
    policy = (1 << 15, 1000, 1)
    for n, ms in ((tick, 1), (tick // 4, 2)):
        run.submit([flood(n, traces.T0 + ms * 1_000_000, policy) for _ in range(world)])
        run.join()
    ticks = run.finish()
    check_exact(run, ticks, "residue")
    refused_report(ticks, report)
    run.close()


def scenario_table_full(world, report):
    per, reps = 1 << 13, 6
    n_new = (world - 1) * per
    ids = np.arange(1, 8 * n_new + 1, dtype=np.uint64)
    ids = ids[owners(ids, world) == 0][:n_new]
    assert len(ids) == n_new
    per_rank = [rows(np.zeros(0, np.uint64), traces.T0, P4)]
    for r in range(1, world):
        mine = ids[(r - 1) * per:r * per]
        per_rank.append(rows(np.tile(mine, reps), traces.T0 + 1_000_000, P4))     # each key 6 times, spread out
    run = Run(world, per * reps, capacity=[1024] + [4_000_000] * (world - 1))
    for lim in run.lims:
        lim.store.track_denied(1 << 16)
    run.submit(per_rank)
    ticks = run.finish()
    check_exact(run, ticks, "table_full")
    refused_report(ticks, report)
    run.close()


def scenario_off_on(world, report):
    per_tick, cap = ragged_config4(world, 6, hot=20)
    out = {}
    for mode in ("off", "on", "later"):
        run = Run(world, cap)
        if mode == "on":
            for lim in run.lims:
                lim.store.track_denied(1 << 20)
        stats0 = None
        for t, tick in enumerate(per_tick):
            if mode == "later" and t == 3:
                run.join()                              # between ticks, after every engine's join
                for lim in run.lims:
                    lim.store.track_denied(1 << 20)
                stats0 = [lim.store.stats()["denied"] for lim in run.lims]
            run.submit(tick)
            run.join()
        ticks = run.finish()
        if mode == "on":
            check_exact(run, ticks, "on", [0] * world)
        elif mode == "later":
            check_exact(run, ticks[3:], "later", stats0)
        out[mode] = (run.launches, b"".join(g.tobytes() for _, g in ticks))
        run.close()
    assert out["on"][1] == out["off"][1], "tracking changed a result"
    assert out["later"][1] == out["off"][1], "tracking changed a result"
    report.update(launches={m: out[m][0] for m in out})


def host_prune(counter, max_keys):
    """gcra_top_denied's cleanup: more than 3 x max_keys keys -> keep the top max_keys"""
    if len(counter) > 3 * max_keys:
        return collections.Counter(dict(ordered(counter)[:max_keys]))
    return collections.Counter(counter)


def scenario_prune(world, report):
    max_keys = 64
    ids = np.arange(1, 40_000, dtype=np.uint64)
    own = owners(ids, world)
    many, few = ids[own == 0][:5 * max_keys], ids[own == 1][:2 * max_keys]       # 320 > 3 x 64 > 128 keys

    def tick(keys, extra, ms):
        """key i: 3 + 1 + (i % 7) rows (burst 3: the rest denied), split between the ranks in order"""
        k = np.repeat(keys, [4 + (i % 7) + extra for i in range(len(keys))])
        sl = rows(k, traces.T0 + ms * 1_000_000, P4)
        return [sl[r::world] for r in range(world)]
    run = Run(world, 8192)
    for lim in run.lims:
        lim.store.track_denied(max_keys)
    first = [np.concatenate(p) for p in zip(tick(many, 0, 1), tick(few, 0, 1))]
    run.submit(first)
    ticks1 = run.finish()
    host = host_counts(ticks1, world)
    assert len(host[0]) > 3 * max_keys and len(host[1]) <= 3 * max_keys
    model = {r: collections.Counter(host[r]) for r in range(world)}
    for r, lim in enumerate(run.lims):
        got, _ = lim.store.top_denied(10)                  # the query that prunes
        assert got == ordered(model[r])[:10], "prune: rank %d top 10" % r
        model[r] = host_prune(model[r], max_keys)
        assert lim.store.top_denied(ALL)[0] == ordered(model[r]), "prune: rank %d after the query" % r
    # a second tick adds to the pruned table: new keys of rank 0, and again the old ones (all still saturated)
    more = ids[own == 0][5 * max_keys:9 * max_keys]
    run.submit([np.concatenate(p) for p in zip(tick(more, 1, 2), tick(many[:50], 0, 2))])
    ticks2 = run.finish()
    host2 = host_counts(ticks2, world)
    for r, lim in enumerate(run.lims):
        model[r] += host2[r]
        got, _ = lim.store.top_denied(ALL)
        assert got == ordered(model[r]), "prune: rank %d after the second tick" % r
        model[r] = host_prune(model[r], max_keys)
        assert lim.store.top_denied(ALL)[0] == ordered(model[r]), "prune: rank %d after the second query" % r
    report.update(keys_before=[len(host[r]) for r in range(world)], keys_after=[len(model[r]) for r in range(world)])
    run.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("scenario", choices=["exact", "flood", "residue", "table_full", "off_on", "prune"])
    ap.add_argument("world", type=int)
    a = ap.parse_args()
    report = {"scenario": a.scenario, "world": a.world}
    globals()["scenario_" + a.scenario](a.world, report)
    print(json.dumps(report))
    print("denied ok")


if __name__ == "__main__":
    main()
