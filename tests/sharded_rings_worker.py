"""Child process of tests/test_gpu_sharded_rings.py: `world` engines in one process (on cuda:0, or one per GPU with
--gpus), connected over peer memory (sharded.connect_local), each with a mixed ring whose submits are peer-memory
ticks (gcra_ring_p2p).  Every connection must give what its protocol's host walk gives at its own rank's row cap, and
its replies must be its protocol's formatter applied to ONE oracle store that decides each tick's rows in rank order.

    sharded_rings_worker.py SCENARIO WORLD [--gpus]

SCENARIO: ticks | seeded | tight | mixed_ticks | world1 | refusals | driver.  Prints "sharded rings ok"."""
import argparse
import ctypes as C
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
import throttlecrab_b200 as tc  # noqa: E402
from throttlecrab_b200 import mixed  # noqa: E402
from throttlecrab_b200.sharded import connect_local  # noqa: E402
from test_gpu_mixed_ring import NOW, NS, SIP, _check, _driver_mix, _expected, _fuzz_conns, _place, _shared_conn  # noqa: E402
from test_mixed_cpu import copy_conns  # noqa: E402
from test_resp import _throttle  # noqa: E402

ROW_CAP = 1 << 12


def engines(world, seed=(0, 0), capacity=1 << 20, flags=0, gpus=False, row_cap=ROW_CAP, cap_rows=ROW_CAP, slots=2):
    lims = [tc.RateLimiter(tc.PeriodicStore(capacity=capacity, device=r if gpus else 0, created_ns=NOW,
                                            max_batch=1 << 16, flags=flags, hash_seed=seed)) for r in range(world)]
    rings = [tc.MixedRing(lim, slots, 256, 1 << 21, row_cap) for lim in lims]
    connect_local(lims, cap_rows)
    for ring in rings:
        ring.peer_memory(True)
    return lims, rings


class Oracle:
    """ONE store for the whole key space, keys named by their hash (every rank hashes under one seed)"""

    def __init__(self):
        self.st = oracle.OracleStore(oracle.PERIODIC, capacity=1 << 14, created_ns=NOW, p0=NS)
        self.keys = set()
        self.counts = np.zeros(3, np.int64)            # allowed, denied, errors

    def decide(self, rows):
        out = np.zeros(len(rows), tc.RES_DTYPE)
        for i, q in enumerate(rows):
            h = int(q["key_hash"])
            self.keys.add(h)
            st, a, rem, reset, retry = self.st.rate_limit("h%d" % h, int(q["max_burst"]), int(q["count_per_period"]),
                                                          int(q["period"]), int(q["quantity"]), int(q["now_ns"]))
            out[i] = (rem, reset, retry, st, a, [0, 0, 0])
            self.counts += (st == tc.OK and a, st == tc.OK and not a, st != tc.OK)
        return out

    def check_final(self, lims, now):
        """every key's entry on its owner, and the engines' summed counters, against the oracle's (the oracle's sweeps
        may have removed an entry that expired by `now`; peer-memory ticks leave sweeping to the caller)"""
        L, world = tc._native.lib(), len(lims)
        for h in self.keys:
            got, want = lims[L.gcra_owner_of(h, world)].store.peek(h), self.st.entry("h%d" % h)
            assert got == want or (want is None and got[1] <= now), (h, got, want)
        s = [lim.store.stats() for lim in lims]
        got = [sum(x[f] for x in s) for f in ("allowed", "denied", "errors")]
        assert got == list(self.counts), (got, list(self.counts))


def ring_conns(rng, nrng, rank, t, n):
    """fuzzed connections of every kind, keys shared across ranks and transports, one hot key in every rank's rows"""
    conns = _fuzz_conns(rng, nrng, n // 2) + [_shared_conn(rng, rng.choice(["resp", "http", "grpc"]))
                                              for _ in range(n - n // 2)]
    conns.insert(rng.randrange(len(conns) + 1), ("resp", _throttle("hot", 5, 10, 60) * 3, None))
    rng.shuffle(conns)
    return conns


def bulk_rows(rng, lim, n, now):
    rows = np.zeros(n, tc.REQ_DTYPE)
    for i in range(n):
        k = rng.choice(["hot", "t1", "t2", "cold%d" % rng.randrange(1000)])
        rows[i] = (lim.store.hash_key(k.encode()), rng.choice([1, 4]), 10, 60, rng.choice([1, 2]), now)
    return rows


def gave_up(lims):
    e = C.c_uint32()
    for lim in lims:
        lim.store._check(lim._L.gcra_p2p_error(lim._h, C.byref(e)))
        if e.value:
            return True
    return False


def run_ticks(lims, rings, kinds, rng, nrng, sizes, sync_each=False):
    """kinds[t][r]: 'ring' or 'bulk' (gcra_p2p_submit), sizes(t, r) -> connections (or rows) of rank r at tick t.
    Ring slots alternate per rank; a slot is checked when it is reused and at the end, so that up to 2 ring ticks and
    any number of bulk ticks per rank are in flight."""
    import torch
    world = len(lims)
    ora = Oracle()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    pending = [[None, None] for _ in range(world)]      # per rank and slot: (conns, exp, oracle results)
    nxt = [0] * world
    bulk = []                                            # (d_res, n, oracle results)
    keep = []
    stops3 = 0

    def check(r, s):
        nonlocal stops3
        if pending[r][s] is None:
            return
        conns, exp, ores = pending[r][s]
        rings[r].wait(s)
        assert not gave_up(lims), "a wait gave up"
        try:
            _check(rings[r], s, conns, exp, ores)
        except AssertionError:
            _, res = rings[r].rows(s)
            m = min(len(res), len(ores))
            bad = np.nonzero((res[:m].view(np.uint8).reshape(-1, 32) != ores[:m].view(np.uint8).reshape(-1, 32)).any(1))[0]
            print("rank %d slot %d: %d rows, %d differ, first %s: got %s want %s" % (
                r, s, len(res), len(bad), bad[:8], res[bad[:3]], ores[bad[:3]]), file=sys.stderr)
            raise
        stops3 += sum(e[0][2] == 3 for e in exp)
        pending[r][s] = None

    for t, kt in enumerate(kinds):
        now = NOW + t * NS // 4
        jobs = []
        for r in range(world):
            n = sizes(t, r)
            if kt[r] == "ring":
                s = nxt[r]
                nxt[r] ^= 1
                check(r, s)
                conns = ring_conns(rng, nrng, r, t, n) if n else []
                exp = _expected(lims[r], conns, rings[r].row_capacity, now)
                _place(rings[r], s, conns)
                rows = np.concatenate([e[1] for e in exp]) if exp else np.zeros(0, tc.REQ_DTYPE)
                jobs.append(("ring", s, conns, exp, rows))
            else:
                rows = bulk_rows(rng, lims[r], n, now)
                q = torch.from_numpy(rows.view(np.uint8)).to(dev) if n else torch.zeros(48, dtype=torch.uint8,
                                                                                          device=dev)
                res = torch.zeros(max(n, 1) * 32, dtype=torch.uint8, device=dev)
                keep.append(q)
                jobs.append(("bulk", q, res, n, rows))
        torch.cuda.synchronize()
        # one tick: every rank's rows in rank order, decided by the oracle as one sequence
        ores = ora.decide(np.concatenate([j[4] for j in jobs]))
        at = 0
        for r, j in enumerate(jobs):
            mine = ores[at:at + len(j[4])]
            at += len(j[4])
            if j[0] == "ring":
                rings[r].submit_route(j[1], len(j[2]), now)
                pending[r][j[1]] = (j[2], j[3], mine)
            else:
                lims[r].store._check(lims[r]._L.gcra_p2p_submit_route(lims[r]._h, j[3], j[1].data_ptr(),
                                                                      stream.cuda_stream))
                bulk.append((j[2], j[3], mine))
        for r, j in enumerate(jobs):                    # every route of the tick before the first finish
            if j[0] == "ring":
                rings[r].submit_finish(j[1])
            else:
                lims[r].store._check(lims[r]._L.gcra_p2p_submit_finish(lims[r]._h, j[2].data_ptr()))
        if sync_each:
            for r in range(world):
                for s in (0, 1):
                    check(r, s)
    for r in range(world):
        for s in (0, 1):
            check(r, s)
        lims[r].store._check(lims[r]._L.gcra_p2p_join(lims[r]._h, None))
    for res, n, mine in bulk:
        got = res.cpu().numpy().view(tc.RES_DTYPE)[:n]
        assert got.tobytes() == mine.tobytes()
    for lim in lims:
        e = C.c_uint32()
        lim.store._check(lim._L.gcra_p2p_error(lim._h, C.byref(e)))
        assert e.value == 0, "a wait gave up"
    ora.check_final(lims, now)
    return stops3


def scenario_ticks(world, gpus, seed=(0, 0)):
    """keys shared across ranks and transports, a hot key, a rank whose slot fills (stop 3) while the others' do
    not, ranks with 0 connections, 2 ring slots per engine in flight"""
    rng, nrng = random.Random(world), np.random.default_rng(world)
    lims, rings = engines(world, seed, gpus=gpus, row_cap=600, cap_rows=1024)

    def sizes(t, r):
        if world > 1 and r == (t + 1) % world and t % 3 == 1:
            return 0                                      # a rank with no connections
        return 220 if (r == 0 and t % 2 == 0) else rng.randrange(1, 40)   # rank 0 fills its slot every other tick
    stops3 = run_ticks(lims, rings, [["ring"] * world for _ in range(8)], rng, nrng, sizes)
    assert stops3 > 0


def scenario_mixed_ticks(world, gpus):
    """ring ticks interleaved with gcra_p2p_submit ticks (rank r's tick a ring tick while rank s's is not), more ticks
    in flight than P2P_DEPTH"""
    rng, nrng = random.Random(100 + world), np.random.default_rng(100 + world)
    lims, rings = engines(world, SIP, gpus=gpus)
    kinds = [[("ring" if (t + r) % 3 else "bulk") for r in range(world)] for t in range(14)]
    run_ticks(lims, rings, kinds, rng, nrng, lambda t, r: rng.randrange(0, 50))


def scenario_tight(world, gpus):
    """a tight table (GCRA_FLAG_TIGHT_TABLE) that grows on the owners between ring ticks"""
    rng, nrng = random.Random(200 + world), np.random.default_rng(200 + world)
    lims, rings = engines(world, capacity=64, flags=tc._native.FLAG_TIGHT_TABLE, gpus=gpus)
    run_ticks(lims, rings, [["ring"] * world for _ in range(6)], rng, nrng, lambda t, r: rng.randrange(20, 60),
              sync_each=True)
    assert all(lim.store.stats()["grows"] > 0 for lim in lims)


def scenario_world1():
    """world 1: ring p2p gives the outcomes and reply bytes of the plain ring on a twin engine"""
    rng, nrng = random.Random(5), np.random.default_rng(5)
    lims, rings = engines(1, SIP)
    twin = tc.RateLimiter(tc.PeriodicStore(capacity=1 << 20, created_ns=NOW, max_batch=1 << 16, hash_seed=SIP))
    tring = tc.MixedRing(twin, 2, 256, 1 << 21, ROW_CAP)
    for t in range(6):
        conns = ring_conns(rng, nrng, 0, t, rng.randrange(0, 80))
        for ring in (rings[0], tring):
            _place(ring, t % 2, conns)
            ring.submit(t % 2, len(conns), NOW + t * NS)
            ring.wait(t % 2)
        for f in ("consumed", "n_frames", "stop", "reply_off", "reply_len"):
            assert (rings[0].outcome[t % 2][:len(conns)][f] == tring.outcome[t % 2][:len(conns)][f]).all(), (t, f)
        k = sum(p == "grpc" for p, _, _ in conns)
        assert rings[0].grpc_outcome[t % 2][:k].tobytes() == tring.grpc_outcome[t % 2][:k].tobytes()
        if conns:
            end = int(tring.outcome[t % 2][len(conns) - 1]["reply_off"] + tring.outcome[t % 2][len(conns) - 1]["reply_len"])
            assert rings[0].replies[t % 2][:end].tobytes() == tring.replies[t % 2][:end].tobytes()
        a, b = rings[0].rows(t % 2), tring.rows(t % 2)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def _refused(fn):
    try:
        fn()
    except tc.CellError:
        return
    raise AssertionError("not refused")


def scenario_refusals(world, gpus):
    """every refusal of gcra_ring_p2p and its metrics twin, each leaving the engines usable"""
    lone = tc.RateLimiter(tc.PeriodicStore(capacity=1 << 12, created_ns=NOW, max_batch=1 << 12))
    lring = tc.MixedRing(lone, 1, 8, 1 << 16, 256)
    _refused(lambda: lring.peer_memory(True))                                   # not prepared
    w = C.c_void_p()
    lone.store._check(lone._L.gcra_p2p_prepare(lone._h, 0, 1, 256, None, C.byref(w)))
    _refused(lambda: lring.peer_memory(True))                                   # prepared, not connected
    _refused(lambda: lring.submit_route(0, 0, NOW))
    lring.submit(0, 0, NOW)
    lring.wait(0)
    # row_capacity above the peer-memory cap (1024 rows: the power of two >= 1000)
    lims, rings = [tc.RateLimiter(tc.PeriodicStore(capacity=1 << 12, device=r if gpus else 0, created_ns=NOW,
                                                   max_batch=1 << 12)) for r in range(world)], []
    rings = [tc.MixedRing(lim, 1, 8, 1 << 16, 1025) for lim in lims]
    connect_local(lims, 1000)
    for ring in rings:
        _refused(lambda: ring.peer_memory(True))
    # a rank whose key-hash seed differs: every rank refuses
    if world > 1:
        lims = [tc.RateLimiter(tc.PeriodicStore(capacity=1 << 12, device=r if gpus else 0, created_ns=NOW,
                                                max_batch=1 << 12, hash_seed=(1, 2) if r == world - 1 else SIP))
                for r in range(world)]
        rings = [tc.MixedRing(lim, 1, 8, 1 << 16, 256) for lim in lims]
        connect_local(lims, 256)
        for ring in rings:
            _refused(lambda: ring.peer_memory(True))
    # metrics on, both orders; then the engines serve a tick against the oracle
    rng, nrng = random.Random(9), np.random.default_rng(9)
    lims, rings = engines(world, SIP, gpus=gpus)
    rings[0].peer_memory(False)
    lims[0].store.ring_metrics(True)
    _refused(lambda: rings[0].peer_memory(True))
    lims[0].store.ring_metrics(False)
    rings[0].peer_memory(True)
    _refused(lambda: lims[0].store.ring_metrics(True))
    _refused(lambda: rings[0].submit_finish(0))                                 # nothing routed
    run_ticks(lims, rings, [["ring"] * world for _ in range(2)], rng, nrng, lambda t, r: 10)


def scenario_driver(world, gpus):
    """process_connections_sharded over `world` engines gives every connection the bytes that
    process_connections(ring=None) gives on ONE engine over the joined connection list"""
    rng = random.Random(30 + world)
    lims, rings = engines(world, SIP, gpus=gpus, row_cap=1 << 14, cap_rows=1 << 14)
    one = tc.RateLimiter(tc.PeriodicStore(capacity=1 << 20, created_ns=NOW, max_batch=1 << 16, hash_seed=SIP))
    for rnd in range(4):
        per = [_driver_mix(rng, rnd if r == 0 else 1) for r in range(world)]
        if rnd == 2:
            per[world - 1] = []                                                 # a rank with no connections
        joined = copy_conns([c for cs in per for c in cs])
        now = NOW + rnd * NS
        got = mixed.process_connections_sharded([(cs, lim, ring) for cs, lim, ring in zip(per, lims, rings)], now)
        want = mixed.process_connections(joined, one, now, None)
        assert not gave_up(lims), "a wait gave up"
        flat = [x for g in got for x in g]
        if flat != want:
            c = next(i for i, (x, y) in enumerate(zip(flat, want)) if x != y)
            print("round %d: connection %d of %d differs: got %r want %r" % (rnd, c, len(want), flat[c], want[c]),
                  file=sys.stderr)
        assert flat == want, rnd
        assert [len(g) for g in got] == [len(cs) for cs in per]
        for (p, a), (_, b) in zip([c for cs in per for c in cs], joined):
            if p == "grpc":
                assert (bytes(a.out), bytes(a.buf), a.last_stream, a.send_window, a.closed) == \
                    (bytes(b.out), bytes(b.buf), b.last_stream, b.send_window, b.closed)
    s = [lim.store.stats() for lim in lims]
    o = one.store.stats()
    for f in ("allowed", "denied", "errors"):
        assert sum(x[f] for x in s) == o[f], f
    try:
        mixed.process_connections_sharded([([], lim, ring) for lim, ring in zip(lims, rings)], NOW, metrics=print)
    except ValueError:
        pass
    else:
        raise AssertionError("metrics accepted")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("scenario")
    ap.add_argument("world", type=int)
    ap.add_argument("--gpus", action="store_true", help="engine r on GPU r")
    a = ap.parse_args()
    if a.scenario == "ticks":
        scenario_ticks(a.world, a.gpus)
    elif a.scenario == "seeded":
        scenario_ticks(a.world, a.gpus, SIP)
    elif a.scenario == "mixed_ticks":
        scenario_mixed_ticks(a.world, a.gpus)
    elif a.scenario == "tight":
        scenario_tight(a.world, a.gpus)
    elif a.scenario == "world1":
        scenario_world1()
    elif a.scenario == "refusals":
        scenario_refusals(a.world, a.gpus)
    elif a.scenario == "driver":
        scenario_driver(a.world, a.gpus)
    else:
        raise SystemExit("unknown scenario " + a.scenario)
    print("sharded rings ok: %s, world %d" % (a.scenario, a.world))


if __name__ == "__main__":
    main()
