"""Child process of tests/test_gpu_sharded_ring_metrics.py: sharded ring metrics (gcra_ring_metrics_sharded,
gcra_ring_names_keep, gcra_denied_names on a name table) and metrics.ShardedMetrics over `world` engines of one process
(on cuda:0, or one per GPU with --gpus) whose mixed rings' submits are peer-memory ticks.

    sharded_ring_metrics_worker.py SCENARIO WORLD [--gpus]

SCENARIO: counts | world1_text | driver | prune | full | refusals.  Prints "sharded ring metrics ok"."""
import argparse
import os
import random
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
from throttlecrab_b200 import mixed  # noqa: E402
from throttlecrab_b200.metrics import Metrics, ShardedMetrics  # noqa: E402
from throttlecrab_b200.sharded import merge_top_denied  # noqa: E402
import grpc_streams as gs  # noqa: E402
from sharded_rings_worker import Oracle, _refused, engines, gave_up  # noqa: E402
from test_gpu_mixed_ring import MIN_FRAME, NOW, NS, SIP, _check, _expected, _fuzz_conns, _place  # noqa: E402
from test_gpu_ring_metrics import _e2e_conns, _events, _http_responses, _model_text  # noqa: E402
from test_http_cpu import body_of, request  # noqa: E402
from test_mixed_cpu import copy_conns  # noqa: E402
from test_resp import _throttle  # noqa: E402

T = {"resp": 0, "http": 1, "grpc": 2}
KEYS = ["hot", "", "a", "L" * 255, "M" * 256, "N" * 257] + ["s%d" % i for i in range(12)]
GET_METRICS = ("http", b"GET /metrics HTTP/1.1\r\nHost: x\r\n\r\n")


def metric_conns(rng, nrng, n):
    """connections of all three protocols over KEYS (shared by every rank and transport; keys of 0, 1, 255, 256 and
    257 bytes), errors among them, a few fuzzed ones, and a hot RESP connection"""
    def args():
        return rng.choice([1, 2, 5]), rng.choice([1, 10]), 60, rng.choice([None, 1, 1, 2, 5, -1])
    out = []
    for _ in range(n):
        p, k = rng.choice(["resp", "http", "grpc"]), rng.randrange(0, 12)
        if p == "resp":
            out.append(("resp", b"".join(_throttle(rng.choice(KEYS), *args()) for _ in range(k)), None))
        elif p == "http":
            out.append(("http", b"".join(request(body_of(rng.choice(KEYS), *args())) for _ in range(k)), None))
        else:
            cn = gs.established()
            out.append(("grpc", gs.steady_stream(rng, cn, k, KEYS, extras=False), cn.conn_row()))
    out += _fuzz_conns(rng, nrng, 3)
    out.insert(rng.randrange(len(out) + 1), ("resp", _throttle("hot", 1, 1, 60, 2) * 6, None))
    rng.shuffle(out)
    return out


def check_names(lim, r, seen, denied_through, key_of):
    """every hash denied through rank r named on r with its key's exact bytes (or too long); every other UNKNOWN"""
    hs = sorted(seen)
    for h, nm in zip(hs, lim.store.denied_names(hs)):
        if h not in denied_through:
            assert nm == tc.NAME_UNKNOWN, (r, h, nm)
        elif h in key_of:
            want = key_of[h] if len(key_of[h]) <= tc.DENIED_NAME_MAX else tc.NAME_TOO_LONG
            assert nm == want, (r, key_of[h][:20], nm)
        else:                                                  # (a fuzzed key: its name must hash back to it)
            assert nm == tc.NAME_TOO_LONG or lim.store.hash_key(nm) == h, (r, h, nm)


def drive(lims, rings, ticks, rng, nrng, twins=None, ora=None, t0=0):
    """`ticks` ring ticks over every rank (twins: a second set of engines with metrics off, the same connections),
    checked against one oracle store (`ora`, from tick t0 on) -> (oracle, per-rank counts [3, 3], per-rank {hash: denials through it}, every
    hash seen, connections that stopped at a full slot)"""
    world = len(lims)
    ora = ora or Oracle()
    counts = [np.zeros((3, 3), np.uint64) for _ in range(world)]
    through = [dict() for _ in range(world)]
    seen = set()
    stops = 0
    for t in range(ticks):
        now = NOW + (t0 + t) * NS // 4
        s = t % 2
        jobs = []
        for r in range(world):
            # a rank with no connections now and then; rank 0's slot fills every other tick
            n = 0 if world > 1 and r == (t + 1) % world and t % 3 == 1 else \
                90 if r == 0 and t % 2 == 0 else rng.randrange(1, 20)
            conns = metric_conns(rng, nrng, n) if n else []
            exp = _expected(lims[r], conns, rings[r].row_capacity, now)
            rows = np.concatenate([e[1] for e in exp]) if exp else np.zeros(0, tc.REQ_DTYPE)
            stops += sum(e[0][2] == 3 for e in exp)
            jobs.append((conns, exp, rows))
        ores = ora.decide(np.concatenate([j[2] for j in jobs]))
        sets = [(lims, rings)] + ([twins] if twins else [])
        before = [[lim.store.launch_count() for lim in ls] for ls, _ in sets]
        for ls, rs in sets:
            for r in range(world):
                _place(rs[r], s, jobs[r][0])
            for r in range(world):                              # every route of the tick before the first finish
                rs[r].submit_route(s, len(jobs[r][0]), now)
            for r in range(world):
                rs[r].submit_finish(s)
        at = 0
        for r, (conns, exp, rows) in enumerate(jobs):
            mine = ores[at:at + len(rows)]
            at += len(rows)
            for ls, rs in sets:
                rs[r].wait(s)
                _check(rs[r], s, conns, exp, mine)              # rows, results, outcomes and replies
            if twins:
                out, tout = rings[r].outcome[s][:len(conns)], twins[1][r].outcome[s][:len(conns)]
                assert out.tobytes() == tout.tobytes()
                k = sum(p == "grpc" for p, _, _ in conns)
                assert rings[r].grpc_outcome[s][:k].tobytes() == twins[1][r].grpc_outcome[s][:k].tobytes()
                end = max([int(o["reply_off"]) + int(o["reply_len"]) for o in out] + [0])
                assert rings[r].replies[s][:end].tobytes() == twins[1][r].replies[s][:end].tobytes()
                got = lims[r].store.launch_count() - before[0][r]
                tgot = twins[0][r].store.launch_count() - before[1][r]
                bound = min(rings[r].row_capacity, sum(len(d) // MIN_FRAME[p] for p, d, _ in conns))
                assert got == tgot + (1 if bound else 0), (t, r, got, tgot, bound)
            i = 0
            for (p, _, _), e in zip(conns, exp):
                for q, o in zip(e[1], mine[i:i + len(e[1])]):
                    ok, allowed = int(o["status"]) == tc.OK, bool(o["allowed"])
                    cls = 1 if ok and not allowed else 0 if ok or p == "resp" else 2
                    counts[r][T[p], cls] += 1
                    h = int(q["key_hash"])
                    seen.add(h)
                    if cls == 1:
                        through[r][h] = through[r].get(h, 0) + 1
                i += len(e[1])
        assert not gave_up(lims), "a wait gave up"
    return ora, counts, through, seen, stops


def oracle_denied(ora, through):
    """denials per hash of the whole replay"""
    den = {}
    for th in through:
        for h, n in th.items():
            den[h] = den.get(h, 0) + n
    assert sum(den.values()) == ora.counts[1]
    return den


def scenario_counts(world, gpus):
    """1 to `world` loop-back engines: per-rank transport counts and names, the owners' merged top list, results,
    replies, final entries and launches against twins with sharded metrics off; then off: launches equal"""
    rng, nrng = random.Random(world), np.random.default_rng(world)
    lims, rings = engines(world, SIP, gpus=gpus, row_cap=400, cap_rows=1024)
    tl, tr = engines(world, SIP, gpus=gpus, row_cap=400, cap_rows=1024)
    key_of = {lims[0].store.hash_key(k.encode()): k.encode() for k in KEYS}
    for lim in lims + tl:
        lim.store.track_denied(1000)
    for lim in lims:
        lim.store.ring_metrics_sharded(True, 100)
    ora, counts, through, seen, stops = drive(lims, rings, 8, rng, nrng, twins=(tl, tr))
    assert stops > 0                                            # (rank 0's slot filled: stop 3)
    for r in range(world):
        assert (lims[r].store.ring_transport_counts() == counts[r]).all(), (r, lims[r].store.ring_transport_counts(),
                                                                             counts[r])
        assert (tl[r].store.ring_transport_counts() == 0).all()
        check_names(lims[r], r, seen, through[r], key_of)
    assert any(nm == tc.NAME_TOO_LONG for nm in lims[0].store.denied_names(sorted(through[0])))
    den = oracle_denied(ora, through)
    lists = [lim.store.top_denied(1 << 12)[0] for lim in lims]
    assert merge_top_denied(lists, 1 << 12) == sorted(den.items(), key=lambda hc: (-hc[1], hc[0]))
    assert lists == [lim.store.top_denied(1 << 12)[0] for lim in tl]
    ora.check_final(lims, NOW + 8 * NS // 4)
    ora.check_final(tl, NOW + 8 * NS // 4)
    # off: no kernel more than the twins', counts kept, names released
    for lim in lims:
        lim.store.ring_metrics_sharded(False, 0)
    drive(lims, rings, 2, rng, nrng, ora=ora, t0=8)             # (results against the same oracle)
    l0, t0 = [lim.store.launch_count() for lim in lims], [lim.store.launch_count() for lim in tl]
    for ls, rs in ((lims, rings), (tl, tr)):
        for r in range(world):
            _place(rs[r], 0, [("resp", _throttle("hot", 1, 1, 60, 2) * 3, None)])
        for r in range(world):
            rs[r].submit_route(0, 1, NOW + 3 * NS)
        for r in range(world):
            rs[r].submit_finish(0)
        for r in range(world):
            rs[r].wait(0)
    assert [lim.store.launch_count() - a for lim, a in zip(lims, l0)] == \
        [lim.store.launch_count() - a for lim, a in zip(tl, t0)]
    for r in range(world):
        assert (lims[r].store.ring_transport_counts() == counts[r]).all()
        assert lims[r].store.denied_names(sorted(seen)) == [tc.NAME_UNKNOWN] * len(seen)


def _mask(text):
    return re.sub(r"throttlecrab_uptime_seconds \d+\n", "throttlecrab_uptime_seconds U\n", text)


def scenario_world1_text():
    """world 1 with ring p2p off: ShardedMetrics([lim]) serves the text Metrics serves on a twin, over the same
    traffic, scrape after scrape"""
    rng = random.Random(11)
    lims, rings = engines(1, SIP, row_cap=4096, cap_rows=4096)
    rings[0].peer_memory(False)
    twin = tc.RateLimiter(tc.PeriodicStore(capacity=1 << 20, created_ns=NOW, max_batch=1 << 16, hash_seed=SIP))
    tring = tc.MixedRing(twin, 2, 256, 1 << 21, 4096)
    m, tm = ShardedMetrics(lims, 3), Metrics(twin, 3)
    for rnd in range(3):
        conns, _ = _e2e_conns(rng)
        tconns = copy_conns(conns)
        now = NOW + rnd * NS
        a = mixed.process_connections(conns, lims[0], now, rings[0], metrics=m)
        b = mixed.process_connections(tconns, twin, now, tring, metrics=tm)
        assert a == b
        text = _mask(m())
        assert text == _mask(tm()), (text, tm())
        assert "throttlecrab_top_denied_keys{" in text


def scenario_driver(world, gpus):
    """process_connections_sharded with a ShardedMetrics: GET /metrics text against an independent model of metrics.rs
    fed by the replies; other callables still refused"""
    rng = random.Random(40 + world)
    lims, rings = engines(world, SIP, gpus=gpus, row_cap=1 << 14, cap_rows=1 << 14)
    m = ShardedMetrics(lims, 100)
    conns, reqs = _e2e_conns(rng)
    per = [[c for i, c in enumerate(conns) if i % world == r] for r in range(world)]
    preq = [[q for i, q in enumerate(reqs) if i % world == r] for r in range(world)]
    got = mixed.process_connections_sharded([(cs, lim, ring) for cs, lim, ring in zip(per, lims, rings)], NOW,
                                            metrics=m)
    assert not gave_up(lims), "a wait gave up"
    ev = _events([c for cs in per for c in cs], [q for qs in preq for q in qs], [g for gs_ in got for g in gs_])
    assert {o for _, _, o in ev} == {"allowed", "denied", "error"}
    last = world - 1                                            # (the scrape comes in on the last rank)
    scrape = mixed.process_connections_sharded(
        [([GET_METRICS] if r == last else [], lim, ring) for r, (lim, ring) in enumerate(zip(lims, rings))], NOW,
        metrics=m)
    (status, body), = _http_responses(scrape[last][0][0])
    assert status == 200
    text = _mask(body.decode())
    head, top = _model_text(ev)
    assert text.startswith(head), (text, head)
    lines = text[len(head):].splitlines()
    parsed = [re.fullmatch(r'throttlecrab_top_denied_keys\{key="(.*)",rank="(\d+)"\} (\d+)', ln) for ln in lines]
    assert all(parsed) and [int(x.group(2)) for x in parsed] == list(range(1, len(lines) + 1))
    cnt = [int(x.group(3)) for x in parsed]
    assert cnt == sorted(cnt, reverse=True)
    assert {(x.group(1), int(x.group(3))) for x in parsed} == top
    assert any(k.startswith("q") for k, _ in top)
    bads = [lambda: print, lambda: ShardedMetrics(lims + lims[:1])] + \
        ([lambda: ShardedMetrics(lims[::-1])] if world > 1 else [])
    for make in bads:
        bad = make()
        try:
            mixed.process_connections_sharded([([], lim, ring) for lim, ring in zip(lims, rings)], NOW, metrics=bad)
        except ValueError:
            pass
        else:
            raise AssertionError("metrics accepted: %r" % (bad,))


def _deny_conn(keys_times):
    return ("resp", b"".join(_throttle(k, 1, 1, 60, 5) * n for k, n in keys_times))


def scenario_prune(world, gpus):
    """more than 3 x k distinct denied keys on the owners: the scrape's top list, then every rank's name table holds
    exactly the names of the keys that survived their owner's pruning and that rank's connections named"""
    k = 4
    lims, rings = engines(world, SIP, gpus=gpus, row_cap=1 << 14, cap_rows=1 << 14)
    m = ShardedMetrics(lims, k)
    L = tc._native.lib()
    per = [[] for _ in range(world)]
    per[0].append(_deny_conn([("p:%d" % i, i % 7 + 1) for i in range(40)]))
    per[-1].append(_deny_conn([("x:%d" % j, j + 1) for j in range(5)] + [("p:%d" % i, 1) for i in range(5)]))
    cnt, named_on = {}, [set() for _ in range(world)]
    for r, cs in enumerate(per):
        for _, data in cs:
            for key in re.findall(rb"\$\d+\r\n([px]:\d+)\r\n", data):
                h = lims[0].store.hash_key(key)
                cnt[h] = cnt.get(h, 0) + 1
                named_on[r].add(h)
    got = mixed.process_connections_sharded([(cs, lim, ring) for cs, lim, ring in zip(per, lims, rings)], NOW,
                                            metrics=m)
    assert all(g[1] == len(c[1]) for gr, cs in zip(got, per) for g, c in zip(gr, cs))
    name = {lims[0].store.hash_key(b"%s:%d" % (p, i)): "%s:%d" % (p.decode(), i)
            for p in (b"p", b"x") for i in range(40)}
    order = sorted(cnt, key=lambda h: (-cnt[h], h))
    assert m.top_denied_keys() == [(name[h], cnt[h]) for h in order[:k]]
    survivors = set()
    for r in range(world):
        mine = [h for h in order if L.gcra_owner_of(h, world) == r]
        survivors |= set(mine[:k] if len(mine) > 3 * k else mine)
    assert len(survivors) < len(cnt)                            # (some owner pruned)
    hs = sorted(cnt)
    for r in range(world):
        want = [name[h].encode() if h in survivors and h in named_on[r] else tc.NAME_UNKNOWN for h in hs]
        assert lims[r].store.denied_names(hs) == want, r
    assert m.full == 0
    assert m.top_denied_keys() == [(name[h], cnt[h]) for h in order[:k]]    # (the survivors still name the top k)


def scenario_full(world, gpus):
    """a name table driven full (max_keys 1: 1,024 entries) by 1,100 keys denied once: names it holds are exact,
    `full` counts the denied rows of the rest (one of them denied 3 times more); after a keep the table holds the kept names only and names new keys again"""
    lims, rings = engines(world, SIP, gpus=gpus, row_cap=4096, cap_rows=4096)
    lims[0].store.ring_metrics_sharded(True, 1)
    for lim in lims[1:]:
        lim.store.ring_metrics_sharded(True, 100)
    keys = [b"f:%d" % i for i in range(1100)]
    hs = [lims[0].store.hash_key(x) for x in keys]

    def tick(conns):
        for r in range(world):
            _place(rings[r], 0, conns if r == 0 else [])
        for r in range(world):
            rings[r].submit_route(0, len(conns) if r == 0 else 0, NOW)
        for r in range(world):
            rings[r].submit_finish(0)
        for r in range(world):
            rings[r].wait(0)
        assert int(rings[0].outcome[0][0]["consumed"]) == len(conns[0][1])
    half = len(keys) // 2
    tick([("resp", b"".join(_throttle(x.decode(), 1, 1, 60, 5) for x in keys[:half]), None),
          ("resp", b"".join(_throttle(x.decode(), 1, 1, 60, 5) for x in keys[half:]), None)])
    names = lims[0].store.denied_names(hs)
    unknown = sum(nm == tc.NAME_UNKNOWN for nm in names)
    assert unknown >= len(keys) - 1024
    assert all(nm == x for nm, x in zip(names, keys) if nm != tc.NAME_UNKNOWN)
    named = [h for h, nm in zip(hs, names) if nm != tc.NAME_UNKNOWN]
    unnamed = [h for h, nm in zip(hs, names) if nm == tc.NAME_UNKNOWN]
    # a key left out, denied 3 times more: `full` counts denied rows, not keys (its probes meet the same full entries)
    hot = keys[hs.index(unnamed[0])].decode()
    tick([("resp", _throttle(hot, 1, 1, 60, 5) * 3, None)])
    assert lims[0].store.denied_names([unnamed[0]]) == [tc.NAME_UNKNOWN]
    kept = named[:10] + unnamed[:5]
    assert lims[0].store.ring_names_keep(kept) == unknown + 3
    assert lims[0].store.denied_names(hs) == [x if h in set(named[:10]) else tc.NAME_UNKNOWN for h, x in zip(hs, keys)]
    tick([("resp", b"".join(_throttle(x, 1, 1, 60, 5) for x in ("n:1", "n:2", "L" * 300)), None)])
    new = [lims[0].store.hash_key(x) for x in (b"n:1", b"n:2", b"L" * 300)]
    assert lims[0].store.denied_names(new) == [b"n:1", b"n:2", tc.NAME_TOO_LONG]
    assert lims[0].store.ring_names_keep([]) == 0
    assert lims[0].store.denied_names(new + named[:10]) == [tc.NAME_UNKNOWN] * 13


def scenario_refusals(world, gpus):
    """both refusal orders between the two metrics modes, max_keys above 10,000, a keep while off, a switch between a
    slot's route and its finish: each leaves
    the engines as they were, and they then serve ticks with counts and names"""
    rng, nrng = random.Random(77), np.random.default_rng(77)
    lims, rings = engines(world, SIP, gpus=gpus, row_cap=400, cap_rows=1024)
    key_of = {lims[0].store.hash_key(k.encode()): k.encode() for k in KEYS}
    _refused(lambda: lims[0].store.ring_names_keep([]))                         # off
    rings[0].peer_memory(False)
    lims[0].store.ring_metrics(True)
    _refused(lambda: lims[0].store.ring_metrics_sharded(True, 10))
    lims[0].store.ring_metrics(False)
    for lim in lims:
        _refused(lambda: lim.store.ring_metrics_sharded(True, 10_001))
        lim.store.ring_metrics_sharded(True, 10_000)
        _refused(lambda: lim.store.ring_metrics(True))
        _refused(lambda: lim.store.ring_metrics_sharded(True, 10_001))           # (on stays on, with its table)
    rings[0].peer_memory(True)                                                   # accepted in this mode
    # between a slot's route and its finish no switch is taken: the route chose whether key positions are written
    for ring in rings:
        ring.submit_route(1, 0, NOW)
    _refused(lambda: lims[0].store.ring_metrics_sharded(True, 10))
    _refused(lambda: lims[0].store.ring_metrics_sharded(False, 0))
    for ring in rings:
        ring.submit_finish(1)
    for ring in rings:
        ring.wait(1)
    ora, counts, through, seen, _ = drive(lims, rings, 3, rng, nrng)
    for r in range(world):
        assert (lims[r].store.ring_transport_counts() == counts[r]).all()
        check_names(lims[r], r, seen, through[r], key_of)
    assert lims[0].store.ring_names_keep(sorted(through[0])) == 0
    check_names(lims[0], 0, seen, through[0], key_of)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("scenario")
    ap.add_argument("world", type=int)
    ap.add_argument("--gpus", action="store_true", help="engine r on GPU r")
    a = ap.parse_args()
    if a.scenario == "world1_text":
        scenario_world1_text()
    elif a.scenario in ("counts", "driver", "prune", "full", "refusals"):
        globals()["scenario_" + a.scenario](a.world, a.gpus)
    else:
        raise SystemExit("unknown scenario " + a.scenario)
    print("sharded ring metrics ok: %s, world %d" % (a.scenario, a.world))


if __name__ == "__main__":
    main()
