"""mixed.process_connections_sharded without a GPU: its rounds and its owner router, with the engines and rings
stubbed.  Every round submits one tick or more on every rank (all routes, then all finishes), the general paths decide
on the key's owner, and the joined result equals process_connections(ring=None) on one limiter over the joined list.
Also: the peer-memory ring calls are declared in the header."""
import os
import random
import re

import numpy as np
import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import mixed
from test_mixed_cpu import Limiter
from test_resp import _throttle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NS = 10**9
NOW = 1_700_000_000 * NS


class _Rank:
    """one engine of the sharded set: logs the general paths' rows it receives and decides them on the ranks' one
    table (`shared`, a test_mixed_cpu.Limiter)"""

    def __init__(self, log, r, shared):
        self.log, self.r, self.shared, self.store = log, r, shared, shared.store

    def rate_limit_batch(self, requests):
        self.log.append(("general", self.r, [int(k) for k in requests["key_hash"]]))
        return self.shared.rate_limit_batch(requests)


class _Ring:
    """a MixedRing stand-in: submit_route walks the slot's connections on the host (no RESP/HTTP row cap is reached
    here), submit_finish decides them on one shared store in route order, as a tick does"""

    def __init__(self, log, r, shared):
        self.log, self.r, self.shared = log, r, shared
        self.max_conns, self.in_capacity, self.row_capacity = 64, 1 << 20, 1 << 14
        self.input = [np.zeros(self.in_capacity, np.uint8)]
        self.conns = [np.zeros(self.max_conns, tc.MIXED_CONN_DTYPE)]
        self.grpc_conns = [np.zeros(self.max_conns, tc.GRPC_CONN_DTYPE)]
        self.outcome = [np.zeros(self.max_conns, tc.RESP_OUTCOME_DTYPE)]
        self.grpc_outcome = [np.zeros(self.max_conns, tc.GRPC_OUTCOME_DTYPE)]
        self.replies = [np.zeros(1 << 20, np.uint8)]
        self.p2p = False

    def peer_memory(self, on=True):
        self.p2p = on

    def submit_route(self, slot, n, now):
        assert self.p2p
        self.log.append(("route", self.r, n))
        self.n, self.now = n, now

    def submit_finish(self, slot):
        self.log.append(("finish", self.r))
        at = 0
        for j in range(self.n):
            c = self.conns[slot][j]
            assert c["protocol"] == tc.PROTO_RESP             # (the stub serves RESP connections only)
            data = self.input[slot][int(c["off"]):int(c["off"]) + int(c["len"])].tobytes()
            reply, used, k, stop = mixed.host_walk("resp", data, self.shared, self.now)
            self.replies[slot][at:at + len(reply)] = np.frombuffer(reply, np.uint8)
            self.outcome[slot][j] = (used, k, stop, 0, at, len(reply))
            at += len(reply)

    def wait(self, slot):
        pass


def _resp_conns(rng, tag, n):
    out = []
    for c in range(n):
        frames = [_throttle("%s%d" % (tag, rng.randrange(4)), 3, 10, 60) for _ in range(rng.randrange(0, 6))]
        if rng.random() < 0.4:
            frames.insert(rng.randrange(len(frames) + 1), b"*1\r\n$4\r\nPING\r\n")
        if c == 0 or rng.random() < 0.3:                   # (RESP integers: the general path decides it)
            frames.insert(rng.randrange(len(frames) + 1), b"*5\r\n$8\r\nTHROTTLE\r\n$2\r\nk9\r\n:3\r\n:10\r\n:60\r\n")
        out.append(("resp", b"".join(frames)))
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_rounds_and_router(world):
    rng = random.Random(world)
    log = []
    shared = Limiter()                                   # the ranks' one table
    lims = [_Rank(log, r, shared) for r in range(world)]
    rings = [_Ring(log, r, shared) for r in range(world)]
    per = [_resp_conns(rng, "k", rng.randrange(0, 8)) for _ in range(world)]
    per[0] += _resp_conns(rng, "k", 3)
    joined = [c for cs in per for c in cs]
    got = mixed.process_connections_sharded([(cs, lim, ring) for cs, lim, ring in zip(per, lims, rings)], NOW)
    assert [len(g) for g in got] == [len(cs) for cs in per]
    assert [x for g in got for x in g] == mixed.process_connections(joined, Limiter(), NOW, None)
    # every tick: all routes, then all finishes, in rank order
    ticks = [e for e in log if e[0] in ("route", "finish")]
    assert len(ticks) % (2 * world) == 0 and ticks
    for a in range(0, len(ticks), 2 * world):
        assert [e[:2] for e in ticks[a:a + 2 * world]] == \
            [("route", r) for r in range(world)] + [("finish", r) for r in range(world)]
    # the general paths' Throttles went to their keys' owners
    L = tc._native.lib()
    for e in log:
        if e[0] == "general":
            assert all(L.gcra_owner_of(k, world) == e[1] for k in e[2])
    assert any(e[0] == "general" for e in log)


def test_a_round_with_nothing_ready_still_ticks_every_rank():
    """a round ticks every rank even when no rank has a ready connection (a tick of 0 rows each)"""
    log = []
    shared = Limiter()
    rings = [_Ring(log, r, shared) for r in range(3)]
    conns = [("resp", b"*1\r\n$4\r\nPING\r\n")]
    mixed.process_connections_sharded([([], _Rank(log, 0, shared), rings[0]), (conns, _Rank(log, 1, shared), rings[1]),
                                       ([], _Rank(log, 2, shared), rings[2])], NOW)
    assert [e for e in log if e[0] == "route"] == [("route", 0, 0), ("route", 1, 1), ("route", 2, 0)]


@pytest.mark.parametrize("max_conns", [1, 2, 3])
def test_a_rank_that_needs_more_ticks_keeps_the_joined_order(max_conns):
    """a rank whose ready connections need more than one tick leaves the later ranks empty until it is through, so the
    rows go through the ticks in the joined order, as on one engine"""
    rng = random.Random(max_conns)
    log = []
    shared = Limiter()
    rings = [_Ring(log, r, shared) for r in range(3)]
    for ring in rings:
        ring.max_conns = max_conns
    per = [[("resp", _throttle("s%d" % rng.randrange(3), 3, 10, 60) * rng.randrange(1, 4)) for _ in range(n)]
           for n in (5, 3, 4)]
    got = mixed.process_connections_sharded([(cs, _Rank(log, r, shared), ring)
                                             for r, (cs, ring) in enumerate(zip(per, rings))], NOW)
    joined = [c for cs in per for c in cs]
    assert [x for g in got for x in g] == mixed.process_connections(joined, Limiter(), NOW, None)
    routes = [e for e in log if e[0] == "route"]
    assert routes[:3] == [("route", 0, max_conns), ("route", 1, 0), ("route", 2, 0)]


def test_metrics_refused():
    with pytest.raises(ValueError):
        mixed.process_connections_sharded([], NOW, metrics=lambda: "")


def test_header_declares_the_ring_p2p_calls():
    src = open(os.path.join(ROOT, "include", "gcra_b200.h")).read()
    for name in ("gcra_ring_p2p", "gcra_resp_ring_submit_route", "gcra_resp_ring_submit_finish"):
        assert re.search(r"\bint32_t %s\(gcra_engine \*h" % name, src), name
