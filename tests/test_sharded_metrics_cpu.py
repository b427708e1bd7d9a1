"""metrics.ShardedMetrics over fake ranks (no device): summed counts, the order names are taken in, the keep set of
gcra_top_denied's pruning rule, one rank's text equal to Metrics'; the sharded driver's metrics check; the header."""
import os
import re

import numpy as np
import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import _native, mixed
from throttlecrab_b200.metrics import Metrics, ShardedMetrics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class FakeStore:
    """a rank's engine as the metrics see it: ring counts, a denied table (hash -> count) pruned by gcra_top_denied's
    rule, and ring names by hash"""

    def __init__(self, counts=None, denied=None, names=None):
        self.counts = np.asarray(counts if counts is not None else np.zeros((3, 3)), np.uint64)
        self.denied, self.ring_names = dict(denied or {}), dict(names or {})
        self.max_keys, self.calls, self.kept = None, [], None

    def track_denied(self, k):
        self.max_keys = k

    def ring_metrics(self, on):
        self.calls.append(("ring_metrics", on))

    def ring_metrics_sharded(self, on, k):
        self.calls.append(("ring_metrics_sharded", on, k))

    def ring_transport_counts(self):
        return self.counts

    def hash_key(self, kb):
        return tc.hash_key(kb)

    def top_denied(self, k):
        top = sorted(self.denied.items(), key=lambda hc: (-hc[1], hc[0]))
        if len(top) > 3 * self.max_keys:
            self.denied = dict(top[:self.max_keys])
            self.ring_names = {h: n for h, n in self.ring_names.items() if h in self.denied}
        return top[:k], 0

    def denied_names(self, hashes):
        return [self.ring_names.get(h, tc.NAME_UNKNOWN) for h in hashes]

    def ring_names_keep(self, hashes):
        self.kept = list(hashes)
        self.ring_names = {h: n for h, n in self.ring_names.items() if h in set(hashes)}
        return 3


class FakeLimiter:
    def __init__(self, store):
        self.store = store


def _mask(text):
    return re.sub(r"throttlecrab_uptime_seconds \d+\n", "throttlecrab_uptime_seconds U\n", text)


def test_switches_every_rank_and_sums_counts():
    a = FakeStore(counts=[[1, 2, 0], [3, 4, 5], [6, 7, 8]])
    b = FakeStore(counts=[[10, 0, 0], [0, 20, 1], [0, 0, 30]])
    m = ShardedMetrics([FakeLimiter(a), FakeLimiter(b)], 20_000)
    assert m.max_denied_keys == 10_000
    for s in (a, b):
        assert s.max_keys == 10_000 and s.calls == [("ring_metrics_sharded", True, 10_000)]
    m.record_request("http", False, "k")
    m.record_error("grpc")
    assert m.counts() == [[11, 2, 0], [3, 25, 6], [6, 7, 39]]
    assert m.names == {tc.hash_key(b"k"): b"k"}


def test_names_come_from_any_rank_then_the_host():
    h = {k: tc.hash_key(k) for k in (b"a", b"b", b"c", b"long", b"none", b"host")}
    # the denied counts on their owners (disjoint), the names wherever the connections were
    a = FakeStore(denied={h[b"a"]: 9, h[b"long"]: 8, h[b"host"]: 2}, names={h[b"b"]: b"b", h[b"long"]: b"long"})
    b = FakeStore(denied={h[b"b"]: 7, h[b"c"]: 5, h[b"none"]: 4},
                  names={h[b"a"]: b"a", h[b"long"]: tc.NAME_TOO_LONG, h[b"c"]: b"c"})
    m = ShardedMetrics([FakeLimiter(a), FakeLimiter(b)], 10)
    m.names[h[b"host"]] = b"host"
    m.names[h[b"c"]] = b"not this"                              # (a ring's name comes first)
    assert m.top_denied_keys() == [("a", 9), ("b", 7), ("c", 5), ("host", 2)]
    assert m.full == 6                                          # (3 per rank)
    # nothing pruned: every rank keeps every hash of every list
    assert a.kept == b.kept == sorted(h.values())


def test_keep_set_follows_each_owners_pruning():
    k = 2
    a_den = {1000 + i: 100 - i for i in range(7)}               # 7 > 3 x 2: a keeps its top 2
    b_den = {2000 + i: 50 - i for i in range(6)}                # 6 = 3 x 2: b keeps all 6
    names = {hh: b"n%d" % hh for hh in list(a_den) + list(b_den)}
    a, b = FakeStore(denied=a_den, names=names), FakeStore(denied=b_den, names=names)
    m = ShardedMetrics([FakeLimiter(a), FakeLimiter(b)], k)
    m.names = {1005: b"x", 2005: b"y", 9: b"z"}
    assert m.top_denied_keys() == [("n1000", 100), ("n1001", 99)]
    want = sorted([1000, 1001] + list(b_den))
    assert a.kept == b.kept == want
    assert m.names == {2005: b"y"}


def test_no_top_keys_with_max_denied_keys_0():
    a = FakeStore(denied={1: 5}, names={1: b"x"})
    m = ShardedMetrics([FakeLimiter(a)], 0)
    assert m.top_denied_keys() == [] and a.kept is None
    assert "top_denied_keys" not in m()


def test_one_rank_text_equals_metrics():
    h = {k: tc.hash_key(k) for k in (b"a", b'q"\\', b"long", b"host", b"none")}
    den = {h[b"a"]: 5, h[b'q"\\']: 5, h[b"long"]: 3, h[b"host"]: 2, h[b"none"]: 1}
    names = {h[b"a"]: b"a", h[b'q"\\']: b'q"\\', h[b"long"]: tc.NAME_TOO_LONG}
    counts = [[4, 1, 0], [2, 3, 1], [0, 5, 2]]
    one, two = FakeStore(counts, den, names), FakeStore(counts, den, names)
    m, sm = Metrics(FakeLimiter(one), 3), ShardedMetrics([FakeLimiter(two)], 3)
    for x in (m, sm):
        x.record_request("redis", False, "host")
        x.record_request("http", True)
        x.start = 0.0
    assert _mask(sm()) == _mask(m())
    assert 'key="q\\"\\\\"' in sm()


def test_driver_accepts_only_a_sharded_metrics_of_its_ranks():
    lims = [FakeLimiter(FakeStore()), FakeLimiter(FakeStore())]
    for bad in (print, lambda: "", Metrics(lims[0]), ShardedMetrics(lims[:1]), ShardedMetrics(lims[::-1])):
        with pytest.raises(ValueError):
            mixed.process_connections_sharded([([], lim, None) for lim in lims], 0, metrics=bad)


def test_header_declares_the_calls():
    src = open(os.path.join(ROOT, "include", "gcra_b200.h")).read()
    assert "int32_t gcra_ring_metrics_sharded(gcra_engine *h, uint32_t on, uint32_t max_keys);" in src
    assert "int32_t gcra_ring_names_keep(gcra_engine *h, uint32_t n, const uint64_t *key_hashes, uint64_t *full);" in src
    for name in ("gcra_ring_metrics_sharded", "gcra_ring_names_keep"):
        assert name in _native.SYMBOLS
