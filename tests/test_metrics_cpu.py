"""throttlecrab_b200.metrics without a GPU: the Prometheus text of metrics.rs:233-310 byte for byte, its label escaping,
the max_denied_keys clamp, the reference's metrics tests (metrics.rs:327-412, tests/metrics_test.rs,
tests/denied_keys_test.rs) restated, and what the general paths of the drivers record.  A model store stands in for
the engine: its denied-key table counts the denials of the batches it decides (as gcra_track_denied does), and its
ring counts and ring-given names are set by hand."""
import re

import numpy as np
import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import grpc_transport as gt
from throttlecrab_b200 import metrics as mx
from throttlecrab_b200 import mixed, resp
from throttlecrab_b200.metrics import Metrics, escape_label
from test_resp import NOW, OracleEngine, _cmd, _throttle


class ModelStore:
    """what Metrics needs of an engine: denied tracking (a count per key hash, ties by smaller hash), ring counts and
    ring names"""

    def __init__(self):
        self.max_keys, self.on = None, False
        self.gpu = np.zeros((3, 3), np.uint64)
        self.table, self.gpu_names = {}, {}
        self.eng = OracleEngine()

    def _check(self, rc):
        assert rc == 0

    def hash_seed(self):
        return (0, 0)

    def hash_key(self, kb):
        return tc.hash_key(kb)

    def track_denied(self, max_keys):
        self.max_keys, self.table = max_keys, {}

    def ring_metrics(self, on):
        self.on = on

    def ring_transport_counts(self):
        return self.gpu.copy()

    def top_denied(self, k):
        top = sorted(self.table.items(), key=lambda e: (-e[1], e[0]))
        return top[:k], 0

    def denied_names(self, hashes):
        return [self.gpu_names.get(h, tc.NAME_UNKNOWN) for h in hashes]

    def deny(self, key):
        """a denial the engine decided (counted by its denied-key table)"""
        kb = key.encode() if isinstance(key, str) else key
        h = tc.hash_key(kb)
        self.table[h] = self.table.get(h, 0) + 1
        return h


class ModelLimiter:
    def __init__(self):
        from throttlecrab_b200 import _native
        self._L, self._h, self.store = _native.lib(), None, ModelStore()

    def rate_limit_batch(self, req):
        res = self.store.eng(req)
        for r, o in zip(req, res):
            if int(o["status"]) == tc.OK and not o["allowed"] and self.store.max_keys:
                h = int(r["key_hash"])
                self.store.table[h] = self.store.table.get(h, 0) + 1
        return res


def _metrics(max_denied_keys=100):
    lim = ModelLimiter()
    return Metrics(lim, max_denied_keys), lim.store


def _with_key(m, st, transport, allowed, key):
    """record_request_with_key as a server does it: the engine decided the request (and counted a denial)"""
    if not allowed:
        st.deny(key)
    m.record_request(transport, allowed, key)


def _mask(text):
    return re.sub(r"throttlecrab_uptime_seconds \d+\n", "throttlecrab_uptime_seconds U\n", text)


# ---- the text ---------------------------------------------------------------------------------------------------------
def test_export_text_matches_the_reference_format():
    m, st = _metrics()
    st.gpu[:] = [[5, 2, 0], [7, 1, 3], [0, 4, 1]]           # RESP, HTTP, gRPC x allowed, denied, errors
    m.record_request("redis", True)
    m.record_request("http", True, "ok")
    m.record_error("grpc")
    _with_key(m, st, "http", False, "host:key")
    for _ in range(3):
        st.gpu_names[st.deny("gpu:key")] = b"gpu:key"
    st.gpu_names[st.deny("x" * 300)] = tc.NAME_TOO_LONG
    st.deny("nameless")                                     # denied on a path that names nothing: left out
    want = ("# HELP throttlecrab_uptime_seconds Time since server start in seconds\n"
            "# TYPE throttlecrab_uptime_seconds gauge\n"
            "throttlecrab_uptime_seconds U\n\n"
            "# HELP throttlecrab_requests_total Total number of requests processed\n"
            "# TYPE throttlecrab_requests_total counter\n"
            "throttlecrab_requests_total 27\n\n"
            "# HELP throttlecrab_requests_by_transport Total requests by transport type\n"
            "# TYPE throttlecrab_requests_by_transport counter\n"
            'throttlecrab_requests_by_transport{transport="http"} 13\n'
            'throttlecrab_requests_by_transport{transport="grpc"} 6\n'
            'throttlecrab_requests_by_transport{transport="redis"} 8\n\n'
            "# HELP throttlecrab_requests_allowed Total requests allowed\n"
            "# TYPE throttlecrab_requests_allowed counter\n"
            "throttlecrab_requests_allowed 14\n\n"
            "# HELP throttlecrab_requests_denied Total requests denied\n"
            "# TYPE throttlecrab_requests_denied counter\n"
            "throttlecrab_requests_denied 8\n\n"
            "# HELP throttlecrab_requests_errors Total internal errors\n"
            "# TYPE throttlecrab_requests_errors counter\n"
            "throttlecrab_requests_errors 5\n\n"
            "# HELP throttlecrab_top_denied_keys Top keys by denial count\n"
            "# TYPE throttlecrab_top_denied_keys gauge\n"
            'throttlecrab_top_denied_keys{key="gpu:key",rank="1"} 3\n'
            'throttlecrab_top_denied_keys{key="host:key",rank="2"} 1\n')
    assert _mask(m.export_prometheus()) == want
    assert _mask(m()) == want
    assert re.search(r"throttlecrab_uptime_seconds 0\n", m())


@pytest.mark.parametrize("s,want", [
    ('"', '\\"'), ("\\", "\\\\"), ("\n", "\\n"), ("\r", "\\r"), ("\t", "\\t"), ("\x00", "\\x00"),
    ("\x01", "\\x01"), ("\x0b", "\\x0b"), ("\x1b", "\\x1b"), ("\x1f", "\\x1f"), ("\x7f", "\\x7f"),
    ("\x80", "\\x80"), ("\x85", "\\x85"), ("\x9f", "\\x9f"), ("\xa0", "\xa0"), (" ", " "), ("é", "é"),
    ("\u2028", "\u2028"), ('user:"a"\\b\tc', 'user:\\"a\\"\\\\b\\tc'), ("", "")])
def test_label_escaping(s, want):
    assert escape_label(s) == want


def test_escaped_key_in_the_text():
    m, st = _metrics()
    _with_key(m, st, "redis", False, 'q"\\\x01\x7f\x85é')
    assert 'throttlecrab_top_denied_keys{key="q\\"\\\\\\x01\\x7f\\x85é",rank="1"} 1\n' in m()


def test_max_denied_keys_clamp_and_zero():
    m, st = _metrics(20_000)
    assert m.max_denied_keys == 10_000 and st.max_keys == 10_000 and st.on
    m, st = _metrics(0)
    assert m.max_denied_keys == 0 and st.max_keys == 0
    for i in range(5):
        _with_key(m, st, "http", False, "user:%d" % i)
    out = m()
    assert "throttlecrab_top_denied_keys" not in out
    assert "throttlecrab_requests_denied 5\n" in out and out.endswith("throttlecrab_requests_errors 0\n\n")
    assert mx.MAX_DENIED_KEYS_LIMIT == tc.RING_METRICS_MAX_KEYS


# ---- the reference's tests ------------------------------------------------------------------------------------------
def test_reference_metrics_creation_and_record_request():          # metrics.rs:332-361
    m, _ = _metrics()
    assert m.counts() == [[0, 0, 0]] * 3
    m.record_request("http", True)
    assert m.counts()[1] == [1, 0, 0]
    m.record_request("grpc", False)
    c = m.counts()
    assert (c[1], c[2], sum(map(sum, c))) == ([1, 0, 0], [0, 1, 0], 2)


def test_reference_prometheus_export():                             # metrics.rs:363-380
    m, _ = _metrics()
    m.record_request("http", True)
    m.record_request("grpc", False)
    out = m()
    for s in ("throttlecrab_uptime_seconds", "throttlecrab_requests_total 2", "throttlecrab_requests_allowed 1",
              "throttlecrab_requests_denied 1", 'throttlecrab_requests_by_transport{transport="http"} 1',
              'throttlecrab_requests_by_transport{transport="grpc"} 1'):
        assert s in out


def test_reference_counter_consistency():                           # metrics.rs:382-411
    m, _ = _metrics()
    for t, a in (("http", True), ("http", False), ("grpc", True), ("grpc", False)):
        m.record_request(t, a)
    m.record_error("http")
    c = m.counts()
    assert sum(map(sum, c)) == 5 and sum(c[1]) + sum(c[2]) == 5
    assert [sum(r[j] for r in c) for j in range(3)] == [2, 2, 1]


def test_reference_top_denied_keys():                               # tests/metrics_test.rs:5-22
    m, st = _metrics()
    for allowed, key in ((False, "user:123"), (False, "user:123"), (False, "user:456"), (True, "user:789")):
        _with_key(m, st, "http", allowed, key)
    out = m()
    assert "throttlecrab_top_denied_keys" in out and "user:123" in out and "user:456" in out
    assert "user:789" not in out
    assert 'throttlecrab_top_denied_keys{key="user:123",rank="1"} 2\n' in out


def test_reference_request_counting():                              # tests/metrics_test.rs:24-39
    m, st = _metrics()
    for i in range(10):
        _with_key(m, st, "http", i >= 3, "test")
    out = m()
    for s in ("throttlecrab_requests_total 10", "throttlecrab_requests_allowed 7", "throttlecrab_requests_denied 3"):
        assert s in out


@pytest.mark.parametrize("limit,keys,most", [(None, 150, 100), (200, 250, 200), (20_000, 15_000, 10_000)])
def test_reference_configurable_denied_keys(limit, keys, most):      # tests/denied_keys_test.rs:4-34,69-85
    m, st = _metrics() if limit is None else _metrics(limit)
    for i in range(keys):
        _with_key(m, st, "http", False, "user:%d" % i)
    n = m().count("throttlecrab_top_denied_keys{")
    assert n == most


def test_reference_denied_keys_with_multiple_denials():             # tests/denied_keys_test.rs:36-67
    m, st = _metrics(10)
    for key, k in (("top_key", 10), ("medium_key", 5), ("low_key", 2)):
        for _ in range(k):
            _with_key(m, st, "http", False, key)
    for i in range(20):
        _with_key(m, st, "http", False, "single_%d" % i)
    out = m()
    assert 'key="top_key",rank="1"} 10\n' in out and 'key="medium_key",rank="2"} 5\n' in out
    assert 'key="low_key",rank="3"} 2\n' in out
    assert out.count("throttlecrab_top_denied_keys{") == 10


def test_reference_disabled_denied_keys_tracking():                 # tests/denied_keys_test.rs:87-104
    m, st = _metrics(0)
    for i in range(100):
        _with_key(m, st, "http", False, "user:%d" % i)
    out = m()
    assert "throttlecrab_top_denied_keys" not in out
    assert "throttlecrab_requests_total" in out and "throttlecrab_requests_denied 100" in out


def test_long_keys_are_never_named():
    m, st = _metrics()
    _with_key(m, st, "http", False, "k" * 257)
    _with_key(m, st, "http", False, "k" * 256)
    out = m()
    assert out.count("throttlecrab_top_denied_keys{") == 1 and 'key="%s"' % ("k" * 256) in out


# ---- the drivers' general paths -------------------------------------------------------------------------------------
def test_resp_general_path_records_as_process_command():
    lim = ModelLimiter()
    m = Metrics(lim)
    cmds = [_cmd("PING"), _cmd("QUIT2"), _cmd("THROTTLE", "k", 3, 10, 60), _throttle("neg", 3, 10, 60, -1),
            _cmd("THROTTLE", "short"), b"+not an array\r\n", b"*0\r\n", _cmd(5, "x")]
    for c in cmds:
        resp.general(c, lim, NOW, m)
    # counted: PING, the unknown command, the two THROTTLEs (the -ERR reply is allowed) and the argument error
    assert m.counts()[0] == [5, 0, 0]
    for _ in range(10):                                    # 5 at once with a burst of 1: denied
        resp.general(_throttle("hot", 1, 1, 60, 5), lim, NOW, m)
    a, d, e = m.counts()[0]
    assert (a, d, e) == (5, 10, 0)
    assert 'throttlecrab_top_denied_keys{key="hot",rank="1"} %d\n' % d in m()


def test_plain_callables_and_host_walks():
    lim = ModelLimiter()
    m = Metrics(lim)
    with pytest.raises(ValueError):
        mixed.process_connections([("resp", _cmd("PING"))], lim, 0, None, metrics=m)
    with pytest.raises(ValueError):
        gt.process_connections([gt.Connection()], lim, 0, None, metrics=m)
    got = mixed.process_connections([("http", b"GET /metrics HTTP/1.1\r\nHost: x\r\n\r\n")], lim, 0, None,
                                    metrics=lambda: "text")
    assert got[0][0].endswith(b"\r\n\r\ntext")
    assert m.counts() == [[0, 0, 0]] * 3
