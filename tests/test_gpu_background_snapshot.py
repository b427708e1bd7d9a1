"""gcra_snapshot_begin / _poll / _wait: a background save whose cut is the call's place in submission order, written as
a version 3 file (the carried entries only) while traffic continues.  Every comparison is bit-exact against the oracle;
"the oracle at the cut" is a second oracle store that replayed only the batches submitted before begin."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import oracle
import throttlecrab_b200 as tc
import traces
from gpu_util import engine_requests, first_mismatch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
S = 10**9
P3 = tuple(int(x) for x in traces.POLICIES[3])      # (5, 10, 60)

# the file: SnapshotHeader (gcra_b200.cu), then version 2: keys | (tat, off) | ei of every slot; version 3: n, then
# the same sections of the n carried entries
HDR = np.dtype([("magic", "S8"), ("version", "<u4"), ("total_lines", "<u4"), ("nb_main", "<u4"), ("stash_slots", "<u4"),
                ("capacity", "<u8"), ("counters", "<u8", (16,)), ("hash_seed", "<u8", (2,))])
EXP_AT_MAX = np.int64(-2**63)                        # has_state: expiry >= 0, or the saturated code


def read_snapshot(path):
    """(header, keys, state [n, 2] int64, ei) of a version 2 or 3 file, the sections as stored"""
    raw = open(path, "rb").read()
    hd = np.frombuffer(raw, HDR, 1)[0]
    off = HDR.itemsize
    if hd["version"] == 2:
        n = int(hd["total_lines"]) * 4
    else:
        n = int(np.frombuffer(raw, "<u8", 1, off)[0])
        off += 8
        assert len(raw) == HDR.itemsize + 8 + 32 * n
    keys = np.frombuffer(raw, "<u8", n, off)
    state = np.frombuffer(raw, "<i8", 2 * n, off + 8 * n).reshape(n, 2)
    ei = np.frombuffer(raw, "<i8", n, off + 24 * n)
    return hd, keys, state, ei


def carried(keys, state):
    exp = (state[:, 0].astype(np.uint64) + state[:, 1].astype(np.uint64)).astype(np.int64)
    return (keys >= 2) & ((exp >= 0) | (exp == EXP_AT_MAX))


def assert_v3_is_filtered_v2(v2, v3):
    h2, k2, s2, e2 = read_snapshot(v2)
    h3, k3, s3, e3 = read_snapshot(v3)
    assert h2["version"] == 2 and h3["version"] == 3
    for f in ("magic", "total_lines", "nb_main", "stash_slots", "capacity"):
        assert h2[f] == h3[f], f
    assert (h2["counters"] == h3["counters"]).all() and (h2["hash_seed"] == h3["hash_seed"]).all()
    m = carried(k2, s2)
    assert (k3 == k2[m]).all() and (s3 == s2[m]).all() and (e3 == e2[m]).all()
    return int(m.sum())


def _oracle(n_keys):
    return oracle.OracleStore(oracle.PERIODIC, capacity=n_keys, created_ns=traces.T0, p0=10**9)


def _engine(capacity, max_batch=1 << 16, **kw):
    return tc.RateLimiter(tc.ManualStore(capacity=capacity, created_ns=traces.T0, max_batch=max_batch, **kw))


def _run(lim, req):
    return lim.rate_limit_batch(engine_requests(req))


def _totals(res):
    ok = res["status"] == tc.OK
    return int((ok & (res["allowed"] != 0)).sum()), int((ok & (res["allowed"] == 0)).sum()), int((~ok).sum())


def _save_v3(lim, path):
    lim.store.save_begin(path)
    return lim.store.save_wait()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("j", [2, 5])
def test_the_cut_is_the_calls_place_in_submission_order(j, tmp_path, k1_path):
    """Ticks alternate between the pinned ring and submit_device, pipelined, never joined; the save begins right after
    tick j, a Store-trait CAS right after it.  Ticks of 2^15 rows take the index-order pipeline in auto and index modes,
    so tick j's tail may still be in flight at the call."""
    n_keys, tick, n_ticks = 30_000, 1 << 15, 8
    warm = traces.warm_pass(n_keys)
    ticks = [warm] + np.split(traces.config4(n_keys=n_keys, n_ticks=n_ticks, tick_size=tick, hot=20), n_ticks)
    lim = _engine(n_keys, max_batch=tick)
    ring = tc.Ring(lim, len(ticks), tick)
    dev = torch.device("cuda", 0)
    ora, ora_cut = _oracle(n_keys), _oracle(n_keys)
    want, keep = [], []
    path = str(tmp_path / "bg.gcra")
    cas_key, cas_now = "k:%d" % int(ticks[j + 2]["key"][0]), int(ticks[j + 1]["now_ns"][-1])
    for i, t in enumerate(ticks):
        rows = engine_requests(t)
        if i % 2 == 0:
            ring.req[i][:len(t)] = rows
            ring.submit(i, len(t))
            keep.append(("ring", i, len(t)))
        else:
            q = torch.from_numpy(rows.view(np.uint8)).to(dev)
            r = torch.empty(len(t) * 32, dtype=torch.uint8, device=dev)
            lim.submit_device(len(t), q.data_ptr(), r.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
            keep.append(("dev", q, r))
        want.append(ora.replay(t))
        if i == j + 1:                                 # ticks[0] is the warm pass: body tick j is ticks[j + 1]
            ora_cut.replay(np.concatenate(ticks[:i + 1]))
            lim.store.save_begin(path)
            v = ora.get(cas_key, cas_now)
            assert lim.store.get(cas_key, cas_now) == v
            if v is not None:
                assert lim.store.compare_and_swap_with_ttl(cas_key, v, v + 1000, 60 * S, cas_now) is True
                assert ora.compare_and_swap_with_ttl(cas_key, v, v + 1000, 60 * S, cas_now) is True
    entries = lim.store.save_wait()
    lim.join()
    torch.cuda.synchronize()
    for i, (w, k) in enumerate(zip(want, keep)):
        if k[0] == "ring":
            ring.wait(k[1])
            got = ring.res[k[1]][:k[2]].copy()
        else:
            got = k[2].cpu().numpy().view(tc.RES_DTYPE)
        bad = first_mismatch(w, got, ticks[i])
        assert bad is None, "tick %d: %s" % (i, bad)
    assert entries == ora_cut.len()

    b = _engine(100, max_batch=tick)
    b.store.load(path)
    assert b.store.len() == ora_cut.len()
    h = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64))
    for k in range(n_keys):
        assert b.store.peek(int(h[k])) == ora_cut.entry("k:%d" % k), k
    s = b.store.stats()
    assert (s["allowed"], s["denied"], s["errors"]) == _totals(np.concatenate(want[:j + 2]))
    assert s["occupied_slots"] == s["len"]

    two = [_engine(100, max_batch=tick) for _ in range(2)]
    got = [e.store.restore(path, r, 2)[0] for r, e in enumerate(two)]
    assert sum(got) == ora_cut.len() == sum(e.store.len() for e in two)
    L = tc._native.lib()
    for k in np.random.default_rng(7).choice(n_keys, 2000, replace=False):
        o = L.gcra_owner_of(int(h[k]), 2)
        assert two[o].store.peek(int(h[k])) == ora_cut.entry("k:%d" % k), int(k)
        assert two[1 - o].store.peek(int(h[k])) is None, int(k)
    more = traces.config4(n_keys=n_keys, n_ticks=2, tick_size=tick, start_tick=n_ticks, hot=20)
    bad = first_mismatch(ora_cut.replay(more), _run(b, more), more)
    assert bad is None, bad


def _swept_and_denied(n_keys, **kw):
    """An engine holding live entries, expired-unswept entries, swept keys and keys only ever denied"""
    lim = _engine(4 * n_keys, **kw)
    ora = _oracle(n_keys)
    warm = traces.warm_pass(n_keys)
    assert first_mismatch(ora.replay(warm), _run(lim, warm)) is None
    assert lim.store.sweep(traces.T0 + 6 * S) == ora.force_sweep(traces.T0 + 6 * S) == n_keys // 2
    denied = np.zeros(1000, traces.REQ_DTYPE)
    denied["key"] = np.arange(n_keys, n_keys + 1000, dtype=np.uint64)
    denied["max_burst"], denied["count_per_period"], denied["period"] = P3
    denied["quantity"] = 10
    denied["now_ns"] = traces.T0 + 7 * S
    res = _run(lim, denied)
    assert first_mismatch(ora.replay(denied), res) is None and res["allowed"].sum() == 0
    return lim, ora


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_v3_is_the_filtered_v2(tmp_path, k1_path):
    n_keys = 8000
    lim, ora = _swept_and_denied(n_keys)
    s = lim.store.stats()
    assert s["occupied_slots"] == n_keys + 1000 and s["len"] == n_keys // 2
    v2, v3 = str(tmp_path / "a.v2"), str(tmp_path / "a.v3")
    lim.store.save(v2)
    assert _save_v3(lim, v3) == n_keys // 2 == assert_v3_is_filtered_v2(v2, v3)
    # at T0 + 30 s some carried entries have expired unswept: they are still carried
    b = _engine(100)
    b.store.load(v3)
    assert b.store.sweep(traces.T0 + 30 * S) == ora.force_sweep(traces.T0 + 30 * S) == n_keys // 4

    # empty table
    e = _engine(1000)
    e.store.save(v2)
    assert _save_v3(e, v3) == 0 == assert_v3_is_filtered_v2(v2, v3)
    assert os.path.getsize(v3) == HDR.itemsize + 8

    # seeded engine
    seed = (0x0123456789ABCDEF, 0xFEDCBA9876543210)
    sd = tc.RateLimiter(tc.ManualStore(capacity=1000, created_ns=traces.T0, hash_seed=seed))
    req = np.zeros(300, tc.REQ_DTYPE)
    req["key_hash"] = [sd.store.hash_key(b"user:%d" % i) for i in range(300)]
    req["max_burst"], req["count_per_period"], req["period"] = P3
    req["quantity"], req["now_ns"] = 1, traces.T0
    sd.rate_limit_batch(req)
    sd.store.save(v2)
    assert _save_v3(sd, v3) == 300 == assert_v3_is_filtered_v2(v2, v3)
    c = _engine(100)
    c.store.load(v3)
    assert c.store.hash_seed() == seed and c.store.len() == 300


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_v3_of_a_tight_table_with_stash_after_growth(tmp_path, k1_path):
    n_keys = 19_000
    trace = np.concatenate([traces.warm_pass(n_keys), traces.config4(n_keys=n_keys, n_ticks=1, tick_size=1 << 15, hot=20)])
    ora = _oracle(n_keys)
    ora.replay(trace)
    a = _engine(16, flags=tc._native.FLAG_TIGHT_TABLE)
    _run(a, trace)
    s = a.store.stats()
    assert s["grows"] > 0 and s["stash_entries"] > 0, s
    v2, v3 = str(tmp_path / "a.v2"), str(tmp_path / "a.v3")
    a.store.save(v2)
    assert _save_v3(a, v3) == n_keys == assert_v3_is_filtered_v2(v2, v3)
    b = _engine(16, flags=tc._native.FLAG_TIGHT_TABLE)
    b.store.load(v3)
    assert b.store.stats()["table_slots"] == s["table_slots"] and b.store.len() == n_keys
    more = traces.config4(n_keys=n_keys, n_ticks=2, tick_size=1 << 14, start_tick=1, hot=20)
    bad = first_mismatch(ora.replay(more), _run(b, more), more)
    assert bad is None, bad


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_load_and_restore_v3_and_refuse_malformed_files(tmp_path, k1_path):
    n_keys = 3000
    trace = np.concatenate([traces.warm_pass(n_keys), traces.config4(n_keys=n_keys, n_ticks=1, tick_size=1 << 15, hot=20)])
    ora = _oracle(n_keys)
    ora.replay(trace)
    a = _engine(n_keys)
    _run(a, trace)
    path = str(tmp_path / "a.gcra")
    assert _save_v3(a, path) == n_keys
    raw = open(path, "rb").read()
    bad_files = {"truncated": raw[:-4096], "magic": b"X" + raw[1:], "count": raw[:HDR.itemsize] +
                 np.uint64(n_keys - 1).tobytes() + raw[HDR.itemsize + 8:], "short": raw[:HDR.itemsize + 4]}
    for name, data in bad_files.items():
        (tmp_path / name).write_bytes(data)
    b = _engine(100)                                   # another geometry: load replaces the table by the file's
    b.store.restore(path, 0, 2)
    before = b.store.stats()
    for name in bad_files:
        for op in (lambda p: b.store.load(p), lambda p: b.store.restore(p)):
            with pytest.raises(tc.Internal):
                op(str(tmp_path / name))
            s = b.store.stats()
            assert (s["len"], s["table_slots"], s["occupied_slots"]) == (before["len"], before["table_slots"],
                                                                        before["occupied_slots"]), name
    b.store.restore(path, 1, 2)
    c = _engine(100)
    c.store.load(path)
    assert c.store.stats()["table_slots"] == a.store.stats()["table_slots"] and c.store.len() == n_keys
    more = traces.config4(n_keys=n_keys, n_ticks=2, tick_size=1 << 14, start_tick=1, hot=20)
    want = ora.replay(more)
    for e in (b, c):
        bad = first_mismatch(want, _run(e, more), more)
        assert bad is None, bad


def _shifted(req, by):
    req = req.copy()
    req["key"] += np.uint64(by)
    return req


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_load_refuses_malformed_v2_files_and_round_trips_good_ones(tmp_path, k1_path):
    """A version 2 file of engine A, malformed four ways, loaded into an engine of A's geometry that holds other
    entries and into one of another geometry: each load is refused and leaves the engine's stats and its next
    decisions as they were.  The good file, loaded into either engine and saved again, comes back byte for byte."""
    n_keys, cap, tick = 3000, 1 << 16, 1 << 12        # (cap: room for every row of a batch, so that no batch grows it)
    a = _engine(cap)
    _run(a, np.concatenate([traces.warm_pass(n_keys), traces.config4(n_keys=n_keys, n_ticks=1, tick_size=1 << 15, hot=20)]))
    path = str(tmp_path / "a.v2")
    a.store.save(path)
    raw = open(path, "rb").read()
    slots = a.store.stats()["table_slots"]
    assert len(raw) == HDR.itemsize + 32 * slots
    bad_files = {"truncated in ei": raw[:-4096], "truncated in keys": raw[:HDR.itemsize + 8 * (slots // 2)],
                 "magic": b"X" + raw[1:], "trailing byte": raw + b"\0"}
    for i, (name, data) in enumerate(bad_files.items()):
        (tmp_path / ("bad%d" % i)).write_bytes(data)
    # (engine, its oracle, its key universe: the keys of the trace shifted by `shift`)
    engines = [(_engine(cap), _oracle(n_keys), n_keys, n_keys),        # A's geometry, other entries
               (_engine(100), _oracle(50), 50, 10 * n_keys)]           # another geometry
    for e, ora, n, shift in engines:
        t = _shifted(np.concatenate([traces.warm_pass(n), traces.config4(n_keys=n, n_ticks=1, tick_size=tick, hot=20)]), shift)
        assert first_mismatch(ora.replay(t), _run(e, t), t) is None
    assert engines[0][0].store.stats()["table_slots"] == slots != engines[1][0].store.stats()["table_slots"]
    keys = ("len", "table_slots", "occupied_slots", "stash_entries")
    for k, (e, ora, n, shift) in enumerate(engines):
        for i, name in enumerate(bad_files):
            before = e.store.stats()
            with pytest.raises(tc.Internal):
                e.store.load(str(tmp_path / ("bad%d" % i)))
            s = e.store.stats()
            assert [s[f] for f in keys] == [before[f] for f in keys], (k, name)
            more = _shifted(traces.config4(n_keys=n, n_ticks=1, tick_size=tick, start_tick=1 + i, hot=20), shift)
            bad = first_mismatch(ora.replay(more), _run(e, more), more)
            assert bad is None, (k, name, bad)
        e.store.load(path)
        again = str(tmp_path / ("again%d" % k))
        e.store.save(again)
        assert open(again, "rb").read() == raw, k


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_errors_and_lifecycle(tmp_path, k1_path):
    n_keys, tick = 20_000, 1 << 15
    lim = _engine(n_keys, max_batch=tick)
    ora = _oracle(n_keys)
    ticks = [traces.warm_pass(n_keys)] + np.split(traces.config4(n_keys=n_keys, n_ticks=24, tick_size=tick, hot=20), 24)
    good = str(tmp_path / "good.gcra")
    assert _save_v3(lim, good) == 0
    good_bytes = open(good, "rb").read()
    assert lim.store.save_poll() is True
    for i, t in enumerate(ticks[:4]):
        assert first_mismatch(ora.replay(t), _run(lim, t)) is None
    # a second begin while the first is in flight (its writer still has to fsync): refused, the first completes
    lim.store.save_begin(str(tmp_path / "first.gcra"))
    with pytest.raises(tc.Internal, match="in flight"):
        lim.store.save_begin(str(tmp_path / "second.gcra"))
    assert lim.store.save_wait() == ora.len()
    assert os.path.exists(str(tmp_path / "first.gcra")) and not os.path.exists(str(tmp_path / "second.gcra"))
    # a missing directory: begin fails, nothing is written, traffic continues exactly
    with pytest.raises(tc.Internal):
        lim.store.save_begin(str(tmp_path / "missing" / "x.gcra"))
    assert not os.path.exists(str(tmp_path / "missing"))
    assert first_mismatch(ora.replay(ticks[4]), _run(lim, ticks[4])) is None
    # a failed begin leaves the good file at the path untouched (a directory this user cannot write to)
    if os.geteuid() != 0:
        ro = tmp_path / "ro"
        ro.mkdir()
        (ro / "good.gcra").write_bytes(good_bytes)
        ro.chmod(0o555)
        try:
            with pytest.raises(tc.Internal):
                lim.store.save_begin(str(ro / "good.gcra"))
            assert (ro / "good.gcra").read_bytes() == good_bytes and os.listdir(str(ro)) == ["good.gcra"]
        finally:
            ro.chmod(0o755)
    # poll reports done only once the file is in place
    p = str(tmp_path / "polled.gcra")
    lim.store.save_begin(p)
    while not lim.store.save_poll():
        time.sleep(0.001)
    assert os.path.exists(p) and os.path.getsize(p) == HDR.itemsize + 8 + 32 * ora.len()
    assert not [f for f in os.listdir(str(tmp_path)) if ".tmp." in f]
    assert lim.store.save_wait() == ora.len()
    # 20 saves in a row (with the one above), interleaved with traffic
    for k, t in enumerate(ticks[5:24]):
        lim.store.save_begin(str(tmp_path / ("s%d.gcra" % (k % 2))))
        assert first_mismatch(ora.replay(t), _run(lim, t)) is None
        assert lim.store.save_wait() > 0
    # destroy right after begin: the file is complete and loadable
    d = str(tmp_path / "at_destroy.gcra")
    lim.store.save_begin(d)
    lim.store.close()
    b = _engine(100, max_batch=tick)
    b.store.load(d)
    assert b.store.len() == ora.len()
    more = ticks[24]
    assert first_mismatch(ora.replay(more), _run(b, more), more) is None


@pytest.mark.timeout(1500)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_full_size_background_save(tmp_path, k1_path):
    """The 10 M-key table (2^25 slots): a background save begins between 2^20-row ticks that keep coming."""
    n_keys, tick = 10_000_000, 1 << 20
    lim = _engine(n_keys, max_batch=tick)
    warm = traces.warm_pass(n_keys)
    body = np.split(traces.config4(n_keys=n_keys, n_ticks=4, tick_size=tick, hot=20), 4)
    pre = [warm[a:a + tick] for a in range(0, n_keys, tick)] + body[:1]
    for t in pre:
        lim.rate_limit_batch(engine_requests(t))
    ora_cut = _oracle(n_keys)
    ora_cut.replay(np.concatenate(pre))
    v2 = str(tmp_path / "full.v2")
    t0 = time.perf_counter()
    lim.store.save(v2)
    t_v2 = time.perf_counter() - t0
    dev = torch.device("cuda", 0)
    qs = [torch.from_numpy(engine_requests(t).view(np.uint8)).to(dev) for t in body[1:]]
    rs = [torch.empty(tick * 32, dtype=torch.uint8, device=dev) for _ in body[1:]]
    torch.cuda.synchronize()
    path = str(tmp_path / "full.gcra")
    t0 = time.perf_counter()
    lim.store.save_begin(path)
    t_begin = time.perf_counter() - t0
    for q, r in zip(qs, rs):
        lim.submit_device(tick, q.data_ptr(), r.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    lim.join()
    torch.cuda.synchronize()
    t_ticks = time.perf_counter() - t0
    entries = lim.store.save_wait()
    t_file = time.perf_counter() - t0
    assert entries == ora_cut.len() == n_keys
    assert os.path.getsize(path) == HDR.itemsize + 8 + 32 * n_keys
    b = _engine(1000, max_batch=tick)
    b.store.load(path)
    assert b.store.len() == n_keys
    h = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64))
    for k in np.random.default_rng(29).choice(n_keys, 20_000, replace=False):
        assert b.store.peek(int(h[k])) == ora_cut.entry("k:%d" % k), int(k)
    print("\nfull-size background save (%s): v2 %.3f GB blocking %.2f s; v3 %.3f GB, begin %.1f ms, 3 ticks %.3f s, "
          "file complete %.2f s" % (torch.cuda.get_device_name(0), os.path.getsize(v2) / 1e9, t_v2,
                                    os.path.getsize(path) / 1e9, t_begin * 1e3, t_ticks, t_file))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("src,dst,n_keys", [(2, 3, 54_000), (3, 1, 40_000), (4, 2, 40_000)])
def test_several_engines_save_without_a_join(src, dst, n_keys, tmp_path, k1_path):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")     # see test_gpu_sharded.py's loop-back test
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "background_snapshot_worker.py"),
                          str(src), str(dst), str(n_keys), str(tmp_path)],
                         capture_output=True, text=True, timeout=800, env=env)
    assert out.returncode == 0 and "background ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
