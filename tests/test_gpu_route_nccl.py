"""The route kernels and the host-driven sharded ticks on ONE GPU.

`make_sharded` falls back to the native NCCL tick (gcra_shard_*) when the ranks cannot map each other's memory, and
ShardedLimiter (the torch.distributed tick) runs the same route kernels through gcra_route_partition and
gcra_route_unpermute.  Outside this file, route_scan_kernel, route_scatter_kernel and route_unpermute_kernel run only in
the 2-GPU cases of test_gpu_sharded.py and test_gpu_sharded_denied.py, which skip on one GPU.

1. gcra_route_partition / gcra_route_unpermute in this process against a numpy restatement of their contract: a
   stable partition by gcra_owner_of (np.argsort(owner, kind="stable")), per-owner counts and the source index of
   every output row.  Row counts around a 256-row tile and a 256-tile scan chunk (65536 rows) up to max_batch, 1 to 16
   shards, key sets that fill one shard, skip one, or give lane i of every warp shard i % n_shards, and rows past n of
   a shard no valid row uses.  Every output is surrounded by a sentinel that must stay.
2. ShardedLimiter with the real kernels over gloo (CUDA tensors), worlds 2-4, one process and one engine per rank,
   all on cuda:0 (route_nccl_worker.py): 9 ragged ticks back to back, one of them sending 1.25 x max_rows rows to
   one owner so that its decide is cut into two engine batches.  No kernel waits for another engine's kernel here,
   so engines of several processes can share the GPU.
3. The native tick at world 1 over a single-rank NCCL group (route_nccl_worker.py), then ShardedLimiter over that
   group.  NCCL refuses two ranks on one GPU, so the native tick's host logic at world >= 2 -- the per-peer send and
   receive offsets, and shard_issue_decide_return's loop over max_batch chunks (an owner receives at most max_rows <=
   max_batch rows at world 1) -- is covered only by the 2-GPU tests.

Parts 2 and 3 check every row against ONE oracle store fed the union trace in global order (tick by tick, rank 0's
rows first), the collective top_denied against a host count of the oracle's denied rows, and the engines' counters."""
import collections
import json
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import route_nccl_worker as w  # noqa: E402

MAX_SHARDS = 16                 # ROUTE_MAX_SHARDS
MAX_BATCH = 1 << 20
PAD = 256                       # rows of input past n (the rest of the last tile), and sentinel rows around outputs
SENT8 = 0xA5
SENT32 = int(np.array(0xA5A5A5A5, np.uint32).view(np.int32))


def test_owner_of_restatement_matches_the_library():
    """The numpy owner map that parts 1-3 build their expectations from is gcra_owner_of, at every shard count."""
    L = w.tc._native.lib()
    rng = np.random.default_rng(7)
    h = np.frombuffer(rng.bytes(8 * 100_000), np.uint64).copy()
    h[:4] = (0, 1, 2**64 - 1, 0xA24BAED4963EE407)
    for n in range(1, MAX_SHARDS + 1):
        want = np.fromiter((L.gcra_owner_of(int(x), n) for x in h), np.int64, len(h))
        got = w.owner_of(h, n)
        assert (got == want).all(), (n, int(np.argmax(got != want)))
        assert got.min() >= 0 and got.max() < n
    assert np.bincount(w.owner_of(h, 16), minlength=16).min() > 5000


# ------------------------------------------------------------------------------------------------- 1. route kernels
@pytest.fixture(scope="module")
def engine():
    st = w.tc.ManualStore(capacity=1000, device=0, created_ns=w.traces.T0, max_batch=MAX_BATCH)
    yield st
    st.close()
    torch.cuda.empty_cache()            # the 2^20-row buffers go back to the device for the tests that follow


class Keys:
    """random key hashes grouped by their owner at every shard count (one pool for the module), and a generator"""
    _by_owner = None

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        if Keys._by_owner is None:
            pool = np.frombuffer(np.random.default_rng(11).bytes(8 << 17), np.uint64)
            Keys._by_owner = {s: [pool[w.owner_of(pool, s) == o] for o in range(s)] for s in range(1, MAX_SHARDS + 1)}
        self.by_owner = Keys._by_owner

    def of(self, owners, s):
        """one key hash per row, each owned by owners[i] among s shards"""
        out = np.empty(len(owners), np.uint64)
        for o in np.unique(owners):
            idx = np.nonzero(owners == o)[0]
            cand = self.by_owner[s][o]
            out[idx] = cand[self.rng.integers(0, len(cand), len(idx))]
        return out


def key_sets(keys, n, s):
    """(name, n + PAD key hashes); rows past n are the padding of the last tile"""
    rng = keys.rng

    def pad(owner=None):
        if owner is None:
            return np.frombuffer(rng.bytes(8 * PAD), np.uint64)
        return keys.of(np.full(PAD, owner), s)
    uniform = np.frombuffer(rng.bytes(8 * n), np.uint64)
    yield "uniform", np.concatenate([uniform, pad()])
    yield "last_shard", np.concatenate([keys.of(np.full(n, s - 1), s), pad()])
    yield "shard_0", np.concatenate([keys.of(np.zeros(n, np.int64), s), pad()])
    if s > 1:
        skip = s // 2
        others = np.array([o for o in range(s) if o != skip])
        yield "all_but_one", np.concatenate([keys.of(others[rng.integers(0, s - 1, n)], s), pad()])
    yield "lane_per_shard", np.concatenate([keys.of(np.arange(n) % 32 % s, s), pad()])
    # the padding's keys belong to a shard that no valid row uses (at one shard, to the only one)
    free = s - 1
    valid = rng.integers(0, max(s - 1, 1), n)
    yield "partial_tile", np.concatenate([keys.of(valid, s), pad(free)])


class Guarded:
    """a device buffer of `rows` rows of `width` elements with PAD sentinel rows before and after; the kernels get
    the rows in the middle (ptr), the checks split the host copy into (before, middle, after)"""

    def __init__(self, rows, width, dtype, fill):
        self.rows, self.width = rows, width
        self.t = torch.full(((rows + 2 * PAD) * width,), fill, dtype=dtype, device="cuda:0")
        self.ptr = self.t.data_ptr() + PAD * width * self.t.element_size()

    def host(self):
        a = self.t.cpu().numpy().reshape(-1, self.width)
        return a[:PAD], a[PAD:PAD + self.rows], a[PAD + self.rows:]


class RouteBuffers:
    """the outputs of one partition + unpermute of n rows, sentinel-filled and guarded"""

    def __init__(self, n):
        self.routed = Guarded(n, 48, torch.uint8, SENT8)
        self.src = Guarded(n, 1, torch.int32, SENT32)
        self.counts = Guarded(1, 2 * MAX_SHARDS, torch.int32, SENT32)
        self.res = Guarded(n, 32, torch.uint8, SENT8)

    def host(self):
        torch.cuda.synchronize()
        return {k: getattr(self, k).host() for k in ("routed", "src", "counts", "res")}


def partition(st, n, d_req, s, buf, stream):
    st._check(st._L.gcra_route_partition(st._h, n, d_req.data_ptr(), s, buf.routed.ptr, buf.src.ptr, buf.counts.ptr,
                                         stream))


def unpermute(st, n, d_rres_ptr, buf, stream):
    st._check(st._L.gcra_route_unpermute(st._h, n, d_rres_ptr, buf.src.ptr, buf.res.ptr, stream))


def assert_guards(got, what):
    for k, sent in (("routed", SENT8), ("src", SENT32), ("counts", SENT32), ("res", SENT8)):
        before, _, after = got[k]
        assert (before == sent).all() and (after == sent).all(), "%s: %s written outside its rows" % (what, k)


def assert_untouched(got, what):
    assert_guards(got, what)
    for k, sent in (("routed", SENT8), ("src", SENT32), ("res", SENT8)):
        assert (got[k][1] == sent).all(), "%s: %s written" % (what, k)


def check_route(st, rows, n, s, streams, what):
    """partition rows[:n] (the buffer holds n + PAD rows) among s shards, unpermute random results through the
    partition's source indices, and compare both with numpy; once on each of `streams` (None = the engine's own)"""
    owner = w.owner_of(rows[:n, 0], s)
    order = np.argsort(owner, kind="stable")
    counts = np.bincount(owner, minlength=s)
    want = rows[:n][order]
    rres = np.frombuffer(np.random.default_rng(n * 17 + s).bytes(32 * n), np.uint64).reshape(n, 4)
    d_req = torch.from_numpy(rows.view(np.uint8).reshape(-1)).to("cuda:0")
    d_rres = torch.from_numpy(rres.copy()).to("cuda:0")
    for stream in streams:
        on = "%s, %s stream" % (what, "engine" if stream is None else "side")
        buf = RouteBuffers(n)
        torch.cuda.synchronize()
        partition(st, n, d_req, s, buf, stream)
        unpermute(st, n, d_rres.data_ptr(), buf, stream)
        got = buf.host()
        assert_guards(got, on)

        c = got["counts"][1][0]
        assert (c[:s] == counts).all(), (on, "counts", c[:s].tolist(), counts.tolist())
        assert (c[s:] == SENT32).all(), (on, "a count past n_shards written")

        routed = got["routed"][1].view(np.uint64)
        if not np.array_equal(routed, want):
            bad = np.nonzero((routed != want).any(axis=1))[0]
            raise AssertionError((on, "routed rows differ", len(bad), int(bad[0])))
        src = got["src"][1][:, 0]
        if not np.array_equal(src, order):
            bad = np.nonzero(src != order)[0]
            raise AssertionError((on, "src_index differs", len(bad), int(bad[0])))
        res = got["res"][1].view(np.uint64)[order]
        if not np.array_equal(res, rres):
            bad = np.nonzero((res != rres).any(axis=1))[0]
            raise AssertionError((on, "unpermuted results differ", len(bad), int(bad[0])))


def request_rows(n, rng):
    """n + PAD request rows of random bytes (the key hash column is set per key set)"""
    return np.frombuffer(rng.bytes(48 * (n + PAD)), np.uint64).reshape(-1, 6).copy()


SIZES = [1, 31, 32, 33, 255, 256, 257, 4095, 65535, 65536, 65537, 3 * 65536 + 17, MAX_BATCH]


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("n", SIZES)
def test_partition_and_unpermute_match_numpy(engine, n, k1_path):
    """65536 rows are exactly one scan chunk of 256 tiles; 65537 and more need the scan's carry across chunks."""
    keys = Keys(seed=n)
    side = torch.cuda.Stream("cuda:0")
    shard_counts = range(1, MAX_SHARDS + 1) if n <= 4095 else (1, 2, 3, 7, 16)
    rows = request_rows(n, keys.rng)
    for s in shard_counts:
        for name, hashes in key_sets(keys, n, s):
            rows[:, 0] = hashes
            check_route(engine, rows, n, s, (None, side.cuda_stream), "n=%d shards=%d %s" % (n, s, name))


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_partition_refusals_write_nothing(engine, k1_path):
    """0 or 17 shards and more rows than max_batch are refused before any launch; 0 rows zero counts[:n_shards] and
    write nothing else.  The engine partitions correctly afterwards."""
    keys = Keys(seed=3)
    big = MAX_BATCH + 1
    rows = request_rows(big, keys.rng)
    d_req = torch.from_numpy(rows.view(np.uint8).reshape(-1)).to("cuda:0")
    for n, s in ((100, 0), (100, MAX_SHARDS + 1), (big, 2), (big, MAX_SHARDS + 1)):
        buf = RouteBuffers(n)
        torch.cuda.synchronize()
        with pytest.raises(w.tc.Internal):
            partition(engine, n, d_req, s, buf, None)
        got = buf.host()
        assert_untouched(got, "n=%d shards=%d" % (n, s))
        assert (got["counts"][1] == SENT32).all(), "n=%d shards=%d: counts written" % (n, s)
    for s in (1, 5, MAX_SHARDS):
        buf = RouteBuffers(0)
        torch.cuda.synchronize()
        partition(engine, 0, d_req, s, buf, None)
        unpermute(engine, 0, 0, buf, None)
        got = buf.host()
        assert_untouched(got, "0 rows")
        counts = got["counts"][1][0]
        assert (counts[:s] == 0).all() and (counts[s:] == SENT32).all(), counts.tolist()
    check_route(engine, rows[:70_000 + PAD], 70_000, 7, (None,), "after the refusals")


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_shard_init_refusals_leave_the_engine_usable(k1_path):
    """gcra_shard_init's checks that need no communicator: world 0 and 17, rank < 0 and >= world, max_rows 0 and past
    max_batch.  Without an init, gcra_shard_submit, _join and _wait_tick are refused too; plain batches still decide
    as the oracle does."""
    from gpu_util import engine_requests, first_mismatch
    import oracle
    st = w.tc.ManualStore(capacity=1000, device=0, created_ns=w.traces.T0, max_batch=4096)
    L, h = st._L, st._h
    ids = bytes(384)
    for rank, world, max_rows in ((0, 0, 100), (0, 17, 100), (-1, 2, 100), (2, 2, 100), (0, 1, 0), (0, 1, 4097)):
        with pytest.raises(w.tc.Internal):
            st._check(L.gcra_shard_init(h, rank, world, ids, max_rows))
    d = torch.zeros(48, dtype=torch.uint8, device="cuda:0")
    for call in (lambda: L.gcra_shard_submit(h, 1, d.data_ptr(), d.data_ptr(), None),
                 lambda: L.gcra_shard_join(h, None), lambda: L.gcra_shard_wait_tick(h, 0, None)):
        with pytest.raises(w.tc.Internal):
            st._check(call())
    req = w.traces.config1(n=20_000, keys=500)
    res = np.empty(len(req), w.tc.RES_DTYPE)
    lim = w.tc.RateLimiter(st)
    ereq = engine_requests(req)
    for a in range(0, len(req), 4096):
        lim.rate_limit_batch(ereq[a:a + 4096], out=res[a:a + 4096])
    want = oracle.OracleStore(oracle.PERIODIC, capacity=1000, created_ns=w.traces.T0, p0=10**9).replay(req)
    bad = first_mismatch(want, res, req)
    assert bad is None, bad
    st.close()


# ------------------------------------------------------------------------------------------------- 2, 3. the ticks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def run_procs(cmds, log_dir, timeout):
    """Run the commands side by side.  Once one fails or the time is up, every process still running is killed, so a
    failed rank leaves no peer waiting behind.  The processes stay in this one's process group, and each one dies
    with this process (route_nccl_worker.py sets its parent-death signal), so nothing outlives the test."""
    procs, logs = [], []
    try:
        for i, cmd in enumerate(cmds):
            logs.append(open(os.path.join(log_dir, "proc%d.log" % i), "w"))
            procs.append(subprocess.Popen(cmd + [str(os.getpid())], stdout=logs[-1], stderr=subprocess.STDOUT))
        deadline = time.monotonic() + timeout
        while any(p.poll() is None for p in procs) and time.monotonic() < deadline:
            if any(p.returncode not in (None, 0) for p in procs):
                break
            time.sleep(0.2)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
        for f in logs:
            f.close()
    for i, p in enumerate(procs):
        with open(os.path.join(log_dir, "proc%d.log" % i)) as f:
            log = f.read()
        assert p.returncode == 0 and "route worker ok" in log, "process %d of %d exited %s:\n%s" % (
            i, len(procs), p.returncode, log[-4000:])


def host_top(glob, res):
    """the oracle's denied rows (status OK, not allowed) counted per key hash, in gcra_top_denied's order"""
    import throttlecrab_b200 as tc
    d = (res["status"] == tc.OK) & (res["allowed"] == 0)
    cnt = collections.Counter(tc.hash_key_ids(glob["key"][d]).tolist())
    return sorted(((int(h), int(c)) for h, c in cnt.items()), key=lambda hc: (-hc[1], hc[0]))


def check_run(ticks, out_dir, name, world):
    """every rank's results of every tick against ONE oracle store fed the union trace in global order; the
    collective and per-rank top denied lists against the host count; the counters against the oracle's"""
    import oracle
    import throttlecrab_b200 as tc
    from gpu_util import first_mismatch
    per_rank = [np.load(os.path.join(out_dir, "%s_rank%d.npy" % (name, r))).view(oracle.RES_DTYPE) for r in range(world)]
    reports = [json.load(open(os.path.join(out_dir, "%s_rank%d.json" % (name, r)))) for r in range(world)]
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=w.N_KEYS, created_ns=w.traces.T0, p0=10**9)
    ofs = [0] * world
    globs, wants = [], []
    for t, tick in enumerate(ticks):
        glob = np.concatenate(tick)
        want = ora.replay(glob)
        got = np.concatenate([per_rank[r][ofs[r]:ofs[r] + len(tick[r])] for r in range(world)])
        for r in range(world):
            ofs[r] += len(tick[r])
        bad = first_mismatch(want, got, glob) if len(glob) else None
        assert bad is None, "%s tick %d (%s rows per rank): %s" % (name, t, [len(x) for x in tick], bad)
        globs.append(glob)
        wants.append(want)
    assert ofs == [len(p) for p in per_rank]
    glob, want = np.concatenate(globs), np.concatenate(wants)
    assert want["allowed"].sum() > 0 and (want["allowed"] == 0).sum() > 0

    host = host_top(glob, want)
    assert len(host) > 20, "too few denied keys to test anything"
    own = w.owner_of(np.array([h for h, _ in host], np.uint64), world)
    for r, rep in enumerate(reports):
        assert rep["dropped"] == 0 and rep["own_dropped"] == 0, (name, r)
        assert [tuple(x) for x in rep["top"]] == host, (name, r, "collective top_denied", len(rep["top"]), len(host))
        mine = [hc for hc, o in zip(host, own) if o == r]
        assert [tuple(x) for x in rep["own"]] == mine, (name, r, "the rank's own list", len(rep["own"]), len(mine))
        assert rep["errors"] == 0, (name, r)
    assert sum(rep["allowed"] for rep in reports) == int(want["allowed"].sum()), name
    assert sum(rep["denied"] for rep in reports) == int(((want["status"] == tc.OK) & (want["allowed"] == 0)).sum()), name
    return reports, wants


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("world", [2, 3, 4])
def test_torch_sharded_tick_over_gloo_matches_one_oracle(world, tmp_path):
    """ShardedLimiter's CUDA branch with the real route kernels: three streams, events, every one of the 4 buffer slots
    reused, an empty slice and slices of exactly max_rows, and one owner receiving 1.25 x max_rows rows (two engine
    batches in _decide).  gloo all-to-alls CUDA tensors; a refusal to do so fails the test."""
    ticks = w.gloo_ticks(world)
    sizes = [[len(x) for x in t] for t in ticks]
    assert any(0 in s for s in sizes) and any(w.GLOO_MAX_ROWS in s for s in sizes)
    recv = [np.bincount(w.owner_of(w.tc.hash_key_ids(np.concatenate(t)["key"]), world), minlength=world) for t in ticks]
    assert max(recv[w.FLOOD_TICK]) > w.GLOO_MAX_ROWS
    port = _free_port()
    cmds = [[sys.executable, os.path.join(ROOT, "tests", "route_nccl_worker.py"), "gloo", str(world), str(r), str(port),
             str(tmp_path)] for r in range(world)]
    run_procs(cmds, str(tmp_path), timeout=800)
    check_run(ticks, str(tmp_path), "gloo", world)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_native_tick_at_world_one_matches_one_oracle(tmp_path):
    """gcra_shard_* end to end over a single-rank NCCL group: ticks of 0, 1, 255, 256, 4097 and max_rows rows, 9 back
    to back; wait_tick(0..2) on a torch stream with each tick's results read there before the join; wait_tick(3) and
    past the submitted ticks refused; a second gcra_shard_init refused.  Then the same ticks through ShardedLimiter over
    the same group."""
    ticks = w.nccl1_ticks()
    assert sorted({len(t[0]) for t in ticks}) == [0, 1, 255, 256, 4097, w.NCCL1_MAX_ROWS]
    assert len(ticks[4][0]) == 0 and len(ticks[0][0]) > 0         # the 0-row tick reuses a slot that held rows
    cmd = [sys.executable, os.path.join(ROOT, "tests", "route_nccl_worker.py"), "nccl1", str(_free_port()), str(tmp_path)]
    run_procs([cmd], str(tmp_path), timeout=800)
    reports, wants = check_run(ticks, str(tmp_path), "native", 1)
    early = reports[0]["early"]
    assert sorted(int(t) for t in early) == [w.N_TICKS - 3, w.N_TICKS - 2, w.N_TICKS - 1]
    for t, hexed in early.items():
        assert bytes.fromhex(hexed) == wants[int(t)].tobytes(), "tick %s read after wait_tick differs" % t
    check_run(ticks, str(tmp_path), "torch_nccl", 1)
