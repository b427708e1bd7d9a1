"""gcra_snapshot_restore: a snapshot file's entries re-inserted into engines of any world size, each keeping the keys its
shard owns.  Continuations are checked row by row against ONE oracle store that ran the whole trace without a restart.
Restore does not touch the decision path, so these tests run with the engine's own K1 pipeline choice only."""
import os
import socket
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
P3 = tuple(int(x) for x in traces.POLICIES[3])      # (5, 10, 60)
S = 10**9


def _oracle(n_keys):
    return oracle.OracleStore(oracle.PERIODIC, capacity=n_keys, created_ns=traces.T0, p0=10**9)


def _engine(capacity, **kw):
    return tc.RateLimiter(tc.ManualStore(capacity=capacity, created_ns=traces.T0, max_batch=1 << 16, **kw))


def _warm_and_tick(n_keys, ticks=1):
    return np.concatenate([traces.warm_pass(n_keys),
                           traces.config4(n_keys=n_keys, n_ticks=ticks, tick_size=1 << 15, hot=20)])


def _run(lim, req):
    return lim.rate_limit_batch(engine_requests(req))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("src,dst,n_keys", [(1, 2, 40_000), (1, 3, 54_000), (1, 4, 36_000),
                                            (2, 3, 54_000), (4, 2, 40_000), (3, 1, 40_000)])
def test_restore_into_another_world_size_continues_exactly(src, dst, n_keys, tmp_path, k1_path):
    """SRC engines run the first half and save after the same joined tick; DST fresh small engines each restore every
    file and run the second half through the peer-memory loop-back (tests/snapshot_restore_worker.py)."""
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")     # see test_gpu_sharded.py's loop-back test
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "snapshot_restore_worker.py"),
                          str(src), str(dst), str(n_keys), str(tmp_path)],
                         capture_output=True, text=True, timeout=800, env=env)
    assert out.returncode == 0 and "restore ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_tight_table_restore_grows_into_second_buckets_and_stash(tmp_path, k1_path):
    """GCRA_FLAG_TIGHT_TABLE: a 64-slot engine takes 19 000 entries (the grown table ends up near its 13/16 fill
    limit), so growth, second-choice buckets and the stash all happen inside the restore."""
    n_keys = 19_000
    trace = _warm_and_tick(n_keys)
    ora = _oracle(n_keys)
    ora.replay(trace)
    a = _engine(n_keys)
    _run(a, trace)
    path = str(tmp_path / "a.gcra")
    a.store.save(path)
    b = _engine(16, flags=tc._native.FLAG_TIGHT_TABLE)
    assert b.store.restore(path) == (n_keys, 0)
    s = b.store.stats()
    assert s["grows"] > 0 and s["stash_entries"] > 0 and s["len"] == n_keys, s
    h = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64))
    for k in range(n_keys):
        assert b.store.peek(int(h[k])) == ora.entry("k:%d" % k), k
    more = traces.config4(n_keys=n_keys, n_ticks=2, tick_size=1 << 14, start_tick=1, hot=20)
    bad = first_mismatch(ora.replay(more), _run(b, more), more)
    assert bad is None, bad


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_restore_carries_entries_only(tmp_path, k1_path):
    """Swept keys and keys only ever denied keep their slots in the source but hold no entry: not carried.  Entries
    that expired but were not swept are carried, and a later sweep removes exactly what the oracle's sweep removes."""
    n_keys = 8000
    ora = _oracle(n_keys)
    a = _engine(4 * n_keys)                             # room enough: no purge reclaims the entry-less keys' slots
    warm = traces.warm_pass(n_keys)
    bad = first_mismatch(ora.replay(warm), _run(a, warm))
    assert bad is None, bad
    # warm-pass entries expire at T0 + {0, .5, 5.4, 5.94, 17.1, 24, 356, 594} s (by key % 8)
    assert a.store.sweep(traces.T0 + 6 * S) == ora.force_sweep(traces.T0 + 6 * S) == n_keys // 2
    denied = np.zeros(1000, traces.REQ_DTYPE)          # fresh keys asking for more than their burst
    denied["key"] = np.arange(n_keys, n_keys + 1000, dtype=np.uint64)
    denied["max_burst"], denied["count_per_period"], denied["period"] = P3
    denied["quantity"] = 10
    denied["now_ns"] = traces.T0 + 7 * S
    res = _run(a, denied)
    assert first_mismatch(ora.replay(denied), res) is None and res["allowed"].sum() == 0
    sa = a.store.stats()
    assert sa["len"] == n_keys // 2 and sa["occupied_slots"] == n_keys + 1000, sa
    path = str(tmp_path / "a.gcra")
    a.store.save(path)
    b = _engine(1000)
    assert b.store.restore(path) == (n_keys // 2, 0)
    sb = b.store.stats()
    assert sb["len"] == sa["len"] and sb["occupied_slots"] == sa["len"], sb
    # at T0 + 30 s the 17.1 s and 24 s entries have expired unswept in both stores
    assert b.store.sweep(traces.T0 + 30 * S) == ora.force_sweep(traces.T0 + 30 * S) == n_keys // 4
    assert b.store.len() == ora.len()
    more = traces.warm_pass(n_keys + 1000, now_ns=traces.T0 + 31 * S)
    bad = first_mismatch(ora.replay(more), _run(b, more), more)
    assert bad is None, bad


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_restore_twice_conflicts_and_hash_seeds(tmp_path, k1_path):
    n_keys = 5000
    trace = _warm_and_tick(n_keys)
    ora = _oracle(n_keys)
    ora.replay(trace)
    a = _engine(n_keys)
    _run(a, trace)
    path = str(tmp_path / "a.gcra")
    a.store.save(path)
    b = _engine(100)
    first = b.store.restore(path)
    assert first == (n_keys, 0)
    assert b.store.restore(path) == (0, n_keys)       # every key already holds an entry: it stays
    assert b.store.len() == n_keys and b.store.stats()["occupied_slots"] == n_keys
    more = traces.config4(n_keys=n_keys, n_ticks=2, tick_size=1 << 14, start_tick=1, hot=20)
    bad = first_mismatch(ora.replay(more), _run(b, more), more)
    assert bad is None, bad

    # a seeded table: an empty engine adopts the seed; one holding entries under another seed refuses the file
    seed = (0x0123456789ABCDEF, 0xFEDCBA9876543210)
    s = tc.RateLimiter(tc.ManualStore(capacity=1000, created_ns=traces.T0, hash_seed=seed))
    keys = [b"user:%d" % i for i in range(300)]
    req = np.zeros(len(keys), tc.REQ_DTYPE)
    req["key_hash"] = np.array([s.store.hash_key(k) for k in keys], np.uint64)
    req["max_burst"], req["count_per_period"], req["period"] = P3
    req["quantity"], req["now_ns"] = 1, traces.T0
    s.rate_limit_batch(req)
    seeded = str(tmp_path / "seeded.gcra")
    s.store.save(seeded)
    c = _engine(100)
    assert c.store.restore(seeded) == (len(keys), 0)
    assert c.store.hash_seed() == seed
    assert [c.store.hash_key(k) for k in keys] == [s.store.hash_key(k) for k in keys]
    len_b = b.store.len()
    with pytest.raises(tc.Internal, match="seed"):
        b.store.restore(seeded)
    assert b.store.len() == len_b and b.store.hash_seed() == (0, 0)


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_malformed_restore_leaves_the_engine_untouched(tmp_path, k1_path):
    n_keys = 3000
    trace = _warm_and_tick(n_keys)
    ora = _oracle(n_keys)
    ora.replay(trace)
    a = _engine(n_keys)
    _run(a, trace)
    path = str(tmp_path / "a.gcra")
    a.store.save(path)
    raw = (tmp_path / "a.gcra").read_bytes()
    truncated, wrong_magic = tmp_path / "truncated.gcra", tmp_path / "magic.gcra"
    truncated.write_bytes(raw[:len(raw) - 4096])
    wrong_magic.write_bytes(b"X" + raw[1:])
    b = _engine(100)
    b.store.restore(path, 0, 2)
    before = b.store.stats()
    for p, rank, world in [(str(truncated), 0, 1), (str(wrong_magic), 0, 1), (path, 2, 2), (path, 0, 0),
                           (str(tmp_path / "missing.gcra"), 0, 1)]:
        with pytest.raises(tc.Internal):
            b.store.restore(p, rank, world)
        s = b.store.stats()
        assert (s["len"], s["table_slots"], s["occupied_slots"]) == (before["len"], before["table_slots"],
                                                                    before["occupied_slots"]), (p, rank, world)
    b.store.restore(path, 1, 2)                        # the other half: b now holds the whole table
    more = traces.config4(n_keys=n_keys, n_ticks=2, tick_size=1 << 14, start_tick=1, hot=20)
    bad = first_mismatch(ora.replay(more), _run(b, more), more)
    assert bad is None, bad


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _two_gpu_worker(rank, world, port, n_keys, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from throttlecrab_b200.sharded import PeerShardedLimiter
    tick = 1 << 15
    lim = tc.RateLimiter(tc.ManualStore(capacity=4 * n_keys, device=rank, created_ns=traces.T0, max_batch=2 * tick))
    sh = PeerShardedLimiter(lim, dist, dev)
    glob = traces.config4(n_keys=n_keys, n_ticks=4, tick_size=tick * world, hot=20)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    ress = []
    for t in range(4):
        sl = glob[t * tick * world:(t + 1) * tick * world][rank * tick:(rank + 1) * tick]
        q = torch.from_numpy(engine_requests(sl).view(np.uint8)).to(dev)
        ress.append(torch.empty(tick * 32, dtype=torch.uint8, device=dev))
        sh.submit(q, ress[-1])
    sh.save(out_dir)
    assert sh.error() == 0
    np.save(os.path.join(out_dir, "res%d.npy" % rank), np.concatenate([r.cpu().numpy() for r in ress]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_two_gpu_save_restores_into_one_engine(tmp_path, k1_path):
    """A 2-GPU peer-memory run saves (PeerShardedLimiter.save); one engine restores both files and continues."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, n_keys, tick = 2, 50_000, 1 << 15
    mp.spawn(_two_gpu_worker, args=(world, _free_port(), n_keys, str(tmp_path)), nprocs=world, join=True)
    glob = traces.config4(n_keys=n_keys, n_ticks=4, tick_size=tick * world, hot=20)
    ora = _oracle(n_keys)
    want = ora.replay(glob)
    per = [np.load(str(tmp_path / ("res%d.npy" % r))).view(tc.RES_DTYPE).reshape(4, tick) for r in range(world)]
    got = np.concatenate([per[r][t] for t in range(4) for r in range(world)])
    assert first_mismatch(want, got, glob) is None
    one = _engine(100)
    restored = sum(one.store.restore(str(tmp_path / ("rank%d.gcra" % r)))[0] for r in range(world))
    assert restored == one.store.len() == ora.len()
    more = traces.config4(n_keys=n_keys, n_ticks=2, tick_size=1 << 15, start_tick=4, hot=20)
    bad = first_mismatch(ora.replay(more), _run(one, more), more)
    assert bad is None, bad


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_full_size_restore_into_four_shards(tmp_path, k1_path):
    """The 10 M-key table of test_gpu_full_size.py's warm pass (2^25 slots, a 1.07 GB file) restored into 4 small
    engines: the lens sum to 10 M, and 20 000 sampled keys sit on their owners with the source engine's entries."""
    n_keys, tick, world = 10_000_000, 1 << 20, 4
    src = tc.RateLimiter(tc.ManualStore(capacity=n_keys, created_ns=traces.T0, max_batch=tick))
    warm = traces.warm_pass(n_keys)
    h = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64))
    req = np.empty(tick, tc.REQ_DTYPE)
    for a in range(0, n_keys, tick):
        w = warm[a:a + tick]
        r = req[:len(w)]
        r["key_hash"] = h[a:a + len(w)]
        for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
            r[f] = w[f]
        src.rate_limit_batch(r)
    assert src.store.len() == n_keys and src.store.stats()["table_slots"] == 1 << 25
    path = str(tmp_path / "full.gcra")
    src.store.save(path)
    dst = [_engine(1000) for _ in range(world)]
    t0 = time.perf_counter()
    restored = [d.store.restore(path, r, world)[0] for r, d in enumerate(dst)]
    wall = time.perf_counter() - t0
    lens = [d.store.len() for d in dst]
    assert lens == restored and sum(lens) == n_keys, lens
    sample = np.random.default_rng(23).choice(n_keys, 20_000, replace=False)
    L = tc._native.lib()
    for k in sample:
        o = L.gcra_owner_of(int(h[k]), world)
        assert dst[o].store.peek(int(h[k])) == src.store.peek(int(h[k])), int(k)
    print("\nfull-size restore: %.3f GB file into %d shards in %.2f s (%s)"
          % (os.path.getsize(path) / 1e9, world, wall, torch.cuda.get_device_name(0)))
