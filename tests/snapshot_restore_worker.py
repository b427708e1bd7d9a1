"""Child process of tests/test_gpu_snapshot_restore.py: a key space moved from SRC engines to DST engines through
snapshot files, every engine in ONE process on cuda:0 (with more than one engine, the peer-memory loop-back of
tests/p2p_loopback_worker.py carries the ticks).

    snapshot_restore_worker.py SRC DST N_KEYS OUT_DIR

The global trace: a warm pass over N_KEYS keys, then 2 config4 ticks (first half, run by SRC engines); 4 config4
ticks of DST x 1024 rows (second half, run by DST engines).  Within a tick, rank r's rows precede rank r+1's.  The SRC
engines each save after the same joined tick; DST fresh engines of capacity 1000 each restore every file with their
own rank and DST as the world.  Every row of both halves must be bit-identical to ONE oracle store that ran the whole
trace.  Also checked: the DST lens and the `restored` counts sum to the SRC lens, and sampled keys sit on their owner
only, with the oracle's (tat, expiry).  Prints one JSON line, then "restore ok".

Every key of the second half is already in the table, so after the restore grew the DST tables only the per-tick room
reservation of the peer-memory pipeline remains; N_KEYS is chosen per DST so that it fits without growing inside a tick
(an engine that grows waits for the device, which in ONE process includes the other engines' waits for its own rows).
"""
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
from gpu_util import engine_requests, first_mismatch  # noqa: E402
from p2p_loopback_worker import owners  # noqa: E402
from throttlecrab_b200.sharded import connect_local  # noqa: E402

FIRST_TICK = 3 * 8192          # rows of a first-half tick (divisible by 1 .. 4)
DST_TICK = 1024                # rows per DST rank of a second-half tick


def engines(world, capacity, cap_rows):
    lims = [tc.RateLimiter(tc.ManualStore(capacity=capacity, device=0, created_ns=traces.T0, max_batch=4 * cap_rows))
            for _ in range(world)]
    if world > 1:
        connect_local(lims, cap_rows)
    return lims


def run_ticks(lims, ticks, stream):
    """ticks: list of global trace ticks; returns the engines' results in global order"""
    world, out = len(lims), []
    dev = torch.device("cuda", 0)
    for g in ticks:
        if world == 1:
            out.append(lims[0].rate_limit_batch(engine_requests(g)))
            continue
        parts = np.array_split(g, world)
        qs = [torch.from_numpy(engine_requests(p).view(np.uint8)).to(dev) for p in parts]
        rs = [torch.zeros(max(len(p), 1) * 32, dtype=torch.uint8, device=dev) for p in parts]
        for lim, p, q in zip(lims, parts, qs):
            lim.store._check(lim._L.gcra_p2p_submit_route(lim._h, len(p), q.data_ptr(), stream.cuda_stream))
        for lim, r in zip(lims, rs):
            lim.store._check(lim._L.gcra_p2p_submit_finish(lim._h, r.data_ptr()))
        for lim in lims:                 # joined after every tick: a cut, and fresh table-room bounds
            lim.store._check(lim._L.gcra_p2p_join(lim._h, stream.cuda_stream))
        stream.synchronize()
        out.append(np.concatenate([r.cpu().numpy().view(tc.RES_DTYPE)[:len(p)] for r, p in zip(rs, parts)]))
    return np.concatenate(out)


def main():
    src, dst, n_keys, out_dir = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), sys.argv[4]
    warm = traces.warm_pass(n_keys)
    body = traces.config4(n_keys=n_keys, n_ticks=2, tick_size=FIRST_TICK, hot=20)
    first = [warm[a:a + FIRST_TICK] for a in range(0, n_keys, FIRST_TICK)] + np.split(body, 2)
    second = np.split(traces.config4(n_keys=n_keys, n_ticks=4, tick_size=dst * DST_TICK, start_tick=2, hot=20), 4)

    stream = torch.cuda.Stream(torch.device("cuda", 0))
    torch.cuda.set_stream(stream)
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=n_keys, created_ns=traces.T0, p0=10**9)
    report = {}

    lims = engines(src, 4_000_000, FIRST_TICK)
    got = run_ticks(lims, first, stream)
    want = ora.replay(np.concatenate(first))
    bad = first_mismatch(want, got)
    assert bad is None, "first half: " + bad
    paths = []
    for r, lim in enumerate(lims):
        paths.append(os.path.join(out_dir, "rank%d.gcra" % r))
        lim.store.save(paths[-1])
    report["src_len"] = [lim.store.len() for lim in lims]
    assert sum(report["src_len"]) == ora.len() == n_keys
    for lim in lims:
        lim.store.close()

    lims = engines(dst, 1000, DST_TICK)
    restored = [[lim.store.restore(p, r, dst) for p in paths] for r, lim in enumerate(lims)]
    report["restored"] = [sum(x[0] for x in rs) for rs in restored]
    report["conflicts"] = [sum(x[1] for x in rs) for rs in restored]
    report["dst_len"] = [lim.store.len() for lim in lims]
    report["grows"] = [lim.store.stats()["grows"] for lim in lims]
    assert sum(report["dst_len"]) == sum(report["restored"]) == n_keys, report
    assert report["dst_len"] == report["restored"] and sum(report["conflicts"]) == 0, report
    assert min(report["grows"]) > 0, report

    sample = np.random.default_rng(3).choice(n_keys, 2000, replace=False).astype(np.uint64)
    own = owners(sample, dst)
    for k, h, o in zip(sample, tc.hash_key_ids(sample), own):
        seen = [lim.store.peek(int(h)) for lim in lims]
        assert seen[o] == ora.entry("k:%d" % k), (int(k), seen, ora.entry("k:%d" % k))
        assert all(s is None for r, s in enumerate(seen) if r != o), (int(k), seen)

    got = run_ticks(lims, second, stream)
    want = ora.replay(np.concatenate(second))
    bad = first_mismatch(want, got)
    assert bad is None, "second half: " + bad
    assert want["allowed"].sum() > 0 and (want["allowed"] == 0).sum() > 0
    for lim in lims:
        lim.store.close()
    report["rows"] = [int(sum(len(t) for t in first)), int(sum(len(t) for t in second))]
    print(json.dumps(report))
    print("restore ok: %d -> %d engines" % (src, dst))


if __name__ == "__main__":
    main()
