"""Child process of tests/test_gpu_background_snapshot.py: SRC engines on cuda:0, connected by the peer-memory loop-back
(tests/p2p_loopback_worker.py), run ticks without joining after any of them; every engine begins a background save
right after submitting tick CUT, again with no join, and the ticks go on.  The saves are then waited for and restored
into DST fresh engines.

    background_snapshot_worker.py SRC DST N_KEYS OUT_DIR

Checked bit-exact against ONE oracle store that ran the whole trace (the live rows of every tick) and against a second
one that ran only the ticks up to CUT (the files: sampled keys sit on their owner only, with that oracle's entry, and
the DST lens sum to its len).  The DST engines then continue that second oracle's trace exactly.  Prints one JSON line,
then "background ok".
"""
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
from gpu_util import engine_requests, first_mismatch  # noqa: E402
from p2p_loopback_worker import owners  # noqa: E402
from snapshot_restore_worker import DST_TICK, FIRST_TICK, engines, run_ticks  # noqa: E402

N_TICKS, CUT = 6, 2            # config4 ticks after the warm pass; the saves begin after body tick CUT


def main():
    src, dst, n_keys, out_dir = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), sys.argv[4]
    warm = traces.warm_pass(n_keys)
    body = np.split(traces.config4(n_keys=n_keys, n_ticks=N_TICKS, tick_size=FIRST_TICK, hot=20), N_TICKS)
    first = [warm[a:a + FIRST_TICK] for a in range(0, n_keys, FIRST_TICK)]
    ticks = first + body
    cut = len(first) + CUT             # ticks[:cut + 1] are before the cut
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=n_keys, created_ns=traces.T0, p0=10**9)
    ora_cut = oracle.OracleStore(oracle.PERIODIC, capacity=n_keys, created_ns=traces.T0, p0=10**9)
    ora_cut.replay(np.concatenate(ticks[:cut + 1]))
    report = {}

    lims = engines(src, 4_000_000, FIRST_TICK)
    keep, paths = [], [os.path.join(out_dir, "rank%d.gcra" % r) for r in range(src)]
    for i, g in enumerate(ticks):
        parts = np.array_split(g, src)
        qs = [torch.from_numpy(engine_requests(p).view(np.uint8)).to(dev) for p in parts]
        rs = [torch.zeros(max(len(p), 1) * 32, dtype=torch.uint8, device=dev) for p in parts]
        for lim, p, q in zip(lims, parts, qs):
            lim.store._check(lim._L.gcra_p2p_submit_route(lim._h, len(p), q.data_ptr(), stream.cuda_stream))
        for lim, r in zip(lims, rs):
            lim.store._check(lim._L.gcra_p2p_submit_finish(lim._h, r.data_ptr()))
        if i == cut:
            for lim, path in zip(lims, paths):        # no gcra_p2p_join: the cut is the call's place
                lim.store.save_begin(path)
        keep.append((parts, qs, rs))
    report["entries"] = [lim.store.save_wait() for lim in lims]
    for lim in lims:
        lim.store._check(lim._L.gcra_p2p_join(lim._h, stream.cuda_stream))
    stream.synchronize()
    err = []
    for lim in lims:
        e = C.c_uint32()
        lim.store._check(lim._L.gcra_p2p_error(lim._h, C.byref(e)))
        err.append(int(e.value))
    assert err == [0] * src, err
    got = np.concatenate([np.concatenate([r.cpu().numpy().view(tc.RES_DTYPE)[:len(p)] for r, p in zip(rs, parts)])
                          for parts, qs, rs in keep])
    bad = first_mismatch(ora.replay(np.concatenate(ticks)), got)
    assert bad is None, "live rows: " + bad
    assert sum(report["entries"]) == ora_cut.len(), (report, ora_cut.len())
    for lim in lims:
        lim.store.close()

    lims = engines(dst, 1000, DST_TICK)
    restored = [[lim.store.restore(p, r, dst) for p in paths] for r, lim in enumerate(lims)]
    report["restored"] = [sum(x[0] for x in rs) for rs in restored]
    report["dst_len"] = [lim.store.len() for lim in lims]
    assert sum(report["dst_len"]) == sum(report["restored"]) == ora_cut.len(), report
    sample = np.random.default_rng(5).choice(n_keys, 2000, replace=False).astype(np.uint64)
    own = owners(sample, dst)
    for k, h, o in zip(sample, tc.hash_key_ids(sample), own):
        seen = [lim.store.peek(int(h)) for lim in lims]
        assert seen[o] == ora_cut.entry("k:%d" % k), (int(k), seen, ora_cut.entry("k:%d" % k))
        assert all(s is None for r, s in enumerate(seen) if r != o), (int(k), seen)
    second = np.split(traces.config4(n_keys=n_keys, n_ticks=4, tick_size=dst * DST_TICK, start_tick=N_TICKS, hot=20), 4)
    bad = first_mismatch(ora_cut.replay(np.concatenate(second)), run_ticks(lims, second, stream))
    assert bad is None, "continuation: " + bad
    for lim in lims:
        lim.store.close()
    print(json.dumps(report))
    print("background ok: %d -> %d engines" % (src, dst))


if __name__ == "__main__":
    main()
