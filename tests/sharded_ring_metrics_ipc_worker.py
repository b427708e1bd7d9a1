"""Sharded ring metrics between processes (tests/test_gpu_sharded_ring_metrics.py): `world` processes, one engine each,
windows exchanged as CUDA IPC handles as in sharded_rings_ipc_worker.py, each engine's mixed ring on peer-memory ticks
with sharded ring metrics and denied tracking on.  Every process builds every rank's connections from the same seeds
and replays the whole tick sequence through ONE oracle store; each checks its own slots, its transport counts, the
names its connections saw denied (and no other), and the denied counts of the keys it owns.

    sharded_ring_metrics_ipc_worker.py WORLD [--gpus]

prints "sharded ring metrics ok"."""
import argparse
import ctypes as C
import os
import random
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
from sharded_rings_ipc_worker import barrier  # noqa: E402
from sharded_rings_worker import Oracle, gave_up  # noqa: E402
from sharded_ring_metrics_worker import KEYS, T, check_names, metric_conns  # noqa: E402
from test_gpu_mixed_ring import NOW, NS, SIP, _check, _expected, _place  # noqa: E402

ROW_CAP, CAP_ROWS, TICKS = 400, 1024, 8


def tick_input(lim, t, r, now):
    rng, nrng = random.Random(1000 * t + r), np.random.default_rng(1000 * t + r)
    n = 90 if (r == 0 and t % 3 == 0) else rng.randrange(0, 20)
    conns = metric_conns(rng, nrng, n) if n else []
    exp = _expected(lim, conns, ROW_CAP, now)
    return conns, exp, (np.concatenate([e[1] for e in exp]) if exp else np.zeros(0, tc.REQ_DTYPE))


def rank_main(rank, world, d, gpus):
    import torch
    dev = torch.device("cuda", rank if gpus else 0)
    torch.cuda.set_device(dev)
    lim = tc.RateLimiter(tc.PeriodicStore(capacity=1 << 20, device=dev.index, created_ns=NOW, max_batch=1 << 16,
                                          hash_seed=SIP))
    ring = tc.MixedRing(lim, 1, 256, 1 << 21, ROW_CAP)
    L, h = lim._L, lim._h
    buf, win = (C.c_char * 64)(), C.c_void_p()
    lim.store._check(L.gcra_p2p_prepare(h, rank, world, CAP_ROWS, C.addressof(buf), C.byref(win)))
    with open(os.path.join(d, ".h%d" % rank), "wb") as f:
        f.write(buf.raw)
    os.rename(os.path.join(d, ".h%d" % rank), os.path.join(d, "h%d" % rank))
    barrier(d, "p", rank, world)
    raw = b"".join(open(os.path.join(d, "h%d" % r), "rb").read() for r in range(world))
    lim.store._check(L.gcra_p2p_connect(h, raw, None))
    barrier(d, "c", rank, world)
    ring.peer_memory(True)
    lim.store.track_denied(100)
    lim.store.ring_metrics_sharded(True, 100)
    key_of = {lim.store.hash_key(k.encode()): k.encode() for k in KEYS}

    ora = Oracle()
    counts, through, seen, den_owned = np.zeros((3, 3), np.uint64), {}, set(), {}
    for t in range(TICKS):
        now = NOW + t * NS // 4
        inputs = [tick_input(lim, t, r, now) for r in range(world)]
        allrows = np.concatenate([rows for _, _, rows in inputs])
        ores = ora.decide(allrows)
        for q, o in zip(allrows, ores):
            k = int(q["key_hash"])
            seen.add(k)
            if L.gcra_owner_of(k, world) == rank and o["status"] == tc.OK and not o["allowed"]:
                den_owned[k] = den_owned.get(k, 0) + 1
        at = sum(len(rows) for _, _, rows in inputs[:rank])
        conns, exp, rows = inputs[rank]
        mine = ores[at:at + len(rows)]
        _place(ring, 0, conns)
        ring.submit(0, len(conns), now)                                # route + finish
        ring.wait(0)
        _check(ring, 0, conns, exp, mine)
        i = 0
        for (p, _, _), e in zip(conns, exp):
            for q, o in zip(e[1], mine[i:i + len(e[1])]):
                ok, allowed = int(o["status"]) == tc.OK, bool(o["allowed"])
                cls = 1 if ok and not allowed else 0 if ok or p == "resp" else 2
                counts[T[p], cls] += 1
                if cls == 1:
                    through[int(q["key_hash"])] = through.get(int(q["key_hash"]), 0) + 1
            i += len(e[1])
    lim.store._check(L.gcra_p2p_join(h, None))
    assert not gave_up([lim]), "rank %d: a wait gave up" % rank
    assert (lim.store.ring_transport_counts() == counts).all(), (rank, lim.store.ring_transport_counts(), counts)
    check_names(lim, rank, seen, through, key_of)
    assert dict(lim.store.top_denied(1 << 12)[0]) == den_owned
    barrier(d, "e", rank, world)                 # no window is released while a peer may still map it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("world", type=int)
    ap.add_argument("--gpus", action="store_true")
    ap.add_argument("--rank", type=int, default=None)
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    if a.rank is not None:
        rank_main(a.rank, a.world, a.dir, a.gpus)
        print("rank %d ok" % a.rank)
        return
    with tempfile.TemporaryDirectory() as d:
        extra = ["--gpus"] if a.gpus else []
        procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), str(a.world), "--rank", str(r),
                                   "--dir", d] + extra, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                 for r in range(a.world)]
        outs = []
        for p in procs:
            try:
                outs.append(p.communicate(timeout=600)[0])
            except subprocess.TimeoutExpired:
                for q in procs:
                    q.kill()
                raise
        for r, (p, o) in enumerate(zip(procs, outs)):
            assert p.returncode == 0 and ("rank %d ok" % r) in o, "rank %d:\n%s" % (r, o[-4000:])
    print("sharded ring metrics ok: ipc, world %d" % a.world)


if __name__ == "__main__":
    main()
