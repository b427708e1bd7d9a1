"""Ring ticks between processes (tests/test_gpu_sharded_rings.py): `world` processes, one engine each, their windows
exchanged as CUDA IPC handles (gcra_p2p_prepare / gcra_p2p_connect with handles), each engine's mixed ring switched to
peer-memory ticks -- which checks every peer's seed through its IPC-mapped window -- and every ring tick one
gcra_resp_ring_submit (route + finish in one call).  Odd ranks make every third tick a gcra_p2p_submit tick.  Every
process builds every rank's connections and rows from the same seeds, so each replays the whole tick sequence, rank
order within a tick, through ONE oracle store and checks its own connections' outcomes and replies, its bulk results,
the final entries of the keys it owns and its engine's counters against that replay.

    sharded_rings_ipc_worker.py WORLD [--gpus] [--bad-seed]

spawns the processes (engine r on GPU r with --gpus, else all on GPU 0) and prints "sharded rings ok".  --bad-seed:
the last rank's engine has another key-hash seed, and every rank's gcra_ring_p2p must refuse."""
import argparse
import ctypes as C
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
from test_gpu_mixed_ring import NOW, NS, SIP, _check, _expected, _place  # noqa: E402
from sharded_rings_worker import Oracle, bulk_rows, gave_up, ring_conns  # noqa: E402

ROW_CAP, CAP_ROWS, TICKS = 600, 1024, 9


def barrier(d, name, rank, world, timeout=120):
    """every rank has written <d>/<name><r> (written whole: a rename)"""
    tmp = os.path.join(d, ".%s%d" % (name, rank))
    with open(tmp, "wb") as f:
        f.write(b"1")
    os.rename(tmp, os.path.join(d, "%s%d" % (name, rank)))
    t0 = time.time()
    while not all(os.path.exists(os.path.join(d, "%s%d" % (name, r))) for r in range(world)):
        if time.time() - t0 > timeout:
            raise SystemExit("rank %d: the other ranks did not reach %s" % (rank, name))
        time.sleep(0.01)


def kind(t, r):
    return "bulk" if r % 2 == 1 and t % 3 == 1 else "ring"


def tick_input(lim, t, r, now):
    """rank r's connections (ring tick) or rows (bulk tick) of tick t: the same in every process"""
    rng, nrng = random.Random(1000 * t + r), np.random.default_rng(1000 * t + r)
    if kind(t, r) == "bulk":
        return None, bulk_rows(rng, lim, rng.randrange(0, 50), now)
    n = 220 if (r == 0 and t % 4 == 0) else rng.randrange(0, 40)          # rank 0's slot fills now and then
    conns = ring_conns(rng, nrng, r, t, n) if n else []
    exp = _expected(lim, conns, ROW_CAP, now)
    return (conns, exp), (np.concatenate([e[1] for e in exp]) if exp else np.zeros(0, tc.REQ_DTYPE))


def rank_main(rank, world, d, gpus, bad_seed):
    import torch
    dev = torch.device("cuda", rank if gpus else 0)
    torch.cuda.set_device(dev)
    seed = (1, 2) if bad_seed and rank == world - 1 else SIP
    lim = tc.RateLimiter(tc.PeriodicStore(capacity=1 << 20, device=dev.index, created_ns=NOW, max_batch=1 << 16,
                                          hash_seed=seed))
    ring = tc.MixedRing(lim, 2, 256, 1 << 21, ROW_CAP)
    L, h = lim._L, lim._h
    buf, win = (C.c_char * 64)(), C.c_void_p()
    lim.store._check(L.gcra_p2p_prepare(h, rank, world, CAP_ROWS, C.addressof(buf), C.byref(win)))
    with open(os.path.join(d, ".h%d" % rank), "wb") as f:
        f.write(buf.raw)
    os.rename(os.path.join(d, ".h%d" % rank), os.path.join(d, "h%d" % rank))
    barrier(d, "p", rank, world)
    raw = b"".join(open(os.path.join(d, "h%d" % r), "rb").read() for r in range(world))
    lim.store._check(L.gcra_p2p_connect(h, raw, None))
    barrier(d, "c", rank, world)                 # every window is mapped everywhere before the first row is stored
    if bad_seed:
        try:
            ring.peer_memory(True)
        except tc.CellError:
            pass
        else:
            raise AssertionError("rank %d: a differing seed was not refused" % rank)
        barrier(d, "e", rank, world)
        return
    ring.peer_memory(True)

    ora = Oracle()
    own_counts = np.zeros(3, np.int64)
    stream = torch.cuda.Stream(dev)
    pending, bulk, keep = [None, None], [], []

    def check(s):
        if pending[s] is None:
            return
        conns, exp, ores = pending[s]
        ring.wait(s)
        _check(ring, s, conns, exp, ores)
        pending[s] = None

    slot = 0
    for t in range(TICKS):
        now = NOW + t * NS // 4
        inputs = [tick_input(lim, t, r, now) for r in range(world)]
        ores = ora.decide(np.concatenate([rows for _, rows in inputs]))
        at = sum(len(rows) for _, rows in inputs[:rank])
        rows = inputs[rank][1]
        mine = ores[at:at + len(rows)]
        for q, o in zip(np.concatenate([rows for _, rows in inputs]), ores):
            if L.gcra_owner_of(int(q["key_hash"]), world) == rank:
                own_counts += (o["status"] == tc.OK and o["allowed"], o["status"] == tc.OK and not o["allowed"],
                               o["status"] != tc.OK)
        if kind(t, rank) == "ring":
            conns, exp = inputs[rank][0]
            check(slot)
            _place(ring, slot, conns)
            ring.submit(slot, len(conns), now)                         # route + finish
            pending[slot] = (conns, exp, mine)
            slot ^= 1
        else:
            n = len(rows)
            q = torch.from_numpy(rows.view(np.uint8)).to(dev) if n else torch.zeros(48, dtype=torch.uint8, device=dev)
            res = torch.zeros(max(n, 1) * 32, dtype=torch.uint8, device=dev)
            keep.append(q)
            torch.cuda.synchronize(dev)
            lim.store._check(L.gcra_p2p_submit(h, n, q.data_ptr(), res.data_ptr(), stream.cuda_stream))
            bulk.append((res, n, mine))
    for s in (0, 1):
        check(s)
    lim.store._check(L.gcra_p2p_join(h, None))
    for res, n, mine in bulk:
        assert res.cpu().numpy().view(tc.RES_DTYPE)[:n].tobytes() == mine.tobytes()
    assert not gave_up([lim]), "rank %d: a wait gave up" % rank
    for k in ora.keys:
        if L.gcra_owner_of(k, world) == rank:
            got, want = lim.store.peek(k), ora.st.entry("h%d" % k)
            assert got == want or (want is None and got[1] <= now), (k, got, want)
    st = lim.store.stats()
    assert [st["allowed"], st["denied"], st["errors"]] == list(own_counts), (st, own_counts)
    barrier(d, "e", rank, world)                 # no window is released while a peer may still map it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("world", type=int)
    ap.add_argument("--gpus", action="store_true")
    ap.add_argument("--bad-seed", action="store_true")
    ap.add_argument("--rank", type=int, default=None)
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    if a.rank is not None:
        rank_main(a.rank, a.world, a.dir, a.gpus, a.bad_seed)
        print("rank %d ok" % a.rank)
        return
    with tempfile.TemporaryDirectory() as d:
        extra = (["--gpus"] if a.gpus else []) + (["--bad-seed"] if a.bad_seed else [])
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
    print("sharded rings ok: ipc, world %d" % a.world)


if __name__ == "__main__":
    main()
