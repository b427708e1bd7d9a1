"""Child process of tests/test_gpu_keyed_batches.py: `world` engines in one process on cuda:0 with the peer-memory
pipeline (gcra_p2p_*) between them, fed string keys twice -- once as key references that gcra_hash_keys_device hashes
on the stream in front of gcra_p2p_submit_route, once as rows hashed on the host.  Results, every rank's entry of
every key and the stats must be equal, and every key must live on gcra_owner_of(its host hash).

    p2p_keyed_worker.py WORLD"""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import throttlecrab_b200 as tc  # noqa: E402
import traces  # noqa: E402
from throttlecrab_b200.sharded import connect_local  # noqa: E402

N_KEYS, TICK, N_TICKS = 20_000, 4096, 5
NAMES = [b"svc-%d/key:%d" % (i % 5, i) for i in range(N_KEYS)]


def run(world, keyed, per_tick):
    dev = torch.device("cuda", 0)
    lims = [tc.RateLimiter(tc.ManualStore(capacity=4 * N_KEYS, device=0, created_ns=traces.T0, max_batch=4 * TICK))
            for _ in range(world)]
    connect_local(lims, TICK)
    stream = torch.cuda.Stream(dev)
    outs, keep = [], []
    with torch.cuda.stream(stream):
        for t in range(N_TICKS):
            ress = []
            for r in range(world):
                sl = per_tick[t][r]
                e = np.empty(len(sl), tc.REQ_DTYPE)
                for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
                    e[f] = sl[f]
                names = [NAMES[int(k)] for k in sl["key"]]
                if keyed:
                    refs, arena = tc.pack_keys(names)
                    e["key_hash"] = refs
                    d_keys = torch.from_numpy(arena.copy()).to(dev)
                    keep.append(d_keys)
                else:
                    e["key_hash"] = [lims[r].store.hash_key(k) for k in names]
                q = torch.from_numpy(e.view(np.uint8).copy()).to(dev)
                if keyed:
                    lims[r].hash_keys_device(len(e), q.data_ptr(), 48, d_keys.data_ptr(), len(arena), stream.cuda_stream)
                res = torch.zeros(len(e) * 32, dtype=torch.uint8, device=dev)
                keep.append(q)
                ress.append(res)
                lims[r].store._check(lims[r]._L.gcra_p2p_submit_route(lims[r]._h, len(e), q.data_ptr(), stream.cuda_stream))
            for r in range(world):
                lims[r].store._check(lims[r]._L.gcra_p2p_submit_finish(lims[r]._h, ress[r].data_ptr()))
            for lim in lims:
                lim.store._check(lim._L.gcra_p2p_join(lim._h, stream.cuda_stream))
            stream.synchronize()
            outs.append(np.concatenate([x.cpu().numpy() for x in ress]))
    for lim in lims:
        e = C.c_uint32()
        lim.store._check(lim._L.gcra_p2p_error(lim._h, C.byref(e)))
        assert e.value == 0, "a wait gave up"
    hashes = [lims[0].store.hash_key(k) for k in NAMES]
    entries = [[lim.store.peek(h) for h in hashes] for lim in lims]
    stats = [lim.store.stats() for lim in lims]
    for lim in lims:
        lim.store.close()
    return np.concatenate(outs), entries, stats, hashes


def main():
    world = int(sys.argv[1])
    g = traces.config4(n_keys=N_KEYS, n_ticks=N_TICKS, tick_size=TICK * world, hot=20)
    per_tick = [np.split(g[t * TICK * world:(t + 1) * TICK * world], world) for t in range(N_TICKS)]
    res_k, ent_k, st_k, hashes = run(world, True, per_tick)
    res_h, ent_h, st_h, _ = run(world, False, per_tick)
    assert res_k.tobytes() == res_h.tobytes(), "results differ"
    assert ent_k == ent_h, "entries differ"
    # (the index-order pipeline's residue feedback counters depend on when events are seen on the host)
    timing = ("index_batches", "residue_rows", "residue_batches", "drains", "path_switches")
    assert [{k: v for k, v in s.items() if k not in timing} for s in st_k] == \
        [{k: v for k, v in s.items() if k not in timing} for s in st_h], (st_k, st_h)
    L = tc._native.lib()
    placed = 0
    for i, h in enumerate(hashes):
        owner = L.gcra_owner_of(h, world)
        for r in range(world):
            assert (ent_k[r][i] is not None) <= (r == owner), (NAMES[i], r, owner)
        placed += ent_k[owner][i] is not None
    res = res_k.view(tc.RES_DTYPE)
    assert placed > 1000 and (res["status"] == tc.OK).all() and res["allowed"].any() and not res["allowed"].all()
    print("keyed loopback ok: %d rows, %d engines, %d keys placed" % (len(res), world, placed))


if __name__ == "__main__":
    main()
