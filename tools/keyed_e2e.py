"""What hashing string keys on the GPU buys end to end: the pinned ring fed host-hashed rows, the keyed ring (key bytes
in the slot's arena, hashed by the hash pass), and host hashing inside the loop on one core.

One run prints one JSON line with:
  gpu          name and power limit (read-only nvidia-smi query)
  ring         decisions/s per ring mode (1: 16-byte requests / 32-byte results, 2: 16 / 16) of
                 hashed      rows hashed on the host before the timed region (the rate a caller with 64-bit hashes gets)
                 keyed       the keyed ring: refs + key bytes copied into the slot, gcra_ring_submit_keyed
                 host_hash   each tick's keys hashed inside the loop on ONE core (gcra_hash_key_seeded, called from C)
               alternated over --reps repetitions (median, min, max)
  hash_pass    device time of the hash pass over one 2^20-row tick (CUDA events around each of --launches launches,
               median), its algorithmic bytes (8 B reference read + key bytes + 8 B hash written) and those bytes over
               that time against the H100 SXM's 3.35 TB/s
  host_hash    keys/s of gcra_hash_key_seeded on one core
  resp         frames/s of gcra_resp_parse_throttle (hashes each key) and gcra_resp_parse_throttle_keyed (copies it),
               one core
The workload: 10 M string keys of 28 bytes ("tenant/<16 hex digits>/api/"), seeded Zipf ticks of 2^20 requests
(traces.config2), the 8-entry policy table, SipHash-2-4 under a fixed engine seed.  Every variant runs on its own
engine over the same ticks; every keyed and host-hash tick's results must equal the hashed tick's byte for byte,
else the script exits with status 1.  Needs a C compiler for the one-core host hashing loop (built in a temporary
directory).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import throttlecrab_b200 as tc  # noqa: E402
import traces  # noqa: E402

TICK = 1 << 20
KEY_LEN = 28
SEED = (0x5eed5eed12345678, 0x0badc0ffee123457)
HOST_LOOP = r"""
#include <stdint.h>
typedef uint64_t (*hash_fn)(const void *, uint64_t, uint64_t, uint64_t);
void hash_refs(void *fn, const uint64_t *refs, const uint8_t *arena, uint64_t n, uint64_t k0, uint64_t k1,
               uint8_t *rows, uint64_t row_bytes) {
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t r = refs[i];
        *(uint64_t *)(rows + i * row_bytes) = ((hash_fn)fn)(arena + (uint32_t)r, r >> 32, k0, k1);
    }
}
"""


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as ex:
        return "nvidia-smi unavailable: %r" % ex


def key_bytes(ids):
    """(len(ids), 28) uint8: "tenant/" + 16 hex digits of a scrambled id + "/api/" """
    hexd = np.frombuffer(b"0123456789abcdef", np.uint8)
    x = ids.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    out = np.empty((len(ids), KEY_LEN), np.uint8)
    out[:, :7] = np.frombuffer(b"tenant/", np.uint8)
    for j in range(16):
        out[:, 7 + j] = hexd[((x >> np.uint64(60 - 4 * j)) & np.uint64(15)).astype(np.int64)]
    out[:, 23:] = np.frombuffer(b"/api/", np.uint8)
    return out


def host_loop():
    """the one-core host hashing loop, compiled with the host compiler nvcc uses; the temporary directory is removed
    once the library is loaded (its mapping stays)"""
    with tempfile.TemporaryDirectory(prefix="keyed_e2e_") as d:
        src, so = os.path.join(d, "loop.c"), os.path.join(d, "loop.so")
        with open(src, "w") as fh:
            fh.write(HOST_LOOP)
        subprocess.check_call(["cc", "-O2", "-shared", "-fPIC", "-o", so, src])
        f = C.CDLL(so).hash_refs
    f.argtypes = [C.c_void_p] * 3 + [C.c_uint64] * 3 + [C.c_void_p, C.c_uint64]
    return f


def stat(xs):
    xs = sorted(xs)
    return {"median": xs[len(xs) // 2], "min": xs[0], "max": xs[-1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=10_000_000)
    ap.add_argument("--ticks", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--slots", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("keyed_e2e: no CUDA device")
    L = tc._native.lib()
    hash_refs = host_loop()
    siphash = C.cast(L.gcra_hash_key_seeded, C.c_void_p).value
    req = traces.config2(n_keys=a.keys, n_ticks=a.ticks, tick_size=TICK)
    ticks = []
    for t in range(a.ticks):
        sl = req[t * TICK:(t + 1) * TICK]
        rows = np.empty(TICK, tc.REQ16_DTYPE)
        rows["quantity"] = sl["quantity"]
        rows["policy"] = (sl["key"] % np.uint64(8)).astype(np.uint32)
        arena = key_bytes(sl["key"]).reshape(-1)
        refs = (np.uint64(KEY_LEN) << np.uint64(32)) | (np.arange(TICK, dtype=np.uint64) * np.uint64(KEY_LEN))
        hashed = rows.copy()
        hash_refs(siphash, refs.ctypes.data, arena.ctypes.data, TICK, SEED[0], SEED[1], hashed.ctypes.data, 16)
        rows["key_hash"] = refs
        ticks.append((int(sl["now_ns"][0]), rows, arena, hashed, refs))

    out = {"gpu": gpu_info(), "keys": a.keys, "tick": TICK, "key_bytes": KEY_LEN, "ring": {}}
    failed = []
    for mode in (1, 2):
        lims = {v: tc.RateLimiter(tc.ManualStore(capacity=a.keys, created_ns=traces.T0, max_batch=TICK, hash_seed=SEED))
                for v in ("hashed", "keyed", "host_hash")}
        rings = {}
        for v, lim in lims.items():
            lim.set_policies(traces.POLICIES)
            rings[v] = tc.Ring(lim, slots=a.slots, slot_capacity=TICK, compact=True if mode == 1 else 2,
                               key_capacity=TICK * KEY_LEN if v == "keyed" else 0)
        rates = {v: [] for v in lims}
        for rep in range(a.reps + 1):                        # rep 0 warms every variant up (and inserts the keys)
            results = {}
            for v, ring in rings.items():
                got, pend = [], {}
                t0 = time.perf_counter()
                for j, (now, rows, arena, hashed, refs) in enumerate(ticks):
                    s = j % a.slots
                    if s in pend:
                        ring.wait(s)
                        got.append(ring.res[s].view(np.uint8).copy())
                        del pend[s]
                    slot = ring.req[s]
                    # (byte views: numpy copies structured rows element by element)
                    if v == "hashed":
                        np.copyto(slot.view(np.uint8), hashed.view(np.uint8))
                        ring.submit(s, TICK, now)
                    elif v == "keyed":
                        np.copyto(slot.view(np.uint8), rows.view(np.uint8))
                        np.copyto(ring.keys[s][:len(arena)], arena)
                        ring.submit(s, TICK, now, keys_len=len(arena))
                    else:
                        np.copyto(slot.view(np.uint8), rows.view(np.uint8))
                        hash_refs(siphash, refs.ctypes.data, arena.ctypes.data, TICK, SEED[0], SEED[1],
                                  slot.ctypes.data, 16)
                        ring.submit(s, TICK, now)
                    pend[s] = j
                for s in sorted(pend, key=pend.get):
                    ring.wait(s)
                    got.append(ring.res[s].view(np.uint8).copy())
                dt = time.perf_counter() - t0
                if rep:
                    rates[v].append(a.ticks * TICK / dt)
                results[v] = np.concatenate(got)
            for v in ("keyed", "host_hash"):
                if results[v].tobytes() != results["hashed"].tobytes():
                    failed.append("mode %d rep %d: %s results differ from host-hashed rows" % (mode, rep, v))
        out["ring"]["mode%d" % mode] = {v: stat(r) for v, r in rates.items()}
        for lim in lims.values():
            lim.store.close()

    # the hash pass alone, one tick of 16-byte rows
    lim = tc.RateLimiter(tc.ManualStore(capacity=1000, created_ns=traces.T0, max_batch=TICK, hash_seed=SEED))
    _, rows, arena, hashed, _ = ticks[0]
    d_rows0 = torch.from_numpy(rows.view(np.uint8).copy()).cuda()
    d_rows, d_keys = d_rows0.clone(), torch.from_numpy(arena.copy()).cuda()
    st = torch.cuda.Stream()                                 # (a stream of its own: NULL would be the engine's)
    ms = []
    with torch.cuda.stream(st):
        for i in range(a.launches + 10):
            d_rows.copy_(d_rows0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            lim.hash_keys_device(TICK, d_rows.data_ptr(), 16, d_keys.data_ptr(), len(arena), st.cuda_stream)
            e1.record(st)
            e1.synchronize()
            if i >= 10:
                ms.append(e0.elapsed_time(e1))
    if not (d_rows.cpu().numpy().view(tc.REQ16_DTYPE)["key_hash"] == hashed["key_hash"]).all():
        failed.append("hash pass differs from the host hash")
    med = stat(ms)["median"]
    nbytes = TICK * 16 + len(arena)
    out["hash_pass"] = {"ms": stat(ms), "bytes": nbytes, "GB_per_s": round(nbytes / med / 1e6, 1),
                        "share_of_3.35TB_s": round(nbytes / med / 1e6 / 3350, 3)}
    lim.store.close()

    # host hashing and RESP parsing, one core
    _, rows, arena, hashed, refs = ticks[0]
    tmp = rows.copy()
    t0 = time.perf_counter()
    hash_refs(siphash, refs.ctypes.data, arena.ctypes.data, TICK, SEED[0], SEED[1], tmp.ctypes.data, 16)
    out["host_hash"] = {"keys_per_s": TICK / (time.perf_counter() - t0)}
    n_frames = 1 << 17
    kb = arena[:n_frames * KEY_LEN].reshape(n_frames, KEY_LEN)
    buf = b"".join(b"*5\r\n$8\r\nTHROTTLE\r\n$28\r\n" + bytes(k) + b"\r\n$3\r\n100\r\n$4\r\n1000\r\n$2\r\n60\r\n"
                   for k in kb)
    lim = tc.RateLimiter(tc.ManualStore(capacity=1000, created_ns=traces.T0, max_batch=TICK, hash_seed=SEED))
    req_out = np.empty(4096, tc.REQ_DTYPE)
    keys_out = np.empty(4096 * KEY_LEN, np.uint8)
    base = np.frombuffer(buf, np.uint8).ctypes.data
    rates = {"hashing": [], "keyed": []}
    for rep in range(a.reps + 1):
        for v in rates:
            pos, frames = 0, 0
            t0 = time.perf_counter()
            while pos < len(buf):
                view = C.cast(base + pos, C.c_char_p)
                used, cnt, stop, kused = C.c_uint64(), C.c_uint32(), C.c_int32(), C.c_uint64(0)
                if v == "hashing":
                    L.gcra_resp_parse_throttle(lim._h, view, len(buf) - pos, traces.T0, 4096, req_out.ctypes.data,
                                               C.byref(used), C.byref(cnt), C.byref(stop))
                else:
                    L.gcra_resp_parse_throttle_keyed(lim._h, view, len(buf) - pos, traces.T0, 4096, req_out.ctypes.data,
                                                     keys_out.ctypes.data, len(keys_out), C.byref(kused),
                                                     C.byref(used), C.byref(cnt), C.byref(stop))
                pos += used.value
                frames += cnt.value
            if rep:
                rates[v].append(frames / (time.perf_counter() - t0))
    out["resp"] = {v + "_frames_per_s": stat(r) for v, r in rates.items()}
    lim.store.close()
    out["failed"] = failed
    print(json.dumps(out))
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
