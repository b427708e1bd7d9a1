"""Key strings hashed on the GPU: the hash pass (hash_keys_kernel) against the host hash for every key layout, and
every keyed path -- keyed ring, hash_keys_device in front of the device / pipelined / small-batch calls,
rate_limit_batch_keys, the peer-memory tick, RESP ingest -- against the same trace with host-hashed rows."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle
import throttlecrab_b200 as tc
import traces
from gpu_util import first_mismatch
from test_resp import NOW, _cmd, _raw_throttle, _throttle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)
SEED = (0x0123456789abcdef, 0xfedcba9876543210)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(DEV)


def _hash_on_gpu(lim, refs, arena, row_bytes, arena_at_end=False):
    """refs -> key_hash column after the hash pass over rows of row_bytes; the device arena is exactly the arena (or
    sits at the very end of its allocation)"""
    rows = np.zeros(len(refs), tc.REQ_DTYPE if row_bytes == 48 else tc.REQ16_DTYPE)
    rows["key_hash"] = refs
    d_rows = _dev(rows)
    if arena_at_end:
        pad = (-len(arena)) % 512
        d_keys = torch.zeros(pad + len(arena), dtype=torch.uint8, device=DEV)
        d_keys[pad:] = torch.from_numpy(np.ascontiguousarray(arena))
        ptr = d_keys.data_ptr() + pad
    else:
        d_keys = _dev(arena) if len(arena) else torch.zeros(1, dtype=torch.uint8, device=DEV)
        ptr = d_keys.data_ptr()
    torch.cuda.synchronize()          # (the fills above are on torch's stream, the pass on the engine's)
    lim.hash_keys_device(len(rows), d_rows.data_ptr(), row_bytes, ptr, len(arena))    # (on the engine's stream)
    torch.cuda.synchronize()
    out = d_rows.cpu().numpy().view(rows.dtype)
    return out["key_hash"].copy(), out


def _layouts(rng):
    """(name, refs, arena) cases: every key length 0..300 and 4 KiB / 64 KiB keys at every offset residue mod 16,
    row order reversed / shuffled, many rows on one range, a 1-byte arena"""
    keys = [rng.integers(0, 256, n).astype(np.uint8).tobytes() for n in list(range(301)) + [4096, 65536]]
    for pad in range(16):
        refs, arena = tc.pack_keys(keys)
        yield "lengths+%d" % pad, refs + np.uint64(pad), np.concatenate([np.full(pad, 0xAB, np.uint8), arena])
    short = [b"tenant-%d/user:%d" % (i % 7, i * 7919) for i in range(2000)]
    refs, arena = tc.pack_keys(short)
    yield "in order", refs, arena
    yield "reversed", refs[::-1].copy(), arena
    yield "shuffled", rng.permutation(refs), arena
    yield "one range", np.full(1000, refs[17], np.uint64), arena
    yield "overlapping", np.array([tc.key_ref(o, ln) for o in range(0, 200, 3) for ln in (0, 1, 7, 8, 9, 40)],
                                  np.uint64), arena
    yield "1-byte arena", np.array([tc.key_ref(0, 1), tc.key_ref(0, 0), tc.key_ref(1, 0)] * 11, np.uint64), \
        np.array([0x5A], np.uint8)


@pytest.mark.parametrize("seed", [(0, 0), SEED])
def test_hash_pass_equals_the_host_hash(seed):
    lim = tc.RateLimiter(tc.ManualStore(capacity=1000, created_ns=traces.T0, max_batch=1 << 16, hash_seed=seed))
    st = lim.store
    rng = np.random.default_rng(5)
    for name, refs, arena in _layouts(rng):
        want = np.array([st.hash_key(bytes(arena[int(r) & 0xFFFFFFFF:(int(r) & 0xFFFFFFFF) + (int(r) >> 32)]))
                         for r in refs], np.uint64)
        for row_bytes in (48, 16):
            for at_end in (False, True):
                got, _ = _hash_on_gpu(lim, refs, arena, row_bytes, at_end)
                bad = np.nonzero(got != want)[0]
                assert len(bad) == 0, (name, row_bytes, at_end, int(bad[0]), hex(int(refs[bad[0]])))
    # n = 1, 31, 33 and max_batch rows of ~28-byte keys, the arena ending at the last key
    names = [b"api-key/%020d" % (i * 2654435761 % 10**12) for i in range(1 << 16)]
    refs, arena = tc.pack_keys(names)
    for n in (1, 31, 33, 1 << 16):
        want = np.array([st.hash_key(k) for k in names[:n]], np.uint64)
        last = (int(refs[n - 1]) & 0xFFFFFFFF) + (int(refs[n - 1]) >> 32)
        for row_bytes in (48, 16):
            got, _ = _hash_on_gpu(lim, refs[:n], arena[:last], row_bytes, True)
            assert (got == want).all(), (n, row_bytes)


# ---- decisions through every keyed path, against host-hashed rows on a twin engine ---------------------------
N_KEYS = 3000
NAMES = [b"tenant-%d/user:%d" % (i % 13, i) for i in range(N_KEYS)]
# stats that depend on timing, not on the decisions: the index-order pipeline's residue feedback (when events are
# seen on the host) and, for batches in flight together, which of the keys that fill a bucket pair lands in the stash
TIMING = ("index_batches", "residue_rows", "residue_batches", "drains", "path_switches", "stash_entries")


def _trace():
    """config1 (it has invalid requests too) and, for the compact formats, its policy table"""
    req = traces.config1(n=40_000, keys=N_KEYS)
    trip = np.stack([req["max_burst"], req["count_per_period"], req["period"]], axis=1)
    uniq, pol = np.unique(trip, axis=0, return_inverse=True)
    table = np.zeros(len(uniq), tc.POLICY_DTYPE)
    table["max_burst"], table["count_per_period"], table["period"] = uniq.T
    return req, [NAMES[int(k)] for k in req["key"]], table, pol.reshape(-1).astype(np.uint32)


def _rows(req, hashes):
    e = np.empty(len(req), tc.REQ_DTYPE)
    e["key_hash"] = hashes
    for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
        e[f] = req[f]
    return e


def _rows16(req, hashes, pol):
    e = np.empty(len(req), tc.REQ16_DTYPE)
    e["key_hash"] = hashes
    e["quantity"] = req["quantity"]
    e["policy"] = pol
    return e


def _oracle(req, names, now=None):
    """ONE oracle store fed the key strings (and `now` per row instead of the trace's clocks, if given)"""
    st = oracle.OracleStore(oracle.PERIODIC, capacity=N_KEYS, created_ns=traces.T0, p0=10**9)
    clocks = req["now_ns"] if now is None else now
    out = np.zeros(len(req), tc.RES_DTYPE)
    for i, (r, k) in enumerate(zip(req, names)):
        s, a, rem, reset, retry = st.rate_limit(k, int(r["max_burst"]), int(r["count_per_period"]), int(r["period"]),
                                                int(r["quantity"]), int(clocks[i]))
        out[i] = (rem, reset, retry, s, a, [0, 0, 0])
    return out


def _pair(seed=(0, 0)):
    mk = lambda: tc.RateLimiter(tc.ManualStore(capacity=N_KEYS, created_ns=traces.T0, max_batch=4096,
                                               hash_seed=seed))
    return mk(), mk()


def _same_state(a, b, names):
    sa, sb = a.store.stats(), b.store.stats()
    for k in TIMING:
        del sa[k], sb[k]
    assert sa == sb, (sa, sb)
    for k in names:
        h = a.store.hash_key(k)
        assert h == b.store.hash_key(k)
        assert a.store.peek(h) == b.store.peek(h), k


def _batches(n, size):
    return [(s, min(s + size, n)) for s in range(0, n, size)]


def _run_ring(lim, req, names, table, pol, mode, keyed, batch=4096, slots=3):
    if mode:
        lim.set_policies(table)
    ring = tc.Ring(lim, slots=slots, slot_capacity=batch, compact={0: False, 1: True, 2: 2}[mode],
                   key_capacity=64 * batch if keyed else 0)
    rdt = tc.RES16_DTYPE if mode == 2 else tc.RES_DTYPE
    out = np.empty(len(req), rdt)
    pending = {}
    for j, (a, b) in enumerate(_batches(len(req), batch)):
        s = j % slots
        if s in pending:
            ring.wait(s)
            pa, pb = pending.pop(s)
            out[pa:pb] = ring.res[s][:pb - pa]
        if keyed:
            refs, arena = tc.pack_keys(names[a:b])
            ring.keys[s][:len(arena)] = arena
            hashes, klen = refs, len(arena)
        else:
            hashes, klen = [lim.store.hash_key(k) for k in names[a:b]], None
        rows = _rows(req[a:b], hashes) if mode == 0 else _rows16(req[a:b], hashes, pol[a:b])
        ring.req[s][:b - a] = rows
        ring.submit(s, b - a, int(req["now_ns"][a]), keys_len=klen)
        pending[s] = (a, b)
    for s, (pa, pb) in pending.items():
        ring.wait(s)
        out[pa:pb] = ring.res[s][:pb - pa]
    return out


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_keyed_ring_equals_host_hashed_ring(mode):
    req, names, table, pol = _trace()
    a, b = _pair(SEED if mode == 1 else (0, 0))
    got = _run_ring(a, req, names, table, pol, mode, keyed=True)
    want = _run_ring(b, req, names, table, pol, mode, keyed=False)
    assert got.tobytes() == want.tobytes()
    _same_state(a, b, NAMES)
    if mode == 0:
        assert first_mismatch(_oracle(req, names), got, req) is None
        return
    # compact rows: the slot's clock for every row, the quantity as the 16-byte row holds it; 16-byte results expanded
    oreq = req.copy()
    oreq["quantity"] = _rows16(req, 0, pol)["quantity"]
    now = np.concatenate([np.full(b - a, req["now_ns"][a]) for a, b in _batches(len(req), 4096)])
    if mode == 2:
        got = np.concatenate([tc.expand_results16(_rows16(req[a:b], 0, pol[a:b]), int(req["now_ns"][a]), table, got[a:b])
                              for a, b in _batches(len(req), 4096)])
    assert first_mismatch(_oracle(oreq, names, now), got, oreq) is None


def _run_device(lim, req, names, keyed, how, batch):
    """how: "serial" (rate_limit_batch_device on one stream) or "pipelined" (submit_device, every batch in flight)"""
    stream = torch.cuda.Stream(DEV)
    keep, outs = [], []
    with torch.cuda.stream(stream):
        for a, b in _batches(len(req), batch):
            if keyed:
                refs, arena = tc.pack_keys(names[a:b])
                d_rows, d_keys = _dev(_rows(req[a:b], refs)), _dev(arena)
                lim.hash_keys_device(b - a, d_rows.data_ptr(), 48, d_keys.data_ptr(), len(arena), stream.cuda_stream)
                keep.append(d_keys)
            else:
                d_rows = _dev(_rows(req[a:b], [lim.store.hash_key(k) for k in names[a:b]]))
            d_res = torch.zeros((b - a) * 32, dtype=torch.uint8, device=DEV)
            if how == "serial":
                lim.rate_limit_batch_device(b - a, d_rows.data_ptr(), d_res.data_ptr(), stream.cuda_stream)
            else:
                lim.submit_device(b - a, d_rows.data_ptr(), d_res.data_ptr(), stream.cuda_stream)
            keep.append(d_rows)
            outs.append(d_res)
        if how != "serial":
            lim.join(stream.cuda_stream)
    stream.synchronize()
    return np.concatenate([o.cpu().numpy() for o in outs]).view(tc.RES_DTYPE)


@pytest.mark.parametrize("how,batch", [("serial", 4096), ("pipelined", 1000), ("serial", 255), ("serial", 37)])
def test_hash_pass_in_front_of_device_batches(how, batch):
    req, names, _, _ = _trace()
    a, b = _pair()
    got = _run_device(a, req, names, True, how, batch)
    want = _run_device(b, req, names, False, how, batch)
    assert got.tobytes() == want.tobytes()
    _same_state(a, b, NAMES)
    assert first_mismatch(_oracle(req, names), got, req) is None


@pytest.mark.parametrize("seed", [(0, 0), SEED])
def test_rate_limit_batch_keys_equals_rate_limit_batch(seed):
    req, names, _, _ = _trace()
    a, b = _pair(seed)
    got = np.concatenate([a.rate_limit_batch_keys(names[x:y], _rows(req[x:y], 0)) for x, y in _batches(len(req), 9000)])
    want = np.concatenate([b.rate_limit_batch(_rows(req[x:y], [b.store.hash_key(k) for k in names[x:y]]))
                           for x, y in _batches(len(req), 9000)])
    assert got.tobytes() == want.tobytes()
    _same_state(a, b, NAMES)
    assert first_mismatch(_oracle(req, names), got, req) is None


# ---- references that leave the arena --------------------------------------------------------------------------
def _bad_refs(n_good_bytes):
    return [tc.key_ref(n_good_bytes, 1), tc.key_ref(0, n_good_bytes + 1), tc.key_ref(0xFFFFFFFF, 2),
            tc.key_ref(5, 0xFFFFFFFF), tc.key_ref(n_good_bytes + 1, 0)]


def test_references_past_the_arena_are_internal_rows():
    req, names, table, pol = _trace()
    req, names, pol = req[:3000], names[:3000], pol[:3000]
    refs, arena = tc.pack_keys(names)
    bad = np.array(_bad_refs(len(arena)), np.uint64)
    at = np.array([0, 1, 700, 1500, 2999])
    refs = refs.copy()
    refs[at] = bad
    a, b = _pair()
    c = _pair()[0]
    # 48-byte rows through gcra_rate_limit_batch_keys
    e0 = a.store.stats()["errors"]
    rows = _rows(req, refs)
    got = np.empty(len(rows), tc.RES_DTYPE)
    a.store._check(a._L.gcra_rate_limit_batch_keys(a._h, len(rows), rows.ctypes.data, arena.ctypes.data, len(arena),
                                                   got.ctypes.data))
    assert (got["status"][at] == tc.INTERNAL).all()
    assert a.store.peek(0) is None
    keep = np.ones(len(req), bool)
    keep[at] = False
    want = b.rate_limit_batch(_rows(req[keep], [b.store.hash_key(k) for k, k_ok in zip(names, keep) if k_ok]))
    assert got[keep].tobytes() == want.tobytes()
    assert a.store.stats()["errors"] - e0 == b.store.stats()["errors"] + len(at)
    assert a.store.len() == b.store.len()
    # 16-byte rows through hash_keys_device + rate_limit_batch16_device
    c.set_policies(table)
    out16_in = _rows16(req, refs, pol)
    _, out16 = _hash_on_gpu(c, refs, arena, 16)
    assert (out16["policy"][at] == 0xFFFFFFFF).all() and (out16["key_hash"][at] == 0).all()
    out16["quantity"], out16["policy"][keep] = out16_in["quantity"], out16_in["policy"][keep]
    _, out48 = _hash_on_gpu(c, refs, arena, 48)
    assert (out48["now_ns"][at] == -1).all() and (out48["key_hash"][at] == 0).all()
    assert (out48["now_ns"][keep] == 0).all()                                           # (neighbours untouched)
    now = int(req["now_ns"][-1])
    d_rows, d_res = _dev(out16), torch.zeros(len(req) * 32, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()          # (the fill is on torch's stream, the batch on the engine's)
    e0 = c.store.stats()["errors"]
    c.rate_limit_batch16_device(len(req), d_rows.data_ptr(), now, d_res.data_ptr())
    c.store.sync()
    res16 = d_res.cpu().numpy().view(tc.RES_DTYPE)
    assert (res16["status"][at] == tc.INTERNAL).all()
    d = _pair()[0]
    d.set_policies(table)
    want16 = d.rate_limit_batch16(_rows16(req[keep], [d.store.hash_key(k) for k, k_ok in zip(names, keep) if k_ok],
                                          pol[keep]), now)
    assert res16[keep].tobytes() == want16.tobytes()
    assert c.store.stats()["errors"] - e0 == d.store.stats()["errors"] + len(at) and c.store.peek(0) is None


def test_keyed_ring_rejects_wrong_sizes_and_stays_usable():
    lim = tc.RateLimiter(tc.ManualStore(capacity=1000, created_ns=traces.T0, max_batch=4096))
    L, h = lim._L, lim._h
    assert L.gcra_ring_create_keyed(h, 2, 64, 0, 0) == tc.INTERNAL
    assert L.gcra_ring_create_keyed(h, 2, 64, 0, (1 << 32) + 1) == tc.INTERNAL
    assert L.gcra_ring_create_keyed(h, 2, 8192, 0, 100) == tc.INTERNAL          # slot_capacity > max_batch
    ring = tc.Ring(lim, slots=2, slot_capacity=64, key_capacity=100)
    assert L.gcra_ring_create_keyed(h, 2, 64, 0, 100) == tc.INTERNAL            # already made
    refs, arena = tc.pack_keys([b"k%d" % i for i in range(10)])
    ring.keys[0][:len(arena)] = arena
    rows = np.zeros(10, tc.REQ_DTYPE)
    rows["key_hash"], rows["max_burst"], rows["count_per_period"], rows["period"] = refs, 10, 100, 60
    rows["quantity"], rows["now_ns"] = 1, traces.T0
    ring.req[0][:10] = rows
    e0, n0 = lim.store.stats(), lim.store.launch_count()
    with pytest.raises(tc.Internal):
        ring.submit(0, 10, traces.T0, keys_len=101)
    with pytest.raises(tc.Internal):
        ring.submit(0, 65, traces.T0, keys_len=len(arena))
    assert lim.store.stats() == e0 and lim.store.launch_count() == n0
    ring.submit(0, 10, traces.T0, keys_len=len(arena))
    ring.wait(0)
    assert (ring.res[0][:10]["status"] == tc.OK).all()
    assert lim.store.peek(lim.store.hash_key(b"k3")) is not None
    # a ring without arenas refuses the keyed submit
    plain = tc.RateLimiter(tc.ManualStore(capacity=1000, created_ns=traces.T0, max_batch=4096))
    tc.Ring(plain, slots=1, slot_capacity=64)
    assert plain._L.gcra_ring_submit_keyed(plain._h, 0, 1, 0, traces.T0) == tc.INTERNAL
    assert plain._L.gcra_ring_keys(plain._h, 0) is None


# ---- multi-GPU: hash pass in front of the peer-memory tick ----------------------------------------------------
@pytest.mark.parametrize("world", [2, 4])
def test_hash_pass_in_front_of_the_peer_memory_tick(world):
    """Runs in a child process with CUDA_DEVICE_MAX_CONNECTIONS=32, like the other loop-back tests (engines of one
    process wait for each other's kernels)."""
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "p2p_keyed_worker.py"), str(world)],
                         capture_output=True, text=True, timeout=500, env=env)
    assert out.returncode == 0 and "keyed loopback ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


# ---- RESP ingest through a keyed ring ---------------------------------------------------------------------------
def _fuzz_frames(rng):
    """the frame generator of test_resp.py's test_native_pipeline_fuzz_against_the_general_pipeline, statement for
    statement (it is local to that test)"""
    keys = [b"a", b"user:1", "kéy".encode(), b"", b"x" * 70, b"\xff\xfe", b"with\r\ncrlf", b"-1", b"*5", b"$3"]
    nums = [0, 1, 2, 3, 5, 60, 100, -1, -5, 2**31, 2**63 - 1, -2**63, 2**63, "abc", "", "+7", "007", " 5", "5 ", "1e3"]

    def frame():
        kind = int(rng.integers(0, 10))
        if kind <= 5:
            args = [nums[int(rng.integers(0, len(nums)))] if rng.random() < 0.15 else int(rng.integers(1, 200))
                    for _ in range(int(rng.choice([3, 3, 3, 4, 4, 2, 5])))]
            f = _raw_throttle(keys[int(rng.integers(0, len(keys)))], *args)
            if rng.random() < 0.1:
                f = f.replace(b"THROTTLE", rng.choice([b"throttle", b"Throttle", b"THROTTLF", b"THROTTL"]).item(), 1)
            return f
        if kind == 6:
            return _cmd(*[["PING"], ["PING", "hello"], ["QUIT"], ["UNKNOWN"], ["throttle", "k", 3, 100, 60],
                          ["THROTTLE", "k", 3, 100, 60, 2]][int(rng.integers(0, 6))])
        if kind == 7:                                               # a damaged throttle frame
            f = bytearray(_raw_throttle(b"dmg", 3, 100, 60))
            for _ in range(int(rng.integers(1, 3))):
                op, pos = int(rng.integers(0, 3)), int(rng.integers(0, len(f)))
                if op == 0:
                    f[pos] = int(rng.integers(0, 256))
                elif op == 1:
                    del f[pos]
                else:
                    f.insert(pos, int(rng.choice([0x0d, 0x0a, 0x24, 0x2a, 0x3a, 0x2d, 0x30, 0x39, 0xff])))
            return bytes(f)
        if kind == 8:
            return [b"+OK\r\n", b":5\r\n", b"$-1\r\n", b"*0\r\n", b"*-1\r\n", b"$5\r\nab\r\n",
                    b"*5\r\n$8\r\nTHROTTLE\r\n$99999999999\r\n", b"*5\r\n$8\r\nTHROTTLE\r\n$-3\r\n", b"*99999999999\r\n",
                    b"\r\n"][int(rng.integers(0, 10))]
        return bytes(rng.integers(0, 256, int(rng.integers(1, 12))).astype(np.uint8))
    return frame


def test_keyed_resp_pipeline_fuzz():
    """test_resp.py's seeded fuzz pipelines (same seed, same frames and mutations): the keyed ring, the plain ring and
    the general parser give byte-identical replies, bytes consumed, commands applied and close reasons."""
    from throttlecrab_b200.resp import process_pipeline, process_pipeline_native
    mk = lambda: tc.RateLimiter(tc.PeriodicStore(capacity=1000, created_ns=NOW, max_batch=4096))
    keyed_lim, plain_lim, general_lim = mk(), mk(), mk()
    keyed = tc.Ring(keyed_lim, slots=1, slot_capacity=256, key_capacity=1 << 16)
    plain = tc.Ring(plain_lim, slots=1, slot_capacity=256)
    rng = np.random.default_rng(20260923)
    frame = _fuzz_frames(rng)
    for case in range(400):
        buf = b"".join(frame() for _ in range(int(rng.integers(1, 12))))
        if rng.random() < 0.4 and len(buf) > 1:
            buf = buf[:int(rng.integers(1, len(buf)))]
        got = process_pipeline_native(buf, keyed_lim, NOW + case, ring=keyed)
        assert got == process_pipeline_native(buf, plain_lim, NOW + case, ring=plain), case
        assert got == process_pipeline(buf, general_lim.rate_limit_batch, NOW + case), case
    assert keyed_lim.store.stats() == plain_lim.store.stats()


def test_keyed_resp_arena_smaller_than_a_batch():
    """A key arena too small for one buffer's keys: the parse stops at the first key that does not fit (stop 3),
    leaves that frame unconsumed, and the next call goes on from there."""
    from throttlecrab_b200.resp import process_pipeline, process_pipeline_native
    mk = lambda: tc.RateLimiter(tc.PeriodicStore(capacity=1000, created_ns=NOW, max_batch=4096))
    a, b = mk(), mk()
    ring = tc.Ring(a, slots=1, slot_capacity=256, key_capacity=40)
    frames = [_throttle("user:%d" % (i % 9), 5, 10, 60) for i in range(100)]
    frames[50] = _cmd("throttle", "user:3", 5, 10, 60)
    buf = b"".join(frames)
    out, pos, calls = [], 0, 0
    while pos < len(buf):
        r, consumed, n, close = process_pipeline_native(buf[pos:], a, NOW, ring=ring)
        assert 0 < n <= 6 and close is None
        out.append(r)
        pos += consumed
        calls += 1
    assert calls >= 100 // 6
    want = process_pipeline(buf, b.rate_limit_batch, NOW)
    assert b"".join(out) == want[0]


def test_keyed_resp_key_longer_than_the_arena():
    """A key longer than the whole key arena, between ordinary frames (as a plain frame and as one with RESP integer
    arguments): it is hashed on the host and decided alone, and the replies equal the general pipeline's byte for
    byte; no call stalls."""
    from throttlecrab_b200.resp import process_pipeline, process_pipeline_native
    mk = lambda: tc.RateLimiter(tc.PeriodicStore(capacity=1000, created_ns=NOW, max_batch=4096))
    a, b = mk(), mk()
    ring = tc.Ring(a, slots=1, slot_capacity=256, key_capacity=64)
    long_key = "L" * 100
    frames = [_throttle("user:%d" % (i % 5), 3, 10, 60) for i in range(30)]
    frames[3] = _throttle(long_key, 3, 10, 60)
    frames[4] = _throttle(long_key, 3, 10, 60, 2)
    frames[12] = _cmd("throttle", long_key, 3, 10, 60)
    frames[20] = _throttle("M" * 64, 3, 10, 60)                        # exactly the arena
    buf = b"".join(frames)
    out, pos = [], 0
    while pos < len(buf):
        r, consumed, n, close = process_pipeline_native(buf[pos:], a, NOW, ring=ring)
        assert consumed > 0 and n > 0 and close is None
        out.append(r)
        pos += consumed
    assert b"".join(out) == process_pipeline(buf, b.rate_limit_batch, NOW)[0]
    assert a.store.peek(a.store.hash_key(long_key)) == b.store.peek(b.store.hash_key(long_key)) is not None
