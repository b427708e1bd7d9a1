"""Key references without a GPU: the host key hashes keep their values now that host and hash pass share one
definition, pack_keys lays keys out as the keyed calls expect, and the keyed RESP parse copies keys and writes
references where the plain parse writes hashes (stop 3 when the arena is full).  The hash pass itself runs in
tests/test_gpu_keyed_batches.py."""
import ctypes as C
import os
import subprocess

import numpy as np

import throttlecrab_b200 as tc
from throttlecrab_b200 import _native
from throttlecrab_b200.resp import process_pipeline, process_pipeline_native
from test_resp import NOW, OracleEngine, _FakeLimiter, _cmd, _raw_throttle, _throttle

SEED = (0x0123456789abcdef, 0xfedcba9876543210)

# (key, gcra_hash_key, gcra_hash_key_seeded under SEED), as the host functions computed them before the hashes moved
# into gcra_device.cuh
PINNED = [
    (b"", 0x952f14f1e8ddc491, 0xb7e67c99394ba858),
    (b"a", 0x314a88a107c49ce2, 0x63178e9b9ce0cb13),
    (b"k:0", 0x804b424deeac8e66, 0x759965716dcd2b00),
    (b"k:17", 0xd862761b3b41d5bd, 0x444da09800e06908),
    (b"user:1", 0x91509a368d51bb9c, 0x28e6391310dd4192),
    (b"abcdefg", 0x85df098684cdd03f, 0xd2e0d31d59ea3f60),
    (b"abcdefgh", 0x0275cdc1b855638c, 0x5d1a23ccd9127a7d),
    (b"abcdefghi", 0x55a6667d88f21456, 0xaa76f37bfc861d90),
    ("kéy".encode(), 0x45f2266b65266322, 0xfb174d3e0bacfca4),
    (b"\x00" * 15, 0x31eaa8b941bac955, 0x994baef640c54f11),
    (b"x" * 70, 0x119ed4bb0e90baf4, 0x8209950caa0fbe0d),
    (b"tenant-42/api/v1/users/9999", 0xfd77039942b44c06, 0x8156c66e03b13a24),
]


def test_host_hashes_keep_their_values():
    L = _native.lib()
    for key, plain, seeded in PINNED:
        assert L.gcra_hash_key(key, len(key)) == plain, key
        assert L.gcra_hash_key_seeded(key, len(key), *SEED) == seeded, key
    # every length 0..300 (every tail length mod 8), folded into one number per hash
    a = b = 0
    for n in range(301):
        k = bytes((7 * i + 3) % 256 for i in range(n))
        a = (a * 31 + L.gcra_hash_key(k, n)) % 2**64
        b = (b * 31 + L.gcra_hash_key_seeded(k, n, *SEED)) % 2**64
    assert (a, b) == (0xd08426cbbcb3cdc0, 0x0d81c512212e382c)


def test_pack_keys_layout():
    keys = ["a", b"", "kéy", b"\xff\x00z", "x" * 300]
    refs, arena = tc.pack_keys(keys)
    assert refs.dtype == np.uint64 and arena.dtype == np.uint8
    assert bytes(arena) == b"".join(k.encode() if isinstance(k, str) else k for k in keys)
    for k, r in zip(keys, refs):
        off, ln = int(r) & 0xFFFFFFFF, int(r) >> 32
        kb = k.encode() if isinstance(k, str) else k
        assert bytes(arena[off:off + ln]) == kb and int(r) == tc.key_ref(off, ln)
    refs, arena = tc.pack_keys([])
    assert len(refs) == 0 and len(arena) == 0


def _parse(buf, max_frames, keyed_cap=None, used0=0):
    L = _native.lib()
    req = np.zeros(max(max_frames, 1), tc.REQ_DTYPE)
    used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
    if keyed_cap is None:
        assert L.gcra_resp_parse_throttle(None, buf, len(buf), NOW, max_frames, req.ctypes.data, C.byref(used),
                                          C.byref(cnt), C.byref(stop)) == 0
        return req[:cnt.value], used.value, stop.value
    arena = np.zeros(keyed_cap, np.uint8)
    kused = C.c_uint64(used0)
    assert L.gcra_resp_parse_throttle_keyed(None, buf, len(buf), NOW, max_frames, req.ctypes.data, arena.ctypes.data,
                                            keyed_cap, C.byref(kused), C.byref(used), C.byref(cnt),
                                            C.byref(stop)) == 0
    return req[:cnt.value], used.value, stop.value, arena, kused.value


def test_keyed_parse_writes_references_where_the_plain_parse_writes_hashes():
    keys = [b"a", b"user:1", "kéy".encode(), b"", b"x" * 70, b"with\r\ncrlf"]
    buf = b"".join(_raw_throttle(k, 3, 100, 60, i) for i, k in enumerate(keys)) + _cmd("PING")
    plain, used, stop = _parse(buf, 64)
    rows, kused_bytes, kstop, arena, kused = _parse(buf, 64, keyed_cap=1000, used0=5)
    assert (kused_bytes, kstop) == (used, stop) == (len(buf) - len(_cmd("PING")), 2)
    assert kused == 5 + sum(map(len, keys))
    for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
        assert (rows[f] == plain[f]).all()
    for r, p, k in zip(rows, plain, keys):
        off, ln = int(r["key_hash"]) & 0xFFFFFFFF, int(r["key_hash"]) >> 32
        assert bytes(arena[off:off + ln]) == k and tc.hash_key(bytes(arena[off:off + ln])) == int(p["key_hash"])


def test_keyed_parse_stops_unconsumed_when_the_arena_is_full():
    frames = [_throttle("key%d" % i, 3, 100, 60) for i in range(5)]      # 4-byte keys
    buf = b"".join(frames)
    rows, used, stop, arena, kused = _parse(buf, 64, keyed_cap=10)
    assert (len(rows), used, stop, kused) == (2, len(frames[0]) * 2, 3, 8)
    rows, used, stop, arena, kused = _parse(buf[used:], 64, keyed_cap=10)        # the next call continues
    assert (len(rows), stop, kused) == (2, 3, 8)
    rows, used, stop, arena, kused = _parse(buf, 64, keyed_cap=10, used0=7)
    assert (len(rows), used, stop, kused) == (0, 0, 3, 7)
    rows, used, stop, arena, kused = _parse(_throttle("", 3, 100, 60), 64, keyed_cap=10, used0=10)
    assert (len(rows), stop, kused) == (1, 0, 10)                          # an empty key always fits


class _HostHashedKeyedRing:
    """tests only (no GPU): a keyed ring whose submit does on the host what the hash pass does on the GPU, then
    decides on the oracle -- so the keyed branch of process_pipeline_native runs without a device"""

    def __init__(self, cap, key_capacity):
        self.cap, self.eng = cap, OracleEngine()
        self.req = [np.zeros(cap, tc.REQ_DTYPE)]
        self.keys = [np.zeros(key_capacity, np.uint8)]
        self.res = [None]
        self.submits = []

    def submit(self, slot, n, now, keys_len=None):
        rows = self.req[slot][:n].copy()
        self.submits.append(keys_len)
        if keys_len is None:                       # rows that already hold key hashes
            self.res[slot] = self.eng(rows)
            return
        assert keys_len <= len(self.keys[slot])
        for r in rows:
            off, ln = int(r["key_hash"]) & 0xFFFFFFFF, int(r["key_hash"]) >> 32
            assert off + ln <= keys_len
            r["key_hash"] = tc.hash_key(bytes(self.keys[slot][off:off + ln]))
        self.res[slot] = self.eng(rows)

    def wait(self, slot):
        pass


def test_keyed_pipeline_matches_the_general_pipeline_on_the_host():
    frames = [_throttle("k%d" % (i % 7), 3, 100, 60) for i in range(40)]
    frames[5] = _cmd("PING")
    frames[9] = _cmd("throttle", "k1", 3, 100, 60)             # RESP integers: the general parser, key into the arena
    frames[20] = _cmd("THROTTLE", "k3", "abc", "100", "60")
    buf = b"".join(frames)
    want = process_pipeline(buf, OracleEngine(), NOW)
    assert process_pipeline_native(buf, _FakeLimiter(), NOW, ring=_HostHashedKeyedRing(64, 4096)) == want
    # an arena too small for the whole pipeline: each call stops where the next key does not fit, and the calls
    # together answer like one general pipeline
    ring, lim, out, pos = _HostHashedKeyedRing(64, 9), _FakeLimiter(), [], 0
    ring.eng = OracleEngine()
    while pos < len(buf):
        r, consumed, n, close = process_pipeline_native(buf[pos:], lim, NOW, ring=ring)
        assert consumed > 0 and close is None
        out.append(r)
        pos += consumed
    assert b"".join(out) == want[0]


def test_keyed_pipeline_answers_a_key_longer_than_the_arena():
    """A key that can never fit the arena (longer than all of it) is hashed on the host and decided alone, so the
    connection goes on: the calls together answer like one general pipeline."""
    long_key = "L" * 100
    frames = [_throttle("k%d" % (i % 5), 3, 100, 60) for i in range(20)]
    frames[0] = _throttle(long_key, 3, 100, 60)                      # first in the buffer
    frames[6] = _throttle(long_key, 3, 100, 60, 2)                   # after frames that fill a batch
    frames[11] = _cmd("throttle", long_key, 3, 100, 60)              # through the general parser
    frames[15] = _throttle("M" * 64, 3, 100, 60)                     # exactly the arena: keyed as usual
    buf = b"".join(frames)
    ring, lim, out, pos = _HostHashedKeyedRing(64, 64), _FakeLimiter(), [], 0
    while pos < len(buf):
        r, consumed, n, close = process_pipeline_native(buf[pos:], lim, NOW, ring=ring)
        assert consumed > 0 and n > 0 and close is None
        out.append(r)
        pos += consumed
    assert b"".join(out) == process_pipeline(buf, OracleEngine(), NOW)[0]
    assert ring.submits.count(None) == 3 and len(ring.submits) > 3


STAGE_CHECK = r"""
// every address the hash pass's staging reads lies inside the arena, and every key byte of the span is staged once
#include <cstdio>
#include <vector>
#include "gcra_device.cuh"
using namespace gcra;
int main() {
    long spans = 0;
    const u64 lens[] = {1, 2, 15, 16, 17, 31, 33, 100, 2047, 2048, 2049, 4000};
    for (uintptr_t base = 0x10000; base < 0x10000 + 16; base++)
        for (u64 keys_len : lens)
            for (u32 lo = 0; lo < keys_len; lo += (lo < 40 ? 1 : 37))
                for (u32 ext = 1; lo + ext <= keys_len; ext += (ext < 40 ? 1 : 29)) {
                    const uintptr_t g0 = chunk_begin(base, lo), g1 = chunk_end(base, lo, ext);
                    std::vector<int> seen(g1 - g0, 0);
                    bool ok = true;
                    for (u32 lane = 0; lane < 32; lane++)
                        stage_key_span(base, keys_len, lo, ext, lane, 32,
                            [&](uintptr_t src, u32 dst) {
                                ok &= src % 16 == 0 && src >= base && src + 16 <= base + keys_len && src - g0 == dst;
                                for (int j = 0; j < 16; j++) seen[dst + j]++;
                            },
                            [&](uintptr_t src, u32 dst) {
                                ok &= src >= base + lo && src < base + lo + ext && src - g0 == dst;
                                seen[dst]++;
                            });
                    for (uintptr_t b = base + lo; b < base + lo + ext; b++) ok &= seen[b - g0] == 1;
                    for (int s : seen) ok &= s <= 1;
                    if (!ok) { printf("FAIL base=%lx len=%llu lo=%u ext=%u\n", (unsigned long)base, keys_len, lo, ext); return 1; }
                    spans++;
                }
    printf("ok %ld\n", spans);
    return 0;
}
"""


def test_staging_reads_nothing_outside_the_arena(tmp_path):
    """stage_key_span, the function hash_keys_kernel copies a warp's key span into shared memory with, run on the host
    with callbacks that record each read: for every arena alignment mod 16 and many spans, each 16-byte load lies
    wholly inside the arena, each byte copy inside the span, and every byte of the span is staged exactly once."""
    src, exe = tmp_path / "stage_check.cu", tmp_path / "stage_check"
    src.write_text(STAGE_CHECK)
    subprocess.check_call(["nvcc", "-std=c++17", "-arch=sm_90a", "-diag-suppress", "20013",
                           "-I" + os.path.join(os.path.dirname(_native.__file__), "csrc"), "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout + out.stderr
