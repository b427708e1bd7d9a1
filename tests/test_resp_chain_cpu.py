"""A CPU model of how ring_parse_kernel<RespTraits> (csrc/gcra_resp_ring.cu) finds a connection's frames, against the sequential
host walk (gcra_resp_parse_throttle).  The kernel marks every candidate frame start (a '*' at the segment start or
right after a '\\n'), parses every candidate on its own, then follows the chain of frame ends from the segment start,
and cuts it at the row cap.  Here each candidate is parsed by the host parser with max_frames = 1, which is the same
grammar (csrc/gcra_resp.cuh)."""
import ctypes as C

import numpy as np

from throttlecrab_b200 import _native
import throttlecrab_b200 as tc
from test_resp import NOW, _cmd, _raw_throttle, _throttle


def _parse(seg, cap):
    req = np.zeros(max(cap, 1), tc.REQ_DTYPE)
    used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
    assert _native.lib().gcra_resp_parse_throttle(None, seg, len(seg), NOW, cap, req.ctypes.data, C.byref(used),
                                                  C.byref(cnt), C.byref(stop)) == 0
    return used.value, cnt.value, stop.value


def _chain_model(seg, room):
    cands = [p for p in range(len(seg)) if seg[p] == 0x2a and (p == 0 or seg[p - 1] == 0x0a)]
    word = {}
    for p in cands:                                        # speculative: each candidate on its own
        used, cnt, stop = _parse(seg[p:], 1)
        word[p] = (p + used, 0) if cnt else (None, stop)
    starts, p, why = [], 0, 0
    while p < len(seg):
        if seg[p] != 0x2a:
            why = 2
            break
        end, kind = word[p]
        if kind:
            why = kind
            break
        starts.append(p)
        p = end
    n = len(starts)
    if n > room or (n == room and p < len(seg)):
        return (starts[room] if room < n else p), room, 3
    return p, n, why


def test_chain_model_matches_the_sequential_walk():
    inner = _raw_throttle(b"k", 3, 100, 60)
    minimal = _raw_throttle(b"", 5, 5, 5)
    segs = [b"", inner * 4, _raw_throttle(b"\r\n" + inner * 3, 3, 100, 60) * 3, _raw_throttle(b"\n*" * 300, 1, 2, 3),
            b"*\n" * 500, minimal * 40 + minimal[:20], inner + _raw_throttle(b"bad\xff", 3, 100, 60) + inner,
            inner + _raw_throttle(b"d20", 10**19, 1, 1), inner + _cmd("PING") + inner, b"garbage" + inner,
            _throttle("q", 5, 10, 60, 2) * 3 + b"\r\n", inner[:-1]]
    rng = np.random.default_rng(3)
    for _ in range(200):
        k = bytes(rng.choice(list(b"*\r\n$5TH"), int(rng.integers(0, 40))).astype(np.uint8))
        segs.append(_raw_throttle(k, 3, 100, 60) * int(rng.integers(1, 4)) + k)
    for seg in segs:
        for room in (0, 1, 2, 3, 1000):
            assert _chain_model(seg, room) == _parse(seg, room), (seg[:80], room)
