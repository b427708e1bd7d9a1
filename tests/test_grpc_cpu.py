"""The gRPC host walk (gcra_grpc_parse_throttle), its responses (gcra_grpc_format_replies), the header classes and
the general path's HPACK and Huffman code, without a GPU."""
import random
import struct
from fractions import Fraction

import numpy as np
import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import grpc_transport as gt
import grpc_streams as gs
from grpc_server import request_bytes

NS = 10**9
NOW = 1_700_000_000 * NS


def walk(cn, data, max_calls=1 << 20):
    cn.buf = bytearray(data)
    o, _, req, _, sids = gt.host_walk(cn, _Zero(), NOW, max_calls)
    return o, req, sids


class _Zero:
    store = None                                 # (no engine: keys hashed with tc.hash_key)

    def rate_limit_batch(self, req):
        return np.zeros(len(req), tc.RES_DTYPE)


def _call(cn, msg=b"\x0a\x01k\x10\x05", block=None, sid=None, **kw):
    sid = sid or cn.last_stream + 2
    return gs.call(sid, gs.steady_block(cn.hpack) if block is None else block, msg, **kw)


# ---- Huffman (RFC 7541 Appendix B, transcribed) -----------------------------------------------------------------
def test_huffman_code_is_complete_and_canonical():
    assert sum(Fraction(1, 2**n) for _, n in gt.HUFFMAN) == 1
    order = sorted(range(257), key=lambda s: (gt.HUFFMAN[s][1], s))
    code, prev = 0, gt.HUFFMAN[order[0]][1]
    for k, s in enumerate(order):
        c, n = gt.HUFFMAN[s]
        if k:
            code = (code + 1) << (n - prev)
        assert c == code, s
        prev = n


def test_huffman_decodes_the_rfc_examples_and_round_trips_every_byte():
    assert gt.huffman_decode(bytes.fromhex("f1e3c2e5f23a6ba0ab90f4ff")) == b"www.example.com"
    assert gt.huffman_decode(bytes.fromhex("a8eb10649cbf")) == b"no-cache"
    assert gt.huffman_decode(bytes.fromhex("25a849e95ba97d7f")) == b"custom-key"
    assert gt.huffman_decode(bytes.fromhex("25a849e95bb8e8b4bf")) == b"custom-value"
    every = bytes(range(256))
    assert gt.huffman_decode(gt.huffman_encode(every)) == every
    with pytest.raises(gt.ConnectionError_):
        gt.huffman_decode(b"\x00")                     # padding that is not all ones


def test_hpack_decoder_on_the_rfc_c3_requests():
    d = gt.Decoder()
    assert d.decode(bytes.fromhex("828684410f7777772e6578616d706c652e636f6d")) == [
        (b":method", b"GET"), (b":scheme", b"http"), (b":path", b"/"), (b":authority", b"www.example.com")]
    assert d.decode(bytes.fromhex("828684be58086e6f2d6361636865"))[-1] == (b"cache-control", b"no-cache")
    assert d.size == 110 and len(d.table) == 2


# ---- header classes ----------------------------------------------------------------------------------------------
def test_header_classes():
    c = gt.header_class
    assert c(b":method", b"POST") == 1 and c(b":method", b"GET") == 7
    assert c(b":path", gt.PATH) == 2 and c(b":path", b"/x") == 7
    assert c(b":scheme", b"http") == 3 and c(b":authority", b"h:1") == 4
    assert c(b"content-type", b"application/grpc") == 5 and c(b"content-type", b"application/grpc+proto") == 5
    assert c(b"content-type", b"application/json") == 7 and c(b"grpc-encoding", b"identity") == 6
    assert c(b"grpc-encoding", b"gzip") == 7 and c(b"te", b"trailers") == 0 and c(b"te", b"x") == 7
    assert c(b"user-agent", b"x") == 0 and c(b"x-custom", b"v") == 0 and c(b"X-Custom", b"v") == 7
    assert c(b"connection", b"x") == 7 and c(b":status", b"200") == 7 and c(b"x", b"a\nb") == 7
    assert [c(n) for n in (b":method", b":path", b"content-type", b"grpc-encoding", b"te", b"grpc-timeout")] == \
        [8, 9, 10, 11, 12, 0]


@pytest.mark.parametrize("i", range(1, 62))
def test_every_static_entry_indexed_and_as_a_literal_name(i):
    """the compiled static class table against header_class of the RFC table's strings"""
    name, value = gt.STATIC[i - 1]
    cls = gt.header_class(name, value)
    base = b"\x83" + bytes([0x04, len(gt.PATH)]) + gt.PATH + b"\x5f\x10application/grpc"
    cn = gs.established()
    cn.hpack = gt.Decoder()
    cn.hpack.decode(b"\x5f\x10application/grpc")             # (the literal above inserts it; drop it from the block)
    base = b"\x83" + bytes([0x04, len(gt.PATH)]) + gt.PATH + b"\xbe"
    pseudo_ok = cls in (3, 4)
    want = cls in (0, 6) or pseudo_ok
    o, _, _ = walk(cn, _call(cn, block=(bytes([0x80 | i]) + base) if pseudo_ok else base + bytes([0x80 | i])))
    assert (int(o["stop"]) == 0) == want, (i, name, value, cls)
    ncls = gt.header_class(name)
    lit_cls = gt.header_class(name, b"x")
    o, _, _ = walk(cn, _call(cn, block=base + bytes([i if i < 15 else 15] + ([i - 15] if i >= 15 else []))
                             + b"\x01x"))
    assert (int(o["stop"]) == 0) == (lit_cls in (0, 6)), (i, ncls, lit_cls)


# ---- the walk ----------------------------------------------------------------------------------------------------
def test_steady_stream_every_truncation_point():
    cn = gs.established()
    data = gs.steady_stream(random.Random(5), cn, 6, ["a", "été"])
    full, req, sids = walk(cn, data)
    assert int(full["stop"]) == 0 and int(full["n_frames"]) == 6 and int(full["consumed"]) == len(data)
    assert int(full["ping"]) == 1 and list(sids) == [3, 5, 7, 9, 11, 13]
    for cut in range(len(data)):
        o, r, s = walk(cn, data[:cut])
        n = int(o["n_frames"])
        assert int(o["stop"]) in (0, 1) and np.array_equal(r, req[:n]) and list(s) == list(sids[:n]), cut


def test_row_fields_as_prost_reads_them():
    cn = gs.established()
    msg = (b"\x10\xff\xff\xff\xff\x0f" + b"\x18" + bytes([0x80] * 9) + b"\x01"   # 2: low 32 bits of 2^32-1 -> -1
           + b"\x0a\x01a" + b"\x0a\x02bb" + b"\x30\x07" + b"\x3d" + b"\0" * 4 + b"\x39" + b"\0" * 8
           + b"\x42\x01z" + b"\x20\x3c")
    o, req, _ = walk(cn, _call(cn, msg=msg))
    assert int(o["stop"]) == 0
    r = req[0]
    assert (int(r["max_burst"]), int(r["count_per_period"]), int(r["period"]), int(r["quantity"])) == (-1, 0, 60, 0)
    assert int(r["key_hash"]) == tc.hash_key(b"bb")


NEAR_MISSES = {
    "group": b"\x0b", "bad tag 0": b"\x00", "wire 6": b"\x0e", "key as varint": b"\x08\x01",
    "max_burst as LEN": b"\x12\x01a", "11-byte varint": b"\x10" + b"\x80" * 10 + b"\x00",
    "10th byte 2": b"\x10" + b"\x80" * 9 + b"\x02", "bad utf-8": b"\x0a\x01\xff", "short": b"\x0a\x05ab",
}


@pytest.mark.parametrize("name", sorted(NEAR_MISSES))
def test_message_near_misses(name):
    cn = gs.established()
    ok = _call(cn)
    o, _, _ = walk(cn, ok + _call(cn, msg=NEAR_MISSES[name], sid=cn.last_stream + 4))
    assert (int(o["stop"]), int(o["n_frames"]), int(o["consumed"])) == (2, 1, len(ok))


def _frame_misses(cn):
    blk = gs.steady_block(cn.hpack)
    s = cn.last_stream + 2
    msg = b"\x00\x00\x00\x00\x03\x0a\x01k"
    data = lambda sid=s, flags=gt.END_STREAM: gt.frame(gt.DATA, flags, sid, msg)   # noqa: E731
    hdr = lambda flags=gt.END_HEADERS, sid=s, b=blk: gt.frame(gt.HEADERS, flags, sid, b)   # noqa: E731
    return {
        "settings": gt.frame(gt.SETTINGS, 0, 0),
        "rst": gt.frame(gt.RST_STREAM, 0, s, b"\0\0\0\x08"),
        "ping ack": gt.frame(gt.PING, gt.ACK, 0, b"\0" * 8),
        "two pings": gt.frame(gt.PING, 0, 0, b"\0" * 8) * 2,
        "no end headers": hdr(0) + gt.frame(gt.CONTINUATION, gt.END_HEADERS, s, b"") + data(),
        "end stream on headers": hdr(gt.END_HEADERS | gt.END_STREAM),
        "padded headers": hdr(gt.END_HEADERS | gt.PADDED, b=b"\x00" + blk) + data(),
        "even stream": hdr(sid=s + 1) + data(s + 1),
        "old stream": hdr(sid=cn.last_stream) + data(cn.last_stream),
        "interleaved": hdr() + hdr(sid=s + 2) + data(),
        "data other stream": hdr() + data(s + 2),
        "padded data": hdr() + gt.frame(gt.DATA, gt.END_STREAM | gt.PADDED, s, b"\x00" + msg),
        "two messages": hdr() + data(s, 0) + data(s),
        "compressed": hdr() + gt.frame(gt.DATA, gt.END_STREAM, s, b"\x01" + msg[1:]),
        "length mismatch": hdr() + gt.frame(gt.DATA, gt.END_STREAM, s, msg + b"\x00"),
        "incremental indexing": hdr(b=blk + gs.lit(b"x-a", b"b", 0x40)) + data(),
        "size update": hdr(b=b"\x3f\xe1\x1f" + blk) + data(),
        "dynamic index = n_dyn": hdr(b=blk + bytes([0x80 | (62 + len(cn.hpack.table))])) + data(),
        "huffman path": hdr(b=b"\x83\x86\x04" + bytes([0x80 | len(gt.huffman_encode(gt.PATH))])
                           + gt.huffman_encode(gt.PATH) + b"\xbe") + data(),
        "pseudo after regular": hdr(b=gs.steady_block(cn.hpack) + b"\x86") + data(),
        "two methods": hdr(b=blk + b"\x83") + data(),
        "no content-type": hdr(b=b"\x83\x86" + bytes([0x04, len(gt.PATH)]) + gt.PATH) + data(),
        "window update 0": gt.frame(gt.WINDOW_UPDATE, 0, 0, b"\0\0\0\0"),
        "window overflow": gt.frame(gt.WINDOW_UPDATE, 0, 0, struct.pack(">I", 2**31 - 1)),
        "window idle stream": gt.frame(gt.WINDOW_UPDATE, 0, s + 10, b"\0\0\0\x01"),
        "big frame": gt.frame(gt.DATA, 0, s, b"\0" * 16385),
    }


@pytest.mark.parametrize("name", sorted(_frame_misses(gs.established())))
def test_frame_near_misses(name):
    cn = gs.established()
    bad = _frame_misses(cn)[name]
    o, _, _ = walk(cn, bad)
    first = 17 if name == "two pings" else 0                  # (the first PING is taken)
    assert (int(o["stop"]), int(o["n_frames"]), int(o["consumed"])) == (2, 0, first), name


def test_plain_variants_are_taken():
    cn = gs.established()
    blk = gs.steady_block(cn.hpack)
    for b in (blk + gs.lit(b"x-meta", b"v"), blk + gs.lit(b"x-meta", b"v", 0x10),
              blk + gs.lit(b"grpc-timeout", b"9S", 0x00, huff_value=True),
              blk + b"\x0f\x2b" + b"\x81" + gt.huffman_encode(b"x")[:1],      # user-agent (static 58), Huffman value
              ):
        o, _, _ = walk(cn, _call(cn, block=b))
        assert int(o["stop"]) == 0 and int(o["n_frames"]) == 1, b
    old = gs.established()                   # the oldest entry (the last dynamic index) is ignorable here
    old.hpack = gt.Decoder()
    old.hpack.decode(gs.lit(b"x-first", b"1", 0x40) + gs.first_block())
    o, _, _ = walk(old, _call(old, block=gs.steady_block(old.hpack) + bytes([0x80 | (62 + len(old.hpack.table) - 1)])))
    assert int(o["stop"]) == 0 and int(o["n_frames"]) == 1
    o, _, _ = walk(cn, gt.frame(gt.HEADERS, gt.END_HEADERS | gt.PRIO, 3, b"\0\0\0\0\x0f" + blk)
                   + gt.frame(gt.DATA, gt.END_STREAM, 3, b"\0" * 5))
    assert int(o["stop"]) == 0 and int(o["n_frames"]) == 1


def test_windows():
    cn = gs.established()
    data = b"".join(_call(cn, sid=cn.last_stream + 2 * k) for k in range(1, 4))
    no_wu = data.replace(gt.frame(gt.WINDOW_UPDATE, 0, 0, struct.pack(">I", 10)), b"")
    for w, want in ((153, 3), (152, 2), (51, 1), (50, 0)):
        cn.send_window = w
        o, _, _ = walk(cn, no_wu)
        assert int(o["n_frames"]) == want, w
    cn.send_window = 51                  # each call's connection WINDOW_UPDATE (10) is counted
    o, _, _ = walk(cn, data[:len(_call(cn))] + gt.frame(gt.WINDOW_UPDATE, 0, 0, struct.pack(">I", 41)))
    assert int(o["send_window"]) == 51 + 10 + 41
    cn.send_window, cn.init_window = 65535, 40   # 40 + the stream's own update (10) < 51
    o, _, _ = walk(cn, data)
    assert int(o["n_frames"]) == 0 and int(o["stop"]) == 2
    cn.init_window = 41
    o, _, _ = walk(cn, data)
    assert int(o["n_frames"]) == 3 and int(o["data_octets"]) == 30


def test_row_cap_stops_before_the_next_call():
    cn = gs.established()
    data = gs.steady_stream(random.Random(2), cn, 5, ["a"], extras=False)
    o, _, _ = walk(cn, data, 2)
    assert (int(o["stop"]), int(o["n_frames"]), int(o["last_stream"])) == (3, 2, 5)


# ---- responses ---------------------------------------------------------------------------------------------------
def _pb_module():
    pytest.importorskip("google.protobuf")
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    f = descriptor_pb2.FileDescriptorProto(name="tc_test.proto", package="tc", syntax="proto3")
    m = f.message_type.add(name="ThrottleResponse")
    for i, (n, t) in enumerate([("allowed", 8), ("limit", 5), ("remaining", 5), ("retry_after", 5),
                                ("reset_after", 5)], 1):
        m.field.add(name=n, number=i, type=t, label=1)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(f)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("tc.ThrottleResponse"))


def _py_reply(q, r, sid):
    """the response as this test writes it"""
    def i32(v):
        return ((int(v) + 2**31) % 2**32) - 2**31

    def varint(v):
        v &= 2**64 - 1
        out = bytearray()
        while v >= 0x80:
            out.append(v & 0x7f | 0x80)
            v >>= 7
        return bytes(out + bytes([v]))
    if int(r["status"]) == tc.OK:
        m = b"\x08\x01" if r["allowed"] else b""
        for tag, v in ((2, q["max_burst"]), (3, r["remaining"]), (4, int(r["retry_after_ns"]) // NS),
                       (5, int(r["reset_after_ns"]) // NS)):
            if i32(v):
                m += bytes([tag << 3]) + varint(i32(v))
        return (gt.frame(gt.HEADERS, 4, sid, gt.STATUS_CTYPE) + gt.frame(gt.DATA, 0, sid, b"\0" + struct.pack(
            ">I", len(m)) + m) + gt.frame(gt.HEADERS, 5, sid, gt._lit(b"grpc-status", b"0"))), m
    text = {tc.NEGATIVE_QUANTITY: "negative quantity: %d" % int(q["quantity"]),
            tc.INVALID_RATE_LIMIT: "invalid rate limit parameters"}.get(int(r["status"]), "internal error")
    return gt.trailers_only(sid, 13, "Rate limiter error: Rate limit check failed: " + text), None


def test_responses_byte_for_byte_and_against_protobuf():
    Resp = _pb_module()
    rng = np.random.default_rng(3)
    n = 3000
    req = np.zeros(n, tc.REQ_DTYPE)
    res = np.zeros(n, tc.RES_DTYPE)
    big = [0, 1, -1, 2**31 - 1, -2**31, 2**31, 2**32 + 5, -2**40, 2**62]
    req["max_burst"] = rng.choice(big + [5, 300], n)
    req["quantity"] = rng.choice([-2**63, -1, 7, 2**63 - 1], n)
    res["remaining"] = rng.choice(big, n)
    res["retry_after_ns"] = rng.choice([0, 1, NS - 1, NS, 59 * NS + 3, 2**62], n)
    res["reset_after_ns"] = rng.choice([0, NS, 3600 * NS, 2**62], n)
    res["status"] = rng.choice([0, 0, 0, 1, 2, 3], n)
    res["allowed"] = rng.integers(0, 2, n)
    req[0]["max_burst"], res[0] = -1, (-1, -NS, -NS, tc.OK, 1, [0, 0, 0])      # the longest of each kind
    req[1]["quantity"], res[1]["status"] = -2**63, tc.NEGATIVE_QUANTITY
    sids = rng.integers(1, 2**31, n).astype(np.uint32) | 1
    out, sent = gt.format_replies(req, res, sids)
    want, wsent, lens = b"", 0, []
    for q, r, s in zip(req, res, sids):
        b, m = _py_reply(q, r, int(s))
        want += b
        lens.append(len(b))
        if m is not None:
            wsent += 5 + len(m)
            p = Resp.FromString(m)
            assert (p.allowed, p.limit, p.remaining) == (bool(r["allowed"]), (int(q["max_burst"]) + 2**31) % 2**32
                                                         - 2**31, (int(r["remaining"]) + 2**31) % 2**32 - 2**31)
            assert p.SerializeToString() == m                   # prost's and protobuf's encodings agree
    assert out == want and sent == wsent
    ok = max(x for x, r in zip(lens, res) if r["status"] == tc.OK)
    err = max(x for x, r in zip(lens, res) if r["status"] != tc.OK)
    assert (ok, err) == (113, 162) and max(ok, err) <= tc.GRPC_REPLY_MAX == 168


# ---- the general path and a real client ------------------------------------------------------------------------
class _FakeStore:
    def hash_key(self, kb):
        return tc.hash_key(kb)


class _Decider:
    """tests only: a limiter whose decisions come from the oracle"""

    def __init__(self):
        import oracle
        self.store = _FakeStore()
        self.st = oracle.OracleStore(oracle.PERIODIC, capacity=1000, created_ns=NOW, p0=NS)

    def rate_limit_batch(self, req):
        out = np.zeros(len(req), tc.RES_DTYPE)
        for i, r in enumerate(req):
            s, a, rem, reset, retry = self.st.rate_limit("h%d" % int(r["key_hash"]), int(r["max_burst"]),
                                                         int(r["count_per_period"]), int(r["period"]),
                                                         int(r["quantity"]), int(r["now_ns"]))
            out[i] = (rem, reset, retry, s, a, [0, 0, 0])
        return out


def test_general_path_answers_what_the_host_walk_answers():
    """the same steady stream, once through the host walk and once frame by frame through the general path"""
    data = gs.steady_stream(random.Random(9), gs.established(), 30, ["a", "b", "c"])
    a, b = gs.established(), gs.established()
    a.buf += data
    b.buf += data
    gt.process_connections([a], _Decider(), NOW, None)
    d = _Decider()
    while b.buf and not b.closed:
        b.general(d, NOW)
    strip = lambda x: bytes(x).replace(gt.frame(gt.PING, gt.ACK, 0, bytes(range(8))), b"")   # noqa: E731

    def responses(x):
        out, i = [], 0
        while i < len(x):
            n = int.from_bytes(x[i:i + 3], "big")
            if x[i + 3] in (gt.HEADERS, gt.DATA):
                out.append(x[i:i + 9 + n])
            i += 9 + n
        return out
    assert responses(strip(a.out)) == responses(strip(b.out)) and len(responses(a.out)) >= 60
    assert a.last_stream == b.last_stream and not a.buf


def test_connection_errors_send_goaway():
    for bad in (gt.frame(gt.WINDOW_UPDATE, 0, 0, b"\0\0\0\0"), gt.frame(gt.HEADERS, 4, 2, b"\x83"),
                gt.frame(gt.HEADERS, 4, 3, b"\xff\xff\xff\xff\x0f"), gt.frame(gt.PUSH_PROMISE, 4, 3, b"\0" * 4)):
        cn = gs.established()
        cn.buf += bad
        cn.general(_Decider(), NOW)
        assert cn.closed and bytes(cn.out)[-17:][3] == gt.GOAWAY, bad


def test_grpcio_client_burst_of_five_on_the_host_walk():
    grpc = pytest.importorskip("grpc")
    from grpc_server import Server, throttle_stub
    srv = Server(_Decider(), None, now_ns=lambda: NOW)
    try:
        ch = grpc.insecure_channel("127.0.0.1:%d" % srv.port)
        stub = throttle_stub(ch)
        Resp = _pb_module()
        allowed = 0
        for _ in range(15):
            r = Resp.FromString(stub(request_bytes("rate_limit_test", 5, 10, 60, 1), timeout=10))
            if not r.allowed:
                assert allowed == 5 and r.retry_after > 0
                break
            allowed += 1
        assert allowed == 5                                      # grpc.rs:244-295
        with pytest.raises(grpc.RpcError) as e:
            ch.unary_unary("/throttlecrab.RateLimiter/Other")(b"", timeout=10)
        assert e.value.code() == grpc.StatusCode.UNIMPLEMENTED
        with pytest.raises(grpc.RpcError) as e:
            stub(b"\x0b", timeout=10)
        assert e.value.code() == grpc.StatusCode.INTERNAL
        ch.close()
    finally:
        srv.close()
    raw = bytes(srv.capture[0])
    assert raw.startswith(gt.PREFACE)


# ---- flow-control overflow hands back the state as it was ---------------------------------------------------------
def test_window_overflow_stops_with_the_state_unchanged_and_the_general_path_closes():
    cn = gs.established()
    cn.send_window = 2**31 - 1
    wu = gt.frame(gt.WINDOW_UPDATE, 0, 0, struct.pack(">I", 1))
    o, _, _ = walk(cn, wu)
    assert (int(o["stop"]), int(o["consumed"]), int(o["send_window"])) == (2, 0, 2**31 - 1)
    cn.send_window = 2**31 - 2                  # the first update fits, the second does not
    o, _, _ = walk(cn, wu + wu)
    assert (int(o["stop"]), int(o["consumed"]), int(o["send_window"])) == (2, 13, 2**31 - 1)
    cn.send_window, cn.init_window = 65535, 2**31 - 1     # a stream's update that overflows its window
    o, _, _ = walk(cn, _call(cn))
    assert (int(o["stop"]), int(o["consumed"]), int(o["send_window"]), int(o["last_stream"])) == \
        (2, 0, 65535, cn.last_stream)
    cn = gs.established()
    cn.send_window = 2**31 - 1
    cn.buf += wu
    gt.process_connections([cn], _Decider(), NOW, None)
    assert cn.closed and bytes(cn.out) == gt.frame(gt.GOAWAY, 0, 0, struct.pack(">II", 1, gt.FLOW_CONTROL_ERROR))


def test_oversized_message_is_refused_without_buffering_it():
    cn = gs.established()
    blk = gs.steady_block(cn.hpack)
    cn.buf += gt.frame(gt.HEADERS, gt.END_HEADERS, 3, blk)
    d = _Decider()
    chunk = gt.frame(gt.DATA, 0, 3, b"\0" * 16384)
    sent = 0
    while not cn.closed and 3 in cn.streams or sent == 0:
        cn.buf += chunk
        sent += 16384
        cn.general(d, NOW)
        assert sent <= 5 + gt.MAX_MESSAGE + 16384
    assert 3 not in cn.streams and b"grpc-status\x018" in bytes(cn.out)


# ---- a stream captured from a grpcio 1.80 client ----------------------------------------------------------------
# tests/golden/grpcio_throttle_stream.bin: the bytes one grpcio 1.80 channel sent over loopback for 41 Throttle calls
# (keys user:1, user:2, "été", user:1, "" in turn, some with quantity 0, then one call with x-request-id metadata),
# as the server of tests/grpc_server.py received them.
def _capture():
    import os
    with open(os.path.join(os.path.dirname(__file__), "golden", "grpcio_throttle_stream.bin"), "rb") as f:
        return f.read()


@pytest.mark.parametrize("chunk", [1 << 20, 1, 7, 64, 333])
def test_captured_stream_host_walk_against_the_general_path(chunk, monkeypatch):
    raw = _capture()
    taken = []
    real = gt.host_walk

    def counting(*a, **k):
        r = real(*a, **k)
        taken.append(int(r[0]["n_frames"]))
        return r
    monkeypatch.setattr(gt, "host_walk", counting)
    a, b = gt.Connection(), gt.Connection()
    da, db = _Decider(), _Decider()
    n_a = 0
    for i in range(0, len(raw), chunk):
        a.buf += raw[i:i + chunk]
        n_a += gt.process_connections([a], da, NOW, None)[0]
    b.buf += raw
    while b.buf and not b.closed:
        b.general(db, NOW)

    def responses(x):
        out, i = [], 0
        while i < len(x):
            n = int.from_bytes(x[i:i + 3], "big")
            if x[i + 3] in (gt.HEADERS, gt.DATA):
                out.append(bytes(x[i:i + 9 + n]))
            i += 9 + n
        return out
    assert n_a == b.n_throttle == 41 and not a.closed and not b.closed
    assert responses(a.out) == responses(b.out)
    assert sum(taken) >= 30                      # the steady-state calls went through the host walk


def test_huffman_table_through_grpcio_decoder(monkeypatch):
    """grpcio's C-core decodes a Huffman-coded metadata value holding every printable byte"""
    grpc = pytest.importorskip("grpc")
    from grpc_server import Server
    printable = bytes(range(0x21, 0x7f)) + b" " + bytes(range(0x21, 0x7f))
    value = gt.huffman_encode(printable)
    n = bytes([0x80 | len(value)]) if len(value) < 127 else bytes([0xff]) + gt._varint7(len(value) - 127)

    def trailers_with_metadata(sid, status, message=b""):
        block = gt.STATUS_CTYPE + gt._lit(b"grpc-status", str(status).encode()) + \
            b"\x00\x05x-all" + n + value
        return gt.frame(gt.HEADERS, gt.END_STREAM | gt.END_HEADERS, sid, block)
    monkeypatch.setattr(gt, "trailers_only", trailers_with_metadata)
    srv = Server(_Decider(), None, now_ns=lambda: NOW)
    try:
        ch = grpc.insecure_channel("127.0.0.1:%d" % srv.port)
        with pytest.raises(grpc.RpcError) as e:
            ch.unary_unary("/throttlecrab.RateLimiter/Other")(b"", timeout=10)
        ch.close()
    finally:
        srv.close()
    assert e.value.code() == grpc.StatusCode.UNIMPLEMENTED
    assert dict(e.value.trailing_metadata())["x-all"] == printable.decode()
