"""The gRPC ring's kernels (grpc_parse_conn, the reply and outcome kernels) on the inputs the host walk is tested with:
the host's near misses, HPACK and protobuf forms grpcio never sends, frame and call lists at their shared-memory
bounds, the row cap's re-walk, reply tiles, 65,536 connections, and the whole driver against the general path.

Every slot goes through one check (_serve): each connection's whole gRPC outcome, rows (byte for byte, keys hashed
under the engine's seed), replies and DATA octets sent must be what the host walk (gcra_grpc_parse_throttle) gives at
the row cap the connections before it leave, and every decision what an oracle replaying the rows in row order gives.
Right after each connection's last byte lies one more plain request of its protocol (for gRPC a call on stream
2^31 - 1 whose header block is plain whatever the dynamic table), so a walk that read past a connection's end would
take an extra row; connections start at every residue mod 16.  The same check runs on a mixed ring, with plain RESP and HTTP connections
between the gRPC ones, because its parse body is compiled separately."""
import random
import struct

import numpy as np
import pytest

import oracle
import throttlecrab_b200 as tc
from throttlecrab_b200 import grpc_transport as gt
import grpc_streams as gs
import test_gpu_grpc_ring as gr
import test_gpu_mixed_ring as gm
from grpc_server import request_bytes
from test_grpc_cpu import NEAR_MISSES, _call, _frame_misses, _pb_module, _py_reply
from test_http_cpu import body_of, request
from test_resp import _throttle

# (auto only: every ring batch takes the index-order pipeline, see test_gpu_resp_ring_inflight.py)
pytestmark = [pytest.mark.gpu, pytest.mark.parametrize("k1_path", ["auto"], indirect=True)]
NS = 10**9
NOW = 1_700_000_000 * NS
SIP = (0x0706050403020100, 0x0f0e0d0c0b0a0908)
SEEDS = pytest.mark.parametrize("seed", [(0, 0), SIP], ids=["unkeyed", "siphash"])
KINDS = pytest.mark.parametrize("kind", ["grpc", "mixed"])
OUTCOME = ("consumed", "n_frames", "stop", "data_octets", "last_stream", "send_window", "ping")


# ---- the check every case goes through --------------------------------------------------------------------------------
class Rig:
    """an engine, a ring of `kind` on it, and an oracle that replays every row the ring decided"""

    def __init__(self, kind, seed, row_capacity=4096, max_conns=256, in_capacity=1 << 21):
        batch = max(1 << 14, row_capacity)
        self.kind = kind
        self.lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 17, created_ns=NOW, max_batch=batch, hash_seed=seed))
        make = tc.GrpcRing if kind == "grpc" else tc.MixedRing
        self.ring = make(self.lim, 1, max_conns, in_capacity, row_capacity)
        self.ora = oracle.OracleStore(oracle.PERIODIC, capacity=1 << 17, created_ns=NOW, p0=NS)
        self.allowed = self.denied = 0
        self.denied_by_hash = {}


class _Conn:
    """test_gpu_grpc_ring._expected's view of a connection: its bytes and its state row"""

    def __init__(self, data, row):
        self.buf, self.row = data, row

    def conn_row(self):
        return self.row


def _with_fillers(conns, between=True):
    """(mixed ring) a plain RESP or HTTP connection on keys of its own after every gRPC one, or (between False) as
    many after all of them, so that the gRPC rows come first"""
    fill = [("resp", _throttle("fill:%d" % i, 5, 10, 60) * (1 + i % 3), None) if i % 2 else
            ("http", request(body_of("fill:%d" % i)) * (1 + i % 2), None) for i in range(len(conns))]
    if not between:
        return conns + fill
    return [c for pair in zip(conns, fill) for c in pair]


def _place(rig, conns):
    inp = rig.ring.input[0]
    at, k = 0, 0
    for c, (p, data, st) in enumerate(conns):
        at = ((at + 16) & ~15) + c % 16                       # every residue mod 16
        inp[at:at + len(data) + len(AFTER[p])] = np.frombuffer(data + AFTER[p], np.uint8)
        if rig.kind == "grpc":
            rig.ring.conns[0][c] = st
            rig.ring.conns[0][c]["off"], rig.ring.conns[0][c]["len"] = at, len(data)
        else:
            row = rig.ring.conns[0][c]
            row["off"], row["len"], row["protocol"], row["grpc_state"] = at, len(data), gm.P[p], \
                k if p == "grpc" else 7
            if p == "grpc":
                rig.ring.grpc_conns[0][k] = st
                rig.ring.grpc_conns[0][k]["off"], rig.ring.grpc_conns[0][k]["len"] = 0xffffffff, 0xfffffff0
                k += 1
        at += len(data) + len(AFTER[p])
    assert at <= len(inp)


def _serve(rig, conns, now=NOW):
    """conns -- (protocol, bytes, gRPC state row or None), only gRPC ones on a gRPC ring -- through one submit; checks
    everything against the host walks and the oracle.  Returns each gRPC connection's host outcome, rows and stream
    ids and results, and the slot's rows and results."""
    lim, ring = rig.lim, rig.ring
    if rig.kind == "grpc":
        assert all(p == "grpc" for p, _, _ in conns)
        exp = [(None, req, sids, o) for o, req, sids in
               gr._expected(lim, [_Conn(d, st) for _, d, st in conns], ring.row_capacity, now)]
    else:
        exp = gm._expected(lim, conns, ring.row_capacity, now)
    _place(rig, conns)
    ring.submit(0, len(conns), now)
    ring.wait(0)
    rows, res = ring.rows(0)
    want = np.concatenate([e[1] for e in exp]) if exp else np.zeros(0, tc.REQ_DTYPE)
    assert rows.tobytes() == want.tobytes()
    base, k, out = 0, 0, []
    for c, ((p, _, _), (fields, req, sids, o)) in enumerate(zip(conns, exp)):
        n = len(req)
        if p == "grpc":
            g = ring.outcome[0][c] if rig.kind == "grpc" else ring.grpc_outcome[0][k]
            k += 1
            for f in OUTCOME:
                assert int(g[f]) == int(o[f]), (c, f, int(g[f]), int(o[f]))
            assert bytes(g["ping_opaque"]) == bytes(o["ping_opaque"]), c
            want_bytes, sent = gt.format_replies(req, res[base:base + n], sids)
            assert int(g["data_sent"]) == sent, c
            out.append((o, req, sids, res[base:base + n]))
        else:
            g = ring.outcome[0][c]
            assert (int(g["consumed"]), int(g["n_frames"]), int(g["stop"])) == fields, (c, p)
            want_bytes, _ = gm._format(p, req, res[base:base + n], None)
        off, ln = int(g["reply_off"]), int(g["reply_len"])
        assert ring.replies[0][off:off + ln].tobytes() == want_bytes, (c, p)
        if rig.kind == "mixed":
            m = ring.outcome[0][c]
            assert (int(m["consumed"]), int(m["n_frames"]), int(m["reply_off"]), int(m["reply_len"])) == \
                (int(g["consumed"]), int(g["n_frames"]), off, ln), c
        base += n
    # the decisions, replayed in row order on the oracle (a key is its hash under the engine's seed)
    for q, r in zip(rows, res):
        w = rig.ora.rate_limit("h%d" % int(q["key_hash"]), int(q["max_burst"]), int(q["count_per_period"]),
                               int(q["period"]), int(q["quantity"]), int(q["now_ns"]))
        assert (int(r["status"]), bool(r["allowed"]), int(r["remaining"]), int(r["reset_after_ns"]),
                int(r["retry_after_ns"])) == w, q
        rig.allowed += w[0] == tc.OK and w[1]
        if w[0] == tc.OK and not w[1]:
            rig.denied += 1
            h = int(q["key_hash"])
            rig.denied_by_hash[h] = rig.denied_by_hash.get(h, 0) + 1
    st = lim.store.stats()
    assert (st["allowed"], st["denied"]) == (rig.allowed, rig.denied)
    return out, rows, res


def _grpc(conns, kind, between=True):
    """(bytes, row) pairs as _serve's connections of a `kind` ring"""
    g = [("grpc", d, st) for d, st in conns]
    return g if kind == "grpc" else _with_fillers(g, between)


# ---- bytes --------------------------------------------------------------------------------------------------------
def _hint(v, bits, first):
    """an HPACK integer with a `bits`-bit prefix, the prefix byte's other bits `first`"""
    mask = (1 << bits) - 1
    if v < mask:
        return bytes([first | v])
    out, v = bytearray([first | mask]), v - mask
    while v >= 128:
        out.append(v & 0x7f | 0x80)
        v >>= 7
    return bytes(out + bytes([v]))


def _hstr(s, huff=False):
    v = gt.huffman_encode(s) if huff else s
    return _hint(len(v), 7, 0x80 if huff else 0) + v


def _varint(v):
    v &= 2**64 - 1
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7f | 0x80)
        v >>= 7
    return bytes(out + bytes([v]))


def _key(k):
    return b"\x0a" + _varint(len(k)) + k


def _num(tag, v):
    return bytes([tag << 3]) + _varint(v)


def _unknown(tag, wt, body):
    return _varint(tag << 3 | wt) + body


def _frames(sid, payload, msg, hflags=gt.END_HEADERS):
    """HEADERS(payload) and DATA(END_STREAM) of one message on stream sid"""
    return gt.frame(gt.HEADERS, hflags, sid, payload) + \
        gt.frame(gt.DATA, gt.END_STREAM, sid, b"\0" + struct.pack(">I", len(msg)) + msg)


# what lies after each connection: a plain request of its protocol (gRPC: static :method, literal :path and
# content-type with static names, on the highest stream id)
AFTER = {"grpc": _frames(2**31 - 1, b"\x83\x04" + _hstr(gt.PATH) + b"\x0f\x10" + _hstr(b"application/grpc"),
                         request_bytes("spill", 1, 1, 60, 1)),
         "resp": _throttle("spill", 1, 1, 60), "http": request(body_of("spill"))}


# ---- 1. the host's edge cases on the GPU ------------------------------------------------------------------------------
def _host_edge_conns():
    """(name, bytes, row, stop, n_frames, consumed or None): every case of test_grpc_cpu's walk tests, after 0 to 3
    plain calls and before one more"""
    out = []

    def wrap(name, case, stop, extra, cn=None, taken=0):
        cn = cn or gs.established()
        row = cn.conn_row()
        k = len(out) % 4
        blk = gs.steady_block(cn.hpack)
        pre = b"".join(gs.call(3 + 2 * j, blk, request_bytes("e%d" % len(out), 5, 10, 60, 1)) for j in range(k))
        cn.last_stream = 1 + 2 * k                           # (the case's streams follow the prefix's)
        body = case(cn)
        data = pre + body + gs.call(cn.last_stream + 40, blk, request_bytes("e%d" % len(out), 5, 10, 60, 1))
        out.append((name, data, row, stop, k + (2 if stop == 0 else 0), len(data) if stop == 0 else len(pre) + extra))

    for name in sorted(NEAR_MISSES):
        wrap("message " + name, lambda cn, m=NEAR_MISSES[name]: _call(cn, msg=m), 2, 0)
    for name in sorted(_frame_misses(gs.established())):
        wrap("frame " + name, lambda cn, m=name: _frame_misses(cn)[m], 2, 17 if name == "two pings" else 0)
    plain = lambda b: lambda cn: _call(cn, block=b(cn))          # noqa: E731
    sb = lambda cn: gs.steady_block(cn.hpack)                    # noqa: E731
    for i, b in enumerate((lambda cn: sb(cn) + gs.lit(b"x-meta", b"v"), lambda cn: sb(cn) + gs.lit(b"x-meta", b"v", 0x10),
                           lambda cn: sb(cn) + gs.lit(b"grpc-timeout", b"9S", 0x00, huff_value=True),
                           lambda cn: sb(cn) + b"\x0f\x2b" + b"\x81" + gt.huffman_encode(b"x")[:1])):
        wrap("variant %d" % i, plain(b), 0, 0)
    old = gs.established()
    old.hpack = gt.Decoder()
    old.hpack.decode(gs.lit(b"x-first", b"1", 0x40) + gs.first_block())
    wrap("oldest dynamic entry", plain(lambda cn: sb(cn) + bytes([0x80 | (62 + len(cn.hpack.table) - 1)])), 0, 0,
         cn=old)
    wrap("priority", lambda cn: gt.frame(gt.HEADERS, gt.END_HEADERS | gt.PRIO, cn.last_stream + 2,
                                         b"\0\0\0\0\x0f" + sb(cn))
         + gt.frame(gt.DATA, gt.END_STREAM, cn.last_stream + 2, b"\0" * 5), 0, 0)
    prost = (b"\x10\xff\xff\xff\xff\x0f" + b"\x18" + bytes([0x80] * 9) + b"\x01" + b"\x0a\x01a" + b"\x0a\x02bb"
             + b"\x30\x07" + b"\x3d" + b"\0" * 4 + b"\x39" + b"\0" * 8 + b"\x42\x01z" + b"\x20\x3c")
    wrap("row fields as prost reads them", lambda cn: _call(cn, msg=prost), 0, 0)

    # test_windows: the windows in the state row
    cn = gs.established()
    three = b"".join(_call(cn, sid=cn.last_stream + 2 * k) for k in range(1, 4))
    no_wu = three.replace(gt.frame(gt.WINDOW_UPDATE, 0, 0, struct.pack(">I", 10)), b"")
    for w, n in ((153, 3), (152, 2), (51, 1), (50, 0)):
        row = cn.conn_row()
        row["send_window"] = w
        out.append(("send window %d" % w, no_wu, row, 0 if n == 3 else 2, n, None))
    row = cn.conn_row()
    row["send_window"] = 51
    out.append(("window updates counted", three[:len(_call(cn))] + gt.frame(gt.WINDOW_UPDATE, 0, 0,
                                                                            struct.pack(">I", 41)), row, 0, 1, None))
    for iw, n in ((40, 0), (41, 3)):
        row = cn.conn_row()
        row["init_window"] = iw
        out.append(("init window %d" % iw, three, row, 0 if n else 2, n, None))
    return out


@KINDS
@SEEDS
def test_host_edge_cases_on_the_gpu(kind, seed):
    cases = _host_edge_conns()
    rig = Rig(kind, seed, max_conns=256)
    got, _, _ = _serve(rig, _grpc([(d, st) for _, d, st, _, _, _ in cases], kind))
    for (name, data, _, stop, n, consumed), (o, *_) in zip(cases, got):
        assert (int(o["stop"]), int(o["n_frames"])) == (stop, n), name
        if consumed is not None:
            assert int(o["consumed"]) == consumed, name
    assert int(got[[c[0] for c in cases].index("window updates counted")][0]["send_window"]) == 51 + 10 + 41

    # every truncation point of a 6-call steady stream, one connection per cut
    cn = gs.established()
    data = gs.steady_stream(random.Random(5), cn, 6, ["a", "été"])
    rig = Rig(kind, seed, max_conns=2 * len(data) + 2, in_capacity=1 << 21)
    got, _, _ = _serve(rig, _grpc([(data[:cut], cn.conn_row()) for cut in range(len(data) + 1)], kind))
    assert [int(o["stop"]) for o, *_ in got].count(0) >= 7 and int(got[-1][0]["n_frames"]) == 6
    assert all(int(o["stop"]) in (0, 1) for o, *_ in got)


# ---- 2. HPACK forms grpcio never sends ---------------------------------------------------------------------------------
PATH_CLS = gt.class_byte(b":path", gt.PATH)
CTYPE_CLS = gt.class_byte(b"content-type", b"application/grpc")
DYN_BLOCK = b"\x83" + _hint(188, 7, 0x80) + _hint(189, 7, 0x80)     # :path and content-type at dynamic 126, 127


def _dyn_row(last_stream):
    """a 128-entry dynamic table (the row is the contract: no decoder made it), :path and content-type its oldest"""
    row = gs.established().conn_row()
    cls = [gt.class_byte(b"user-agent", b"x"), gt.class_byte(b":authority", b"h:1"), gt.class_byte(b":method", b"GET"),
           gt.class_byte(b"te", b"trailers"), gt.class_byte(b"grpc-encoding", b"identity"), gt.class_byte(b"x-a", b"b")]
    row["n_dyn"] = 128
    row["dyn_class"][:] = [cls[i % len(cls)] for i in range(128)]
    row["dyn_class"][126], row["dyn_class"][127] = PATH_CLS, CTYPE_CLS
    row["last_stream"] = last_stream
    return row


def _pad_block(total):
    """DYN_BLOCK and a literal x-pad header: `total` bytes"""
    for n in range(total, 0, -1):
        b = DYN_BLOCK + b"\x00\x05x-pad" + _hstr(b"v" * n)
        if len(b) == total:
            return b
    raise AssertionError(total)


def _hpack_cases():
    """(name, bytes of one call on `sid`, plain)"""
    ctype = _hint(31, 4, 0x10) + _hstr(b"application/grpc")
    ua_dyn = _hint(62, 4, 0x00) + _hstr(b"anything")                   # dynamic 0: user-agent (ignorable)
    m = request_bytes("hp", 5, 10, 60, 1)
    hdr = lambda blk: lambda sid: _frames(sid, blk, m)            # noqa: E731
    prio = lambda payload: lambda sid: gt.frame(gt.HEADERS, gt.END_HEADERS | gt.PRIO, sid, payload) + \
        gt.frame(gt.DATA, gt.END_STREAM, sid, b"\0" + struct.pack(">I", len(m)) + m)   # noqa: E731
    return [
        ("2-byte dynamic indices", hdr(DYN_BLOCK + b"\xbe"), True),
        ("dynamic index 62 + n_dyn", hdr(DYN_BLOCK + _hint(190, 7, 0x80)), False),
        ("index above 2^21", hdr(DYN_BLOCK + b"\xff\x80\x80\x80\x01"), False),
        ("3-byte index past the table", hdr(DYN_BLOCK + b"\xff\xff\xff\x7f"), False),
        ("literal names: static 31, 58, dynamic", hdr(b"\x83" + _hint(188, 4, 0x00) + _hstr(gt.PATH) + ctype
                                                      + _hint(58, 4, 0x00) + _hstr(b"x") + ua_dyn), True),
        ("never-indexed dynamic names", hdr(b"\x83" + _hint(188, 4, 0x10) + _hstr(gt.PATH) + _hint(189, 4, 0x10)
                                            + _hstr(b"application/grpc+proto")), True),
        ("literal name at n_dyn", hdr(DYN_BLOCK + _hint(190, 4, 0x00) + _hstr(b"x")), False),
        ("huffman values on ignorable names", hdr(DYN_BLOCK + b"\x00\x03x-h" + _hstr(b"abc", True)
                                                  + _hint(58, 4, 0x00) + _hstr(b"grpc/1", True)
                                                  + _hint(62, 4, 0x10) + _hstr(b"zz", True)), True),
        ("huffman :path, static name", hdr(b"\x83" + _hint(4, 4, 0x00) + _hstr(gt.PATH, True)
                                           + _hint(189, 7, 0x80)), False),
        ("huffman :path, dynamic name", hdr(b"\x83" + _hint(188, 4, 0x00) + _hstr(gt.PATH, True)
                                            + _hint(189, 7, 0x80)), False),
        ("huffman content-type", hdr(b"\x83" + _hint(188, 7, 0x80) + _hint(31, 4, 0x00)
                                     + _hstr(b"application/grpc", True)), False),
        ("priority, 5 bytes and a block", prio(b"\0\0\0\x03\x10" + DYN_BLOCK), True),
        ("priority, exactly 5 bytes", prio(b"\0\0\0\0\x0f"), False),
        ("priority, 4 bytes", prio(b"\0\0\0\0"), False),
        ("headers of 16384 bytes", hdr(_pad_block(16384)), True),
        ("headers of 16385 bytes", hdr(_pad_block(16385)), False),
    ]


def _hpack_conns():
    out = []
    for i, (name, call, plain) in enumerate(_hpack_cases()):
        last = 100_001 + 1000 * i
        k = i % 4
        pre = b"".join(_frames(last + 2 + 2 * j, DYN_BLOCK, request_bytes("hp%d" % j, 5, 10, 60, 1))
                       for j in range(k))
        sid = last + 2 + 2 * k
        data = pre + call(sid) + _frames(sid + 2, DYN_BLOCK, request_bytes("hp", 5, 10, 60, 1))
        out.append((name, data, _dyn_row(last), (0, k + 2) if plain else (2, k), len(pre)))
    return out


@KINDS
@SEEDS
def test_hpack_forms_grpcio_never_sends(kind, seed):
    cases = _hpack_conns()
    rig = Rig(kind, seed)
    got, _, _ = _serve(rig, _grpc([(d, st) for _, d, st, _, _ in cases], kind))
    for (name, data, _, want, pre), (o, _, sids, _) in zip(cases, got):
        assert (int(o["stop"]), int(o["n_frames"])) == want, name
        assert int(o["consumed"]) == (len(data) if want[0] == 0 else pre), name
        assert all(s > 0xffff for s in sids)


# ---- 3. protobuf forms prost accepts -------------------------------------------------------------------------------
STD = _num(2, 2) + _num(3, 10) + _num(4, 60) + _num(5, 1)          # burst 2: a key's third and fourth calls are denied


def _proto_cases():
    """(name, message): every key is sent four times"""
    neg = _varint(-1)
    assert len(neg) == 10
    return [
        ("reverse order", _num(5, 1) + _num(4, 60) + _num(3, 10) + _num(2, 2) + _key(b"rev")),
        ("duplicates, the last wins", _key(b"first") + _num(2, 9) + _num(3, 10) + _key("sécond".encode())
         + _num(4, 60) + _num(2, 2) + _num(5, 1)),
        ("negative max_burst", _key(b"n2") + b"\x10" + neg + _num(3, 10) + _num(4, 60) + _num(5, 1)),
        ("negative count", _key(b"n3") + _num(2, 2) + b"\x18" + neg + _num(4, 60) + _num(5, 1)),
        ("negative period", _key(b"n4") + _num(2, 2) + _num(3, 10) + b"\x20" + neg + _num(5, 1)),
        ("negative quantity", _key(b"n5") + _num(2, 2) + _num(3, 10) + _num(4, 60) + b"\x28" + neg),
        ("2^32 + 5 is 5", _key(b"trunc") + _num(2, 2) + _num(3, 2**32 + 5) + _num(4, 60) + _num(5, 2**32 + 1)),
        ("unknown fields", _unknown(2**29 - 1, 0, _varint(2**63)) + _key(b"unk") + _unknown(6, 1, b"\xff" * 8)
         + _unknown(2**29 - 2, 2, _varint(3) + b"\x0a\x01k") + STD + _unknown(2**28, 5, b"\0" * 4)),
        ("key of 0 bytes", STD + _key(b"")),
        ("key of 1 byte", STD + _key(b"z")),
        ("key of 256 bytes", STD + _key("é".encode() * 128)),
        ("key of 257 bytes", STD + _key(b"a" + "é".encode() * 128)),
        ("key of 16000 bytes", STD + _key("é".encode() * 8000)),
        ("empty message", b""),
    ]


@KINDS
@SEEDS
def test_protobuf_forms_and_denied_names(kind, seed):
    rig = Rig(kind, seed)
    lim = rig.lim
    lim.store.track_denied(1024)
    lim.store.ring_metrics(True)
    conns, key_of = [], {}
    for i, (name, msg) in enumerate(_proto_cases()):
        row = gs.established().conn_row()
        row["last_stream"] = 70_001 + 2 * i
        blk = gs.steady_block(gs.established().hpack)
        data = b"".join(gs.call(70_003 + 2 * i + 2 * j, blk, msg) for j in range(4))
        conns.append((data, row))
        key_of[lim.store.hash_key(gt.decode_request(msg)[0])] = gt.decode_request(msg)[0]
    got, _, _ = _serve(rig, _grpc(conns, kind))
    assert all((int(o["stop"]), int(o["n_frames"])) == (0, 4) for o, *_ in got)
    lim.store.sync()
    top, dropped = lim.store.top_denied(4096)
    assert dropped == 0 and dict(top) == rig.denied_by_hash
    names = dict(zip([h for h, _ in top], lim.store.denied_names([h for h, _ in top])))
    for k in (b"rev", "sécond".encode(), b"trunc", b"unk", b"", b"z", "é".encode() * 128, b"a" + "é".encode() * 128,
              "é".encode() * 8000):
        h = lim.store.hash_key(k)
        assert rig.denied_by_hash.get(h) == 2, k[:20]
        assert names[h] == (tc.NAME_TOO_LONG if len(k) > tc.DENIED_NAME_MAX else k), (k[:20], names[h])
    for h, nm in names.items():                                 # (and nothing else: no filler key is denied)
        assert nm == (tc.NAME_TOO_LONG if len(key_of[h]) > tc.DENIED_NAME_MAX else key_of[h])


# ---- 4. shared-memory bounds: 65,536-byte connections ------------------------------------------------------------------
def _min_call(sid):
    """26 bytes: HEADERS(0x83, dynamic :path and content-type) and DATA(END_STREAM) of an empty message"""
    return gt.frame(gt.HEADERS, gt.END_HEADERS, sid, b"\x83\xbe\xbf") + gt.frame(gt.DATA, gt.END_STREAM, sid,
                                                                                 b"\0" * 5)


def _bound_conns():
    """(name, bytes, row, (stop, n_frames, consumed))"""
    out = []
    empty = b"".join(gt.frame(gt.HEADERS if f % 2 == 0 else gt.DATA, gt.END_HEADERS, 3 + 2 * (f // 2))
                     for f in range(7281))
    cn = gs.established()
    out.append(("7281 empty frames", empty + b"\0" * 7, cn.conn_row(), (2, 0, 0)))
    calls = gs.steady_stream(random.Random(4), cn, 3, ["b:0", "b:1"], extras=False)
    rest = 65536 - len(calls)
    tail = b"".join(gt.frame(gt.DATA if f % 2 else gt.HEADERS, gt.END_HEADERS, 101) for f in range(rest // 9))
    out.append(("3 calls and empty frames", calls + tail + b"\0" * (rest % 9), cn.conn_row(), (2, 3, len(calls))))
    wu = gt.frame(gt.WINDOW_UPDATE, 0, 0, b"\0\0\0\x01") * 5041
    out.append(("5041 window updates", wu + b"\0\0\0", cn.conn_row(), (1, 0, 65533)))
    row = cn.conn_row()
    row["n_dyn"], row["dyn_class"][0], row["dyn_class"][1] = 2, PATH_CLS, CTYPE_CLS
    row["send_window"], row["init_window"], row["last_stream"] = 2**31 - 1, 51, 2**31 - 1 - 2 * 2530
    sid0 = int(row["last_stream"]) + 2
    mins = b"".join(_min_call(sid0 + 2 * j) for j in range(2521))[:65536]
    out.append(("2520 minimal calls", mins, row, (1, 2520, 2520 * 26)))
    cn = gs.established()
    blk = gs.steady_block(cn.hpack)
    full = []
    for j in range(4):
        k = ("full%d:" % j).encode()
        msg = _key(k + b"f" * (16379 - 3 - len(k) - 6)) + _num(2, 1) + _num(3, 10) + _num(4, 60)
        assert len(msg) == 16379
        full.append(gs.call(3 + 2 * j, blk, msg))
    big = b"".join(full)
    assert len(big) > 65536 > len(big) - len(full[3]) + 9
    out.append(("16384-byte DATA frames", big[:65536], cn.conn_row(), (1, 3, len(big) - len(full[3]))))
    assert all(len(d) == 65536 for _, d, _, _ in out)
    return out


def _ends_at_segment_end():
    """(bytes, row, stop): one plain call, then a HEADERS frame (frame 4) or a call's DATA frame (frame 5) that ends
    exactly at the connection's end.  Each such connection follows 1000 whose frame at that index ends one byte before
    their end and is judged the other way, so a parse CTA that missed the frame at the end would find their judgement
    in its frame list, not its own."""
    cn = gs.established()
    blk = gs.steady_block(cn.hpack)
    one = gs.call(3, blk, request_bytes("end", 5, 10, 60, 1))
    good = gt.frame(gt.HEADERS, gt.END_HEADERS, 5, blk)
    bad = gt.frame(gt.HEADERS, gt.END_HEADERS, 5, blk + b"\x8d")               # :status: not plain
    msg = request_bytes("end", 5, 10, 60, 1)
    data = gt.frame(gt.DATA, gt.END_STREAM, 5, b"\0" + struct.pack(">I", len(msg)) + msg)
    no = NEAR_MISSES["wire 6"]
    zdata = gt.frame(gt.DATA, gt.END_STREAM, 5, b"\0" + struct.pack(">I", len(no)) + no)    # prost refuses it
    # (the connections before: frame, stop) and (the connection at the end: frame, stop)
    blocks = [((bad + b"\0", 2), (good, 1)), ((good + b"\0", 1), (bad, 2)),
              ((good + zdata + b"\0", 2), (good + data, 0)), ((good + data + b"\0", 1), (good + zdata, 2))]
    out = []
    for (before, s0), (end, s1) in blocks:
        out += [(one + before, cn.conn_row(), s0)] * 1000 + [(one + end, cn.conn_row(), s1)] * 8
    return out


@KINDS
def test_shared_memory_bounds(kind):
    cases = _bound_conns()
    rig = Rig(kind, SIP, row_capacity=4096, max_conns=16, in_capacity=1 << 20)
    got, _, _ = _serve(rig, _grpc([(d, st) for _, d, st, _ in cases], kind))
    for (name, _, _, want), (o, _, sids, _) in zip(cases, got):
        assert (int(o["stop"]), int(o["n_frames"]), int(o["consumed"])) == want, name
    assert int(got[2][0]["send_window"]) == 65535 + 5041
    assert int(got[3][2][-1]) == 2**31 - 1 - 2 * 2530 + 2 * 2520

    ends = _ends_at_segment_end()
    rig = Rig(kind, SIP, row_capacity=8192, max_conns=2 * len(ends), in_capacity=1 << 22)
    got, _, _ = _serve(rig, _grpc([(d, st) for d, st, _ in ends], kind, between=False))
    assert [int(o["stop"]) for o, *_ in got] == [s for _, _, s in ends]


# ---- 5. the row cap and the re-walk ---------------------------------------------------------------------------------
K = 5


def _capped_conns():
    """A: K plain calls, a PING before the last, then a HEADERS that is not plain; B: 3 plain calls; C: a PING and 2
    plain calls; D: SETTINGS, then a plain call"""
    cn = gs.established()
    blk = gs.steady_block(cn.hpack)
    msg = lambda k: request_bytes("cap:%s" % k, 5, 10, 60, 1)     # noqa: E731
    a = b"".join(gs.call(3 + 2 * j, blk, msg("a")) for j in range(K - 1))
    ping_at = len(a)
    a += gt.frame(gt.PING, 0, 0, b"pingpong") + gs.call(3 + 2 * (K - 1), blk, msg("a"))
    a += gs.call(3 + 2 * K, blk + gs.lit(b"x-a", b"b", 0x40), msg("a"))
    b = b"".join(gs.call(3 + 2 * j, blk, msg("b")) for j in range(3))
    c = gt.frame(gt.PING, 0, 0, b"\1" * 8) + b"".join(gs.call(3 + 2 * j, blk, msg("c")) for j in range(2))
    d = gt.frame(gt.SETTINGS, 0, 0) + gs.call(3, blk, msg("d"))
    return [(x, cn.conn_row()) for x in (a, b, c, d)], ping_at


@KINDS
@pytest.mark.parametrize("cap", [K - 1, K, K + 1])
def test_row_cap_and_the_rewalk(kind, cap):
    conns, ping_at = _capped_conns()
    rig = Rig(kind, SIP, row_capacity=cap, max_conns=16)
    got, _, _ = _serve(rig, _grpc(conns, kind))
    a, b, c, d = (g[0] for g in got)
    one = len(gs.call(3, gs.steady_block(gs.established().hpack), request_bytes("cap:a", 5, 10, 60, 1)))
    want_a = {K - 1: (3, K - 1, ping_at + 17), K: (3, K, ping_at + 17 + one), K + 1: (2, K, ping_at + 17 + one)}[cap]
    assert (int(a["stop"]), int(a["n_frames"]), int(a["consumed"]), int(a["ping"])) == (*want_a, 1)
    if cap <= K:                                              # room 0 for every later connection
        assert [(int(o["stop"]), int(o["n_frames"]), int(o["consumed"])) for o in (b, c, d)] == \
            [(3, 0, 0), (3, 0, 17), (2, 0, 0)]
        assert int(c["ping"]) == 1 and bytes(c["ping_opaque"]) == b"\1" * 8
    elif kind == "grpc":                                      # (on a mixed ring a filler takes the one row left)
        assert (int(b["stop"]), int(b["n_frames"])) == (3, 1)


# ---- 6. reply tiles ---------------------------------------------------------------------------------------------------
ROWS = {"decide error": lambda i: request_bytes("neg%d" % i, 5, 10, 60, -2**31),
        "invalid parameters": lambda i: request_bytes("inv%d" % i, -1, 0, -1, 1),
        "ok": lambda i: request_bytes("ok%d" % (i % 7), 2**31 - 1, 3, 2**31 - 1, 1 + i % 3)}


@KINDS
@pytest.mark.parametrize("what", sorted(ROWS))
def test_reply_tiles(kind, what):
    rig = Rig(kind, SIP, row_capacity=8192, max_conns=64, in_capacity=1 << 21)
    try:
        Resp = _pb_module()
    except pytest.skip.Exception:
        Resp = None
    status = set()
    for n in (255, 256, 257, 4097):
        conns, sid = [], 2**31 - 1 - 2 * 5000
        for lo in range(0, n, 500):
            cn = gs.established()
            row = cn.conn_row()
            row["last_stream"] = sid
            blk = gs.steady_block(cn.hpack)
            data = b"".join(gs.call(sid + 2 * (j + 1), blk, ROWS[what](lo + j)) for j in range(min(500, n - lo)))
            conns.append((data, row))
        got, _, _ = _serve(rig, _grpc(conns, kind, between=False))          # (the gRPC rows first: tiles as named)
        assert sum(len(g[1]) for g in got) == n
        for c, (o, rows, sids, res) in enumerate(got):
            g = rig.ring.outcome[0][c] if kind == "grpc" else rig.ring.grpc_outcome[0][c]
            want, sent = b"", 0
            for i, s in enumerate(sids):
                q, r = rows[i], res[i]
                b, m = _py_reply(q, r, int(s))
                want += b
                status.add(int(r["status"]))
                if m is not None:
                    sent += 5 + len(m)
                    if Resp is not None:
                        p = Resp.FromString(m)
                        assert (p.allowed, p.limit, p.remaining) == (bool(r["allowed"]), 2**31 - 1,
                                                                     gt._i32(int(r["remaining"])))
            off, ln = int(g["reply_off"]), int(g["reply_len"])
            assert rig.ring.replies[0][off:off + ln].tobytes() == want and int(g["data_sent"]) == sent
    assert status == {"decide error": {tc.NEGATIVE_QUANTITY}, "invalid parameters": {tc.INVALID_RATE_LIMIT},
                      "ok": {tc.OK}}[what]


# ---- 7. 65,536 connections in one submit ------------------------------------------------------------------------------
def test_65536_connections_with_one_call_each():
    rng = np.random.default_rng(65536)
    n = 65536
    keys = np.minimum(rng.zipf(1.3, n), 5000)
    lasts = rng.integers(0, 2**31 - 3, n)
    lasts[:64] = 2**31 - 3
    blk = gs.steady_block(gs.established().hpack)
    base_row = gs.established().conn_row()
    conns = []
    for i in range(n):
        last = int(lasts[i])
        sid = last + 2 if last % 2 else last + 1
        data = bytearray(gs.call(sid, blk, request_bytes("z%d" % keys[i], 3, 10, 60, 1)))
        if i % 97 == 5:
            data[5] |= 0x80                                   # the reserved bit on the HEADERS' stream id
        row = base_row.copy()
        row["last_stream"] = last
        row["send_window"] = 51 if i % 13 == 1 else 50 if i % 13 == 2 else 65535
        conns.append(("grpc", bytes(data), row))
    rig = Rig("grpc", SIP, row_capacity=n, max_conns=n, in_capacity=1 << 24)
    got, rows, _ = _serve(rig, conns)
    stops = [int(o["stop"]) for o, *_ in got]
    assert stops.count(2) == len(range(2, n, 13)) and len(rows) == n - stops.count(2)
    assert int(got[5][0]["n_frames"]) == 1 and int(got[5][2][0]) == int(lasts[5]) + 1 + int(lasts[5]) % 2
    assert max(int(s) for _, _, sids, _ in got for s in sids) == 2**31 - 1


# ---- 8. the whole driver against the general path ----------------------------------------------------------------------
def _driver_conns():
    """about 60 Connections: the cases of 1 and 3 among plain calls, each connection on keys of its own"""
    out = []
    for name, data, row, _, _, _ in _host_edge_conns():
        cn = gs.established()
        if name == "oldest dynamic entry":
            cn.hpack = gt.Decoder()
            cn.hpack.decode(gs.lit(b"x-first", b"1", 0x40) + gs.first_block())
        cn.last_stream, cn.send_window, cn.init_window = \
            int(row["last_stream"]), int(row["send_window"]), int(row["init_window"])
        assert bytes(cn.conn_row()) == bytes(row), name
        cn.buf += data
        out.append(cn)
    for i, (_, msg) in enumerate(_proto_cases()):
        cn = gs.established()
        blk = gs.steady_block(cn.hpack)
        cn.buf += gs.call(3, blk, request_bytes("drv%d" % i, 2, 10, 60, 1)) + \
            b"".join(gs.call(5 + 2 * j, blk, msg) for j in range(3))
        out.append(cn)
    for i in range(6):
        cn = gs.established()
        cn.buf += gs.steady_stream(random.Random(i), cn, 10, ["plain%d" % i])
        out.append(cn)
    return out


def _frames_of(out):
    """(every frame but WINDOW_UPDATE and PING ACK, in order; WINDOW_UPDATE totals per stream id; PING ACKs in order)"""
    frames, wu, acks, i = [], {}, [], 0
    while i < len(out):
        n = int.from_bytes(out[i:i + 3], "big")
        f = bytes(out[i:i + 9 + n])
        if f[3] == gt.WINDOW_UPDATE:
            sid = int.from_bytes(f[5:9], "big")
            wu[sid] = wu.get(sid, 0) + int.from_bytes(f[9:13], "big")
        elif f[3] == gt.PING:
            acks.append(f)
        else:
            frames.append(f)
        i += 9 + n
    return frames, wu, acks


def _split_streams(data):
    """the streams whose request has a non-empty DATA frame without END_STREAM"""
    out, i = set(), 0
    while len(data) - i >= 9:
        n = int.from_bytes(data[i:i + 3], "big")
        if data[i + 3] == gt.DATA and n and not data[i + 4] & gt.END_STREAM:
            out.add(int.from_bytes(data[i + 5:i + 9], "big") & 0x7fffffff)
        i += 9 + n
    return out


@pytest.mark.parametrize("seed", [(0, 0), SIP], ids=["unkeyed", "siphash"])
def test_driver_against_the_general_path(seed):
    """The same frames, in the same order, but for WINDOW_UPDATE and PING ACK: a ring walk sends its connection update
    and its PING ACK after its calls' responses (Connection.take_outcome), the general path as each frame arrives, so
    those are compared as totals per stream and as the ACKs in order.  The one difference allowed: the general path
    opens a stream's window after each DATA frame that does not end the stream; a walk takes a call only whole, with
    its END_STREAM, so it sends no update for a stream whose request it has already read to the end."""
    conns, twins = _driver_conns(), _driver_conns()
    assert len(conns) >= 60
    inputs = [bytes(b.buf) for b in twins]
    lim = tc.RateLimiter(tc.ManualStore(capacity=1 << 14, created_ns=NOW, max_batch=1 << 14, hash_seed=seed))
    twin = tc.RateLimiter(tc.ManualStore(capacity=1 << 14, created_ns=NOW, max_batch=1 << 14, hash_seed=seed))
    ring = tc.GrpcRing(lim, 1, 128, 1 << 22, 4096)
    counts = gt.process_connections(conns, lim, NOW, ring)
    for b in twins:
        while b.buf and not b.closed:
            had = len(b.buf)
            b.general(twin, NOW)
            if len(b.buf) == had:
                break
    skipped = 0
    for i, (a, b) in enumerate(zip(conns, twins)):
        assert counts[i] == b.n_throttle and a.closed == b.closed and a.last_stream == b.last_stream, i
        fa, wa, pa = _frames_of(a.out)
        fb, wb, pb = _frames_of(b.out)
        assert fa == fb and pa == pb, i
        split = _split_streams(inputs[i])
        for sid in set(wa) | set(wb):
            if wa.get(sid) != wb.get(sid):
                assert sid in split and sid not in wa, (i, sid, wa.get(sid), wb.get(sid))
                skipped += 1
    assert skipped > 0                                        # (the split calls some walk took)
    assert sum(counts) > 100 and any(a.closed for a in conns)
    sa, sb = lim.store.stats(), twin.store.stats()
    assert (sa["allowed"], sa["denied"], sa["errors"]) == (sb["allowed"], sb["denied"], sb["errors"])
