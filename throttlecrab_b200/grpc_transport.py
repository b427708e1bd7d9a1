"""gRPC ingest for the batched engine: the general HTTP/2 path beside the GPU's fast path.

Serves the reference's gRPC transport (throttlecrab-server/src/transport/grpc.rs, proto/throttlecrab.proto): the
unary call /throttlecrab.RateLimiter/Throttle over cleartext HTTP/2 (no TLS, no ALPN).  Plain calls go to a GrpcRing
(gcra_grpc.cuh defines "plain"); everything else comes here:

- the connection preface and SETTINGS (acknowledged), PING, RST_STREAM, GOAWAY, CONTINUATION, PRIORITY;
- an HPACK decoder (RFC 7541) with the dynamic table and Huffman decoding, which also writes the class bytes the GPU
  walk reads (gcra_grpc_header_class of each entry);
- stream and flow-control state, interleaved streams, messages over several DATA frames, responses queued until the
  peer's windows take them;
- gRPC statuses: UNIMPLEMENTED (12) for another path or an unknown grpc-encoding, INTERNAL (13) with the reference's
  text for a decide error and with this module's own detail text for a message prost would not decode;
- RFC 9113 connection errors (PROTOCOL_ERROR, COMPRESSION_ERROR, FLOW_CONTROL_ERROR, FRAME_SIZE_ERROR) as GOAWAY, and
  the connection closes.

Responses are written without HPACK state (literals without indexing), as gcra_grpc_format_replies writes them.
"""
import ctypes as C
import struct

import numpy as np

from . import REQ_DTYPE, RES_DTYPE, GRPC_REPLY_MAX, GRPC_MAX_DYN, OK, _native
from .metrics import Metrics

PREFACE = b"PRI * HTTP/2.0\r\n\r\nSM\r\n\r\n"
PATH = b"/throttlecrab.RateLimiter/Throttle"
DATA, HEADERS, PRIORITY, RST_STREAM, SETTINGS, PUSH_PROMISE, PING, GOAWAY, WINDOW_UPDATE, CONTINUATION = range(10)
END_STREAM, ACK, END_HEADERS, PADDED, PRIO = 0x1, 0x1, 0x4, 0x8, 0x20
NO_ERROR, PROTOCOL_ERROR, FLOW_CONTROL_ERROR, STREAM_CLOSED, FRAME_SIZE_ERROR, COMPRESSION_ERROR = 0, 1, 3, 5, 6, 9
MAX_WINDOW = 2**31 - 1
MAX_FRAME = 16384
TABLE_SIZE = 4096                    # SETTINGS_HEADER_TABLE_SIZE this server keeps (the default: never raised)
MAX_MESSAGE = 4 * 1024 * 1024        # the largest request message decoded (tonic's default decoding limit)

STATIC = [(b":authority", b""), (b":method", b"GET"), (b":method", b"POST"), (b":path", b"/"),
          (b":path", b"/index.html"), (b":scheme", b"http"), (b":scheme", b"https"), (b":status", b"200"),
          (b":status", b"204"), (b":status", b"206"), (b":status", b"304"), (b":status", b"400"),
          (b":status", b"404"), (b":status", b"500"), (b"accept-charset", b""),
          (b"accept-encoding", b"gzip, deflate"), (b"accept-language", b""), (b"accept-ranges", b""),
          (b"accept", b""), (b"access-control-allow-origin", b""), (b"age", b""), (b"allow", b""),
          (b"authorization", b""), (b"cache-control", b""), (b"content-disposition", b""),
          (b"content-encoding", b""), (b"content-language", b""), (b"content-length", b""),
          (b"content-location", b""), (b"content-range", b""), (b"content-type", b""), (b"cookie", b""),
          (b"date", b""), (b"etag", b""), (b"expect", b""), (b"expires", b""), (b"from", b""), (b"host", b""),
          (b"if-match", b""), (b"if-modified-since", b""), (b"if-none-match", b""), (b"if-range", b""),
          (b"if-unmodified-since", b""), (b"last-modified", b""), (b"link", b""), (b"location", b""),
          (b"max-forwards", b""), (b"proxy-authenticate", b""), (b"proxy-authorization", b""), (b"range", b""),
          (b"referer", b""), (b"refresh", b""), (b"retry-after", b""), (b"server", b""), (b"set-cookie", b""),
          (b"strict-transport-security", b""), (b"transfer-encoding", b""), (b"user-agent", b""), (b"vary", b""),
          (b"via", b""), (b"www-authenticate", b"")]

# RFC 7541 Appendix B: (code, bit length) of symbols 0..255 and EOS (256), transcribed from the RFC.  The tests
# check that it is a complete prefix code (Kraft sum exactly 1) and canonical, and decode the RFC's examples.
HUFFMAN = [
    (0x1ff8, 13), (0x7fffd8, 23), (0xfffffe2, 28), (0xfffffe3, 28), (0xfffffe4, 28), (0xfffffe5, 28),
    (0xfffffe6, 28), (0xfffffe7, 28), (0xfffffe8, 28), (0xffffea, 24), (0x3ffffffc, 30), (0xfffffe9, 28),
    (0xfffffea, 28), (0x3ffffffd, 30), (0xfffffeb, 28), (0xfffffec, 28), (0xfffffed, 28), (0xfffffee, 28),
    (0xfffffef, 28), (0xffffff0, 28), (0xffffff1, 28), (0xffffff2, 28), (0x3ffffffe, 30), (0xffffff3, 28),
    (0xffffff4, 28), (0xffffff5, 28), (0xffffff6, 28), (0xffffff7, 28), (0xffffff8, 28), (0xffffff9, 28),
    (0xffffffa, 28), (0xffffffb, 28), (0x14, 6), (0x3f8, 10), (0x3f9, 10), (0xffa, 12), (0x1ff9, 13), (0x15, 6),
    (0xf8, 8), (0x7fa, 11), (0x3fa, 10), (0x3fb, 10), (0xf9, 8), (0x7fb, 11), (0xfa, 8), (0x16, 6), (0x17, 6),
    (0x18, 6), (0x0, 5), (0x1, 5), (0x2, 5), (0x19, 6), (0x1a, 6), (0x1b, 6), (0x1c, 6), (0x1d, 6), (0x1e, 6),
    (0x1f, 6), (0x5c, 7), (0xfb, 8), (0x7ffc, 15), (0x20, 6), (0xffb, 12), (0x3fc, 10), (0x1ffa, 13), (0x21, 6),
    (0x5d, 7), (0x5e, 7), (0x5f, 7), (0x60, 7), (0x61, 7), (0x62, 7), (0x63, 7), (0x64, 7), (0x65, 7), (0x66, 7),
    (0x67, 7), (0x68, 7), (0x69, 7), (0x6a, 7), (0x6b, 7), (0x6c, 7), (0x6d, 7), (0x6e, 7), (0x6f, 7), (0x70, 7),
    (0x71, 7), (0x72, 7), (0xfc, 8), (0x73, 7), (0xfd, 8), (0x1ffb, 13), (0x7fff0, 19), (0x1ffc, 13),
    (0x3ffc, 14), (0x22, 6), (0x7ffd, 15), (0x3, 5), (0x23, 6), (0x4, 5), (0x24, 6), (0x5, 5), (0x25, 6),
    (0x26, 6), (0x27, 6), (0x6, 5), (0x74, 7), (0x75, 7), (0x28, 6), (0x29, 6), (0x2a, 6), (0x7, 5), (0x2b, 6),
    (0x76, 7), (0x2c, 6), (0x8, 5), (0x9, 5), (0x2d, 6), (0x77, 7), (0x78, 7), (0x79, 7), (0x7a, 7), (0x7b, 7),
    (0x7ffe, 15), (0x7fc, 11), (0x3ffd, 14), (0x1ffd, 13), (0xffffffc, 28), (0xfffe6, 20), (0x3fffd2, 22),
    (0xfffe7, 20), (0xfffe8, 20), (0x3fffd3, 22), (0x3fffd4, 22), (0x3fffd5, 22), (0x7fffd9, 23),
    (0x3fffd6, 22), (0x7fffda, 23), (0x7fffdb, 23), (0x7fffdc, 23), (0x7fffdd, 23), (0x7fffde, 23),
    (0xffffeb, 24), (0x7fffdf, 23), (0xffffec, 24), (0xffffed, 24), (0x3fffd7, 22), (0x7fffe0, 23),
    (0xffffee, 24), (0x7fffe1, 23), (0x7fffe2, 23), (0x7fffe3, 23), (0x7fffe4, 23), (0x1fffdc, 21),
    (0x3fffd8, 22), (0x7fffe5, 23), (0x3fffd9, 22), (0x7fffe6, 23), (0x7fffe7, 23), (0xffffef, 24),
    (0x3fffda, 22), (0x1fffdd, 21), (0xfffe9, 20), (0x3fffdb, 22), (0x3fffdc, 22), (0x7fffe8, 23),
    (0x7fffe9, 23), (0x1fffde, 21), (0x7fffea, 23), (0x3fffdd, 22), (0x3fffde, 22), (0xfffff0, 24),
    (0x1fffdf, 21), (0x3fffdf, 22), (0x7fffeb, 23), (0x7fffec, 23), (0x1fffe0, 21), (0x1fffe1, 21),
    (0x3fffe0, 22), (0x1fffe2, 21), (0x7fffed, 23), (0x3fffe1, 22), (0x7fffee, 23), (0x7fffef, 23),
    (0xfffea, 20), (0x3fffe2, 22), (0x3fffe3, 22), (0x3fffe4, 22), (0x7ffff0, 23), (0x3fffe5, 22),
    (0x3fffe6, 22), (0x7ffff1, 23), (0x3ffffe0, 26), (0x3ffffe1, 26), (0xfffeb, 20), (0x7fff1, 19),
    (0x3fffe7, 22), (0x7ffff2, 23), (0x3fffe8, 22), (0x1ffffec, 25), (0x3ffffe2, 26), (0x3ffffe3, 26),
    (0x3ffffe4, 26), (0x7ffffde, 27), (0x7ffffdf, 27), (0x3ffffe5, 26), (0xfffff1, 24), (0x1ffffed, 25),
    (0x7fff2, 19), (0x1fffe3, 21), (0x3ffffe6, 26), (0x7ffffe0, 27), (0x7ffffe1, 27), (0x3ffffe7, 26),
    (0x7ffffe2, 27), (0xfffff2, 24), (0x1fffe4, 21), (0x1fffe5, 21), (0x3ffffe8, 26), (0x3ffffe9, 26),
    (0xffffffd, 28), (0x7ffffe3, 27), (0x7ffffe4, 27), (0x7ffffe5, 27), (0xfffec, 20), (0xfffff3, 24),
    (0xfffed, 20), (0x1fffe6, 21), (0x3fffe9, 22), (0x1fffe7, 21), (0x1fffe8, 21), (0x7ffff3, 23),
    (0x3fffea, 22), (0x3fffeb, 22), (0x1ffffee, 25), (0x1ffffef, 25), (0xfffff4, 24), (0xfffff5, 24),
    (0x3ffffea, 26), (0x7ffff4, 23), (0x3ffffeb, 26), (0x7ffffe6, 27), (0x3ffffec, 26), (0x3ffffed, 26),
    (0x7ffffe7, 27), (0x7ffffe8, 27), (0x7ffffe9, 27), (0x7ffffea, 27), (0x7ffffeb, 27), (0xffffffe, 28),
    (0x7ffffec, 27), (0x7ffffed, 27), (0x7ffffee, 27), (0x7ffffef, 27), (0x7fffff0, 27), (0x3ffffee, 26),
    (0x3fffffff, 30)]
_HUFF_DECODE = {(code, n): sym for sym, (code, n) in enumerate(HUFFMAN)}


class ConnectionError_(Exception):
    """an RFC 9113 connection error: GOAWAY with `code`, then close"""

    def __init__(self, code, msg=""):
        super().__init__(msg)
        self.code = code


def huffman_decode(data):
    """RFC 7541 5.2: padding is at most 7 bits, all ones; EOS inside the string is an error"""
    out, code, n = bytearray(), 0, 0
    for b in data:
        for k in range(7, -1, -1):
            code, n = code << 1 | (b >> k & 1), n + 1
            sym = _HUFF_DECODE.get((code, n))
            if sym is not None:
                if sym == 256:
                    raise ConnectionError_(COMPRESSION_ERROR, "EOS in a Huffman string")
                out.append(sym)
                code, n = 0, 0
            elif n > 30:
                raise ConnectionError_(COMPRESSION_ERROR, "not a Huffman code")
    if n > 7 or code != (1 << n) - 1:
        raise ConnectionError_(COMPRESSION_ERROR, "bad Huffman padding")
    return bytes(out)


def huffman_encode(data):
    acc, n = 0, 0
    for b in data:
        code, k = HUFFMAN[b]
        acc, n = acc << k | code, n + k
    pad = -n % 8
    acc, n = acc << pad | ((1 << pad) - 1), n + pad
    return acc.to_bytes(n // 8, "big")


def header_class(name, value=None):
    """gcra_grpc_header_class: the class of a field, or of a name alone (value None)"""
    L = _native.lib()
    return L.gcra_grpc_header_class(name, len(name), value, 0 if value is None else len(value))


def class_byte(name, value):
    """the class byte of a dynamic-table entry, as gcra_grpc_conn.dyn_class holds it"""
    return header_class(name, value) | header_class(name) << 4


# ---- HPACK -------------------------------------------------------------------------------------------------------
def _int(b, i, bits):
    if i >= len(b):
        raise ConnectionError_(COMPRESSION_ERROR, "truncated integer")
    mask = (1 << bits) - 1
    v = b[i] & mask
    i += 1
    if v < mask:
        return v, i
    m = 0
    while True:
        if i >= len(b) or m > 28:
            raise ConnectionError_(COMPRESSION_ERROR, "bad integer")
        v += (b[i] & 0x7f) << m
        m += 7
        i += 1
        if not b[i - 1] & 0x80:
            return v, i


def _str(b, i):
    huff = i < len(b) and b[i] & 0x80
    n, i = _int(b, i, 7)
    if n > len(b) - i:
        raise ConnectionError_(COMPRESSION_ERROR, "truncated string")
    s = bytes(b[i:i + n])
    return (huffman_decode(s) if huff else s), i + n


class Decoder:
    """RFC 7541 decoder with its dynamic table (newest first) and the entries' class bytes"""

    def __init__(self, max_size=TABLE_SIZE):
        self.table, self.size, self.max_size, self.limit = [], 0, max_size, max_size
        self.cls = []                  # the entries' class bytes, kept in step with the table

    def _get(self, idx):
        if idx == 0:
            raise ConnectionError_(COMPRESSION_ERROR, "index 0")
        if idx <= len(STATIC):
            return STATIC[idx - 1]
        if idx - 62 < len(self.table):
            return self.table[idx - 62]
        raise ConnectionError_(COMPRESSION_ERROR, "index %d beyond the table" % idx)

    def _evict(self):
        while self.size > self.max_size:
            n, v = self.table.pop()
            self.cls.pop()
            self.size -= 32 + len(n) + len(v)

    def _add(self, n, v):
        self.table.insert(0, (n, v))
        self.cls.insert(0, class_byte(n, v))
        self.size += 32 + len(n) + len(v)
        self._evict()

    def decode(self, block):
        out, i, first = [], 0, True
        b = bytes(block)
        while i < len(b):
            c = b[i]
            if c & 0x80:
                idx, i = _int(b, i, 7)
                out.append(self._get(idx))
            elif c & 0x40 or not c & 0x20:
                inc = bool(c & 0x40)
                idx, i = _int(b, i, 6 if inc else 4)
                if idx:
                    name = self._get(idx)[0]
                else:
                    name, i = _str(b, i)
                value, i = _str(b, i)
                out.append((name, value))
                if inc:
                    self._add(name, value)
            else:
                if not first:
                    raise ConnectionError_(COMPRESSION_ERROR, "size update after a field")
                size, i = _int(b, i, 5)
                if size > self.limit:
                    raise ConnectionError_(COMPRESSION_ERROR, "size update above the limit")
                self.max_size = size
                self._evict()
                continue
            first = False
        return out

    def classes(self):
        return self.cls


# ---- responses ---------------------------------------------------------------------------------------------------
def frame(ftype, flags, sid, payload=b""):
    return struct.pack(">I", len(payload))[1:] + bytes((ftype, flags)) + struct.pack(">I", sid) + payload


def _lit(name, value):
    """a literal without indexing with a new name, no Huffman coding"""
    def s(x):
        return (bytes([len(x)]) if len(x) < 127 else bytes([127]) + _varint7(len(x) - 127)) + x
    return b"\x00" + s(name) + s(value)


def _varint7(n):
    out = bytearray()
    while n >= 128:
        out.append(n & 0x7f | 0x80)
        n >>= 7
    out.append(n)
    return bytes(out)


STATUS_CTYPE = b"\x88\x0f\x10\x10application/grpc"
_PCT = set(range(0x20)) | set(range(0x7f, 0x100)) | set(b'% "#<>`?{}')


def percent_encode(text):
    return "".join("%%%02X" % c if c in _PCT else chr(c) for c in text.encode()).encode()


def trailers_only(sid, status, message=b""):
    block = STATUS_CTYPE + _lit(b"grpc-status", str(status).encode())
    if message:
        block += _lit(b"grpc-message", percent_encode(message))
    return frame(HEADERS, END_STREAM | END_HEADERS, sid, block)


def format_replies(req, res, stream_ids):
    """gcra_grpc_format_replies of REQ_DTYPE rows, their RES_DTYPE results and stream ids -> (bytes, data_sent)"""
    req = np.ascontiguousarray(req, REQ_DTYPE)
    res = np.ascontiguousarray(res, RES_DTYPE)
    sids = np.ascontiguousarray(stream_ids, np.uint32)
    buf = C.create_string_buffer(max(len(req), 1) * GRPC_REPLY_MAX)
    sent = C.c_uint32()
    w = _native.lib().gcra_grpc_format_replies(req.ctypes.data, res.ctypes.data, sids.ctypes.data, len(req), buf,
                                               len(buf), C.byref(sent))
    return buf.raw[:w], sent.value


# ---- ThrottleRequest as prost decodes it --------------------------------------------------------------------------
class DecodeError(ValueError):
    pass


def _pvarint(b, i):
    v = 0
    for k in range(10):
        if i >= len(b):
            raise DecodeError("invalid varint")
        x = b[i]
        i += 1
        if k == 9 and x > 1:
            raise DecodeError("invalid varint")
        v |= (x & 0x7f) << (7 * k)
        if not x & 0x80:
            return v, i
    raise DecodeError("invalid varint")


def _i32(v):
    v &= 0xffffffff
    return v - (1 << 32) if v >= 1 << 31 else v


def decode_request(msg):
    """-> (key bytes, max_burst, count_per_period, period, quantity); DecodeError with a detail text"""
    b, i = bytes(msg), 0
    key, nums = b"", [0, 0, 0, 0]
    while i < len(b):
        k, i = _pvarint(b, i)
        if k > 0xffffffff:
            raise DecodeError("invalid key value: %d" % k)
        wt, tag = k & 7, k >> 3
        if tag == 0:
            raise DecodeError("invalid tag value: 0")
        if wt > 5:
            raise DecodeError("invalid wire type value: %d" % wt)
        if 1 <= tag <= 5 and wt != (2 if tag == 1 else 0):
            raise DecodeError("invalid wire type: %d (field %d)" % (wt, tag))
        if wt == 0:
            v, i = _pvarint(b, i)
            if tag >= 2 and tag <= 5:
                nums[tag - 2] = _i32(v)
        elif wt in (1, 5):
            n = 8 if wt == 1 else 4
            if len(b) - i < n:
                raise DecodeError("buffer underflow")
            i += n
        elif wt == 2:
            n, i = _pvarint(b, i)
            if n > len(b) - i:
                raise DecodeError("buffer underflow")
            if tag == 1:
                key = b[i:i + n]
                try:
                    key.decode("utf-8")
                except UnicodeDecodeError:
                    raise DecodeError("invalid string value: data is not UTF-8 encoded")
            i += n
        else:
            raise DecodeError("groups are not supported")
    return (key, *nums)


# ---- a connection ------------------------------------------------------------------------------------------------
class Stream:
    def __init__(self, sid, send_window):
        self.sid, self.send_window = sid, send_window
        self.headers, self.block, self.data = None, bytearray(), bytearray()
        self.remote_done = False
        self.pending = []              # frames to send: (payload flow-controlled DATA or not, bytes)


class Connection:
    """One HTTP/2 connection's state, kept between calls of process_connections.  Append received bytes to `buf`;
    process_connections consumes them and appends what to send to `out`; `closed` becomes True after a GOAWAY."""

    def __init__(self):
        self.buf, self.out = bytearray(), bytearray()
        self.preface = False
        self.hpack = Decoder()
        self.last_stream = 0
        self.send_window = 65535
        self.init_window = 65535
        self.streams = {}
        self.cont = None               # the stream whose header block awaits CONTINUATION
        self.closed = False
        self.first_settings = False    # the client's SETTINGS have arrived
        self.n_throttle = 0
        self.metrics = None            # (general's `metrics`, for the calls it decides)

    def state(self, row):
        """write this connection's state into a GRPC_CONN_DTYPE row (not off / len)"""
        cls = self.hpack.classes()
        assert len(cls) <= GRPC_MAX_DYN
        row["last_stream"], row["send_window"], row["init_window"] = self.last_stream, self.send_window, \
            self.init_window
        row["n_dyn"] = len(cls)
        row["dyn_class"][:len(cls)] = cls

    def take_state(self, row):
        """take last_stream and send_window from a GRPC_CONN_DTYPE row: what the ring walks since the last general
        call left (they never change the HPACK table, init_window or the streams, which stay here)"""
        self.last_stream, self.send_window = int(row["last_stream"]), int(row["send_window"])

    def conn_row(self):
        from . import GRPC_CONN_DTYPE
        row = np.zeros((), GRPC_CONN_DTYPE)
        self.state(row)
        return row

    @property
    def plain_ready(self):
        """whether the GPU walk may take the connection: preface done, no stream open, no header block pending"""
        return self.preface and not self.streams and self.cont is None and not self.closed

    def take_outcome(self, o):
        """apply a walk's outcome (after its responses went to `out`)"""
        self.last_stream = int(o["last_stream"])
        self.send_window = int(o["send_window"]) - int(o["data_sent"])
        if int(o["data_octets"]):
            self.out += frame(WINDOW_UPDATE, 0, 0, struct.pack(">I", int(o["data_octets"])))
        if int(o["ping"]):
            self.out += frame(PING, ACK, 0, bytes(o["ping_opaque"]))

    # -- the general path --
    def general(self, limiter, now_ns, metrics=None):
        """Take frames off `buf` until no stream is open and nothing is pending (at least one frame, or the preface).
        Returns the Throttle decisions made.  A metrics.Metrics as `metrics` records each Throttle call decided here
        as grpc.rs:170-180 does: an error when the engine returns a status other than OK, else allowed or denied."""
        self.metrics = metrics
        before = self.n_throttle
        try:
            if not self.preface:
                if len(self.buf) < len(PREFACE):
                    if not PREFACE.startswith(bytes(self.buf)):
                        raise ConnectionError_(PROTOCOL_ERROR, "bad preface")
                    return 0
                if bytes(self.buf[:len(PREFACE)]) != PREFACE:
                    raise ConnectionError_(PROTOCOL_ERROR, "bad preface")
                del self.buf[:len(PREFACE)]
                self.preface = True
                self.out += frame(SETTINGS, 0, 0)
            while not self.closed:
                if len(self.buf) < 9:
                    break
                n = int.from_bytes(self.buf[:3], "big")
                if n > MAX_FRAME:
                    raise ConnectionError_(FRAME_SIZE_ERROR, "frame above SETTINGS_MAX_FRAME_SIZE")
                if len(self.buf) < 9 + n:
                    break
                ftype, flags = self.buf[3], self.buf[4]
                sid = int.from_bytes(self.buf[5:9], "big") & 0x7fffffff
                payload = bytes(self.buf[9:9 + n])
                del self.buf[:9 + n]
                self._frame(ftype, flags, sid, payload, limiter, now_ns)
                self._flush()
                if not self.streams and self.cont is None and self.first_settings:
                    break
        except ConnectionError_ as e:
            self.out += frame(GOAWAY, 0, 0, struct.pack(">II", self.last_stream, e.code))
            self.closed = True
        return self.n_throttle - before

    def _frame(self, ftype, flags, sid, p, limiter, now_ns):
        if self.cont is not None and ftype != CONTINUATION:
            raise ConnectionError_(PROTOCOL_ERROR, "CONTINUATION expected")
        if ftype == SETTINGS:
            if sid:
                raise ConnectionError_(PROTOCOL_ERROR, "SETTINGS on a stream")
            if flags & ACK:
                if p:
                    raise ConnectionError_(FRAME_SIZE_ERROR, "SETTINGS ACK with a payload")
                return
            if len(p) % 6:
                raise ConnectionError_(FRAME_SIZE_ERROR, "SETTINGS length")
            for k in range(0, len(p), 6):
                ident, v = struct.unpack(">HI", p[k:k + 6])
                if ident == 4:                                   # SETTINGS_INITIAL_WINDOW_SIZE
                    if v > MAX_WINDOW:
                        raise ConnectionError_(FLOW_CONTROL_ERROR, "initial window above 2^31-1")
                    for s in self.streams.values():
                        s.send_window += v - self.init_window
                    self.init_window = v
                elif ident == 5 and not 16384 <= v <= 2**24 - 1:
                    raise ConnectionError_(PROTOCOL_ERROR, "max frame size")
                elif ident == 2 and v > 1:
                    raise ConnectionError_(PROTOCOL_ERROR, "ENABLE_PUSH")
            self.out += frame(SETTINGS, ACK, 0)
            self.first_settings = True
        elif ftype == PING:
            if sid or len(p) != 8:
                raise ConnectionError_(PROTOCOL_ERROR if sid else FRAME_SIZE_ERROR, "PING")
            if not flags & ACK:
                self.out += frame(PING, ACK, 0, p)
        elif ftype == GOAWAY:
            self.closed = True
        elif ftype == WINDOW_UPDATE:
            if len(p) != 4:
                raise ConnectionError_(FRAME_SIZE_ERROR, "WINDOW_UPDATE length")
            inc = int.from_bytes(p, "big") & 0x7fffffff
            if sid == 0:
                if inc == 0:
                    raise ConnectionError_(PROTOCOL_ERROR, "WINDOW_UPDATE of 0")
                self.send_window += inc
                if self.send_window > MAX_WINDOW:
                    raise ConnectionError_(FLOW_CONTROL_ERROR, "connection window above 2^31-1")
            elif sid in self.streams:
                s = self.streams[sid]
                if inc == 0:
                    self._reset(sid, PROTOCOL_ERROR)
                    return
                s.send_window += inc
                if s.send_window > MAX_WINDOW:
                    self._reset(sid, FLOW_CONTROL_ERROR)
            elif sid > self.last_stream or not sid & 1:
                raise ConnectionError_(PROTOCOL_ERROR, "WINDOW_UPDATE on an idle stream")
        elif ftype == RST_STREAM:
            if len(p) != 4:
                raise ConnectionError_(FRAME_SIZE_ERROR, "RST_STREAM length")
            if sid == 0 or (sid > self.last_stream and sid not in self.streams):
                raise ConnectionError_(PROTOCOL_ERROR, "RST_STREAM on an idle stream")
            self.streams.pop(sid, None)
        elif ftype == PRIORITY:
            if sid == 0:
                raise ConnectionError_(PROTOCOL_ERROR, "PRIORITY on stream 0")
            if len(p) != 5:
                self._reset(sid, FRAME_SIZE_ERROR)
        elif ftype in (HEADERS, CONTINUATION):
            self._headers(ftype, flags, sid, p, limiter, now_ns)
        elif ftype == DATA:
            self._data(flags, sid, p, limiter, now_ns)
        elif ftype == PUSH_PROMISE:
            raise ConnectionError_(PROTOCOL_ERROR, "PUSH_PROMISE from a client")
        # (frames of unknown types are ignored: RFC 9113 5.5)

    @staticmethod
    def _unpad(flags, p):
        if flags & PADDED:
            if not p or p[0] >= len(p):
                raise ConnectionError_(PROTOCOL_ERROR, "padding")
            return p[1:len(p) - p[0]]
        return p

    def _headers(self, ftype, flags, sid, p, limiter, now_ns):
        if ftype == CONTINUATION:
            if self.cont is None or sid != self.cont[0]:
                raise ConnectionError_(PROTOCOL_ERROR, "unexpected CONTINUATION")
            s_id, block, end_stream = self.cont
            block += p
        else:
            if sid == 0 or not sid & 1:
                raise ConnectionError_(PROTOCOL_ERROR, "HEADERS on stream %d" % sid)
            p = self._unpad(flags, p)
            if flags & PRIO:
                if len(p) < 5:
                    raise ConnectionError_(FRAME_SIZE_ERROR, "priority fields")
                p = p[5:]
            s_id, block, end_stream = sid, bytearray(p), bool(flags & END_STREAM)
        if not flags & END_HEADERS:
            self.cont = (s_id, block, end_stream)
            return
        self.cont = None
        fields = self.hpack.decode(block)                      # (the table changes even for a stream we drop)
        if s_id in self.streams:                               # trailers from the client
            s = self.streams[s_id]
            if not end_stream:
                raise ConnectionError_(PROTOCOL_ERROR, "second HEADERS without END_STREAM")
            s.remote_done = True
            self._complete(s, limiter, now_ns)
            return
        if s_id <= self.last_stream:
            raise ConnectionError_(STREAM_CLOSED, "HEADERS on a closed stream")
        self.last_stream = s_id
        s = Stream(s_id, self.init_window)
        s.headers = fields
        self.streams[s_id] = s
        if end_stream:
            s.remote_done = True
            self._complete(s, limiter, now_ns)

    def _data(self, flags, sid, p, limiter, now_ns):
        if sid == 0:
            raise ConnectionError_(PROTOCOL_ERROR, "DATA on stream 0")
        if len(p):
            self.out += frame(WINDOW_UPDATE, 0, 0, struct.pack(">I", len(p)))
        s = self.streams.get(sid)
        if s is None or s.remote_done:
            if sid > self.last_stream:
                raise ConnectionError_(PROTOCOL_ERROR, "DATA on an idle stream")
            self.out += frame(RST_STREAM, 0, sid, struct.pack(">I", STREAM_CLOSED))
            return
        s.data += self._unpad(flags, p)
        if len(s.data) > 5 + MAX_MESSAGE:                  # answered now; the rest of the stream is not buffered
            self.out += trailers_only(sid, 8, "decoded message length too large: more than %d bytes" % MAX_MESSAGE)
            self._reset(sid, NO_ERROR)
            return
        if flags & END_STREAM:
            s.remote_done = True
            self._complete(s, limiter, now_ns)
        elif len(p):
            self.out += frame(WINDOW_UPDATE, 0, sid, struct.pack(">I", len(p)))

    def _reset(self, sid, code):
        self.out += frame(RST_STREAM, 0, sid, struct.pack(">I", code))
        self.streams.pop(sid, None)

    def _complete(self, s, limiter, now_ns):
        """a stream whose request has ended: decide it and queue its response"""
        h = {}
        for n, v in s.headers:
            h.setdefault(n, v)
        sid = s.sid
        if h.get(b":method") != b"POST" or not (h.get(b"content-type", b"").startswith(b"application/grpc")):
            s.pending = [(False, frame(HEADERS, END_STREAM | END_HEADERS, sid, b"\x8d"))]    # :status 404
            return
        if h.get(b":path") != PATH:
            s.pending = [(False, trailers_only(sid, 12))]
            return
        if h.get(b"grpc-encoding", b"identity") != b"identity":
            s.pending = [(False, trailers_only(sid, 12, "Content is compressed with `%s` which isn't supported"
                                                  % h[b"grpc-encoding"].decode("latin-1")))]
            return
        d = bytes(s.data)
        try:
            if len(d) < 5 or d[0] not in (0, 1) or int.from_bytes(d[1:5], "big") != len(d) - 5:
                raise DecodeError("not one gRPC message")
            if d[0] == 1:
                raise DecodeError("a compressed message without grpc-encoding")
            key, b, c, p, q = decode_request(d[5:])
        except DecodeError as e:
            s.pending = [(False, trailers_only(sid, 13, "failed to decode ThrottleRequest: %s" % e))]
            return
        row = np.zeros(1, REQ_DTYPE)
        row[0] = (limiter.store.hash_key(key), b, c, p, q, now_ns)
        res = limiter.rate_limit_batch(row)
        self.n_throttle += 1
        if isinstance(self.metrics, Metrics):
            if int(res[0]["status"]) != OK:
                self.metrics.record_error("grpc")
            else:
                self.metrics.record_request("grpc", bool(res[0]["allowed"]), key)
        out, _ = format_replies(row, res, [sid])
        frames, i = [], 0
        while i < len(out):
            n = int.from_bytes(out[i:i + 3], "big")
            frames.append((out[i + 3] == DATA, out[i:i + 9 + n]))
            i += 9 + n
        s.pending = frames

    def _flush(self):
        """send what the windows allow, in stream order; a stream whose response is all sent closes"""
        for sid in sorted(self.streams):
            s = self.streams[sid]
            while s.pending:
                flow, f = s.pending[0]
                n = len(f) - 9
                if flow and n > min(self.send_window, s.send_window):
                    break                                  # (a response's DATA is at most 51 octets: never split)
                if flow:
                    self.send_window -= n
                    s.send_window -= n
                self.out += f
                s.pending.pop(0)
            if s.remote_done and not s.pending:
                del self.streams[sid]


def host_walk(cn, limiter, now_ns, max_calls=1 << 20):
    """gcra_grpc_parse_throttle over a connection's bytes, decided by limiter.rate_limit_batch -> (outcome as the
    GPU writes it (GRPC_OUTCOME_DTYPE), response bytes, rows, results, stream ids)"""
    from . import GRPC_OUTCOME_DTYPE
    data = bytes(cn.buf)
    row = cn.conn_row()
    req = np.zeros(len(data) // 26 + 1, REQ_DTYPE)
    sids = np.zeros(len(req), np.uint32)
    o = np.zeros((), GRPC_OUTCOME_DTYPE)
    L = _native.lib()
    # (keys hashed as the general path hashes them, limiter.store.hash_key: under the engine's seed when it has one)
    h = getattr(limiter.store, "_h", None)
    rc = L.gcra_grpc_parse_throttle(h, data, len(data), now_ns, max_calls, row.ctypes.data, req.ctypes.data,
                                    sids.ctypes.data, o.ctypes.data)
    assert rc == 0
    n = int(o["n_frames"])
    res = limiter.rate_limit_batch(req[:n]) if n else np.zeros(0, RES_DTYPE)
    out, sent = format_replies(req[:n], res, sids[:n])
    o["reply_len"], o["data_sent"] = len(out), sent
    return o, out, req[:n], res, sids[:n]


def process_connections(conns, limiter, now_ns, ring, slot=0, metrics=None):
    """Serve every Connection in `conns` from its received bytes: rounds in which the GPU (`ring`, a GrpcRing of
    `limiter`'s engine; None: the host walk, gcra_grpc_parse_throttle, one connection at a time, with keys hashed as
    limiter.store.hash_key hashes them) takes every ready connection's plain prefix, in list order, one batch per submit; then each
    connection that stopped at a frame that is not plain (or has not yet finished its preface, or has a stream open)
    takes the general path until no stream is open, in list order, deciding its calls there and then.  Each
    connection's `buf` must hold at most 65,536 bytes.  Returns the Throttle decisions made per connection.
    `metrics`, a metrics.Metrics of `limiter`'s engine, records the calls of the general path; the GPU counts the
    ring's rows.  It needs a ring: the host walk has no key positions to name denied keys from (ValueError)."""
    from . import RESP_MAX_CONN_BYTES
    if ring is None and isinstance(metrics, Metrics):
        raise ValueError("metrics need a ring: the host walk does not name denied keys")
    now = int(now_ns)
    for cn in conns:
        if len(cn.buf) > (RESP_MAX_CONN_BYTES if ring is None else min(RESP_MAX_CONN_BYTES, ring.in_capacity)):
            raise ValueError("a connection buffer of %d bytes" % len(cn.buf))
    before = [cn.n_throttle for cn in conns]
    live = [cn for cn in conns if cn.buf and not cn.closed]
    while live:
        stops, i = {}, 0
        ready = [cn for cn in live if cn.plain_ready]
        if ring is None:
            for cn in ready:
                o, out, _, _, _ = host_walk(cn, limiter, now)
                cn.out += out
                cn.take_outcome(o)
                del cn.buf[:int(o["consumed"])]
                cn.n_throttle += int(o["n_frames"])
                stops[id(cn)] = int(o["stop"])
            ready = []
        while i < len(ready):
            group, used = [], 0
            while i < len(ready) and len(group) < ring.max_conns:
                cn = ready[i]
                rest = len(cn.buf)
                if used + rest > ring.in_capacity:
                    break
                ring.input[slot][used:used + rest] = np.frombuffer(bytes(cn.buf), np.uint8)
                row = ring.conns[slot][len(group)]
                row["off"], row["len"] = used, rest
                cn.state(row)
                group.append(cn)
                used += rest
                i += 1
            ring.submit(slot, len(group), now)
            ring.wait(slot)
            for j, cn in enumerate(group):
                o = ring.outcome[slot][j]
                off, ln = int(o["reply_off"]), int(o["reply_len"])
                cn.out += ring.replies[slot][off:off + ln].tobytes()
                cn.take_outcome(o)
                del cn.buf[:int(o["consumed"])]
                cn.n_throttle += int(o["n_frames"])
                stops[id(cn)] = int(o["stop"])
        nxt = []
        for cn in live:
            st = stops.get(id(cn), 2)
            if st == 3:
                nxt.append(cn)
                continue
            if st != 2:
                continue
            had = len(cn.buf)
            cn.general(limiter, now, metrics)
            if not cn.closed and cn.buf and len(cn.buf) < had and cn.plain_ready:
                nxt.append(cn)
        live = nxt
    return [cn.n_throttle - b for cn, b in zip(conns, before)]
