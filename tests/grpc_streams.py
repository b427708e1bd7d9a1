"""tests only: HTTP/2 byte streams of Throttle calls, in the shapes grpcio sends them"""
import random
import struct

from throttlecrab_b200 import grpc_transport as gt
from grpc_server import request_bytes

# a grpcio first call's header block inserts these (literal with incremental indexing); later calls index them
FIRST_FIELDS = [(b":scheme", b"http"), (b":method", b"POST"), (b":authority", b"127.0.0.1:50051"),
                (b":path", gt.PATH), (b"te", b"trailers"), (b"content-type", b"application/grpc"),
                (b"user-agent", b"grpc-python/1.80.0 grpc-c/52.0.0 (linux; chttp2)"),
                (b"grpc-accept-encoding", b"identity, deflate, gzip")]


def lit(name, value, kind=0x00, huff_value=False):
    """a literal field with a new name: kind 0x00 without indexing, 0x10 never indexed, 0x40 incremental"""
    v = gt.huffman_encode(value) if huff_value else value
    return bytes([kind]) + bytes([len(name)]) + name + bytes([len(v) | (0x80 if huff_value else 0)]) + v


def first_block():
    """the first call's block: :method POST and :scheme http indexed, the rest inserted"""
    out = b""
    for n, v in FIRST_FIELDS:
        if (n, v) == (b":method", b"POST"):
            out += b"\x83"
        elif (n, v) == (b":scheme", b"http"):
            out += b"\x86"
        else:
            out += lit(n, v, 0x40)
    return out


def steady_block(dec):
    """a later call's block: only indexed fields, as grpcio sends them (dynamic refs for what the table holds)"""
    out = b"\x83\x86"
    for n, v in FIRST_FIELDS:
        if n in (b":method", b":scheme"):
            continue
        out += bytes([0x80 | (62 + dec.table.index((n, v)))])
    return out


def call(sid, block, msg, rng=None, ping=False, split=False):
    """HEADERS, a stream WINDOW_UPDATE, DATA(END_STREAM) and a connection WINDOW_UPDATE, as grpcio sends a call"""
    out = gt.frame(gt.HEADERS, gt.END_HEADERS, sid, block)
    out += gt.frame(gt.WINDOW_UPDATE, 0, sid, struct.pack(">I", 5 + len(msg)))
    if ping:
        out += gt.frame(gt.PING, 0, 0, bytes(range(8)))
    body = b"\x00" + struct.pack(">I", len(msg)) + msg
    if split:
        out += gt.frame(gt.DATA, 0, sid, body) + gt.frame(gt.DATA, gt.END_STREAM, sid)
    else:
        out += gt.frame(gt.DATA, gt.END_STREAM, sid, body)
    return out + gt.frame(gt.WINDOW_UPDATE, 0, 0, struct.pack(">I", 5 + len(msg)))


def established():
    """a Connection past its preface, SETTINGS and first call (its decoder holds grpcio's table)"""
    cn = gt.Connection()
    cn.preface = True
    cn.first_settings = True
    cn.hpack.decode(first_block())
    cn.last_stream = 1
    return cn


def steady_stream(rng, cn, n_calls, keys, sid0=None, extras=True):
    """n_calls plain calls on odd streams after cn.last_stream, keys drawn from `keys`"""
    sid = (sid0 or cn.last_stream) + 2
    out = bytearray()
    block = steady_block(cn.hpack)
    for k in range(n_calls):
        key = rng.choice(keys)
        msg = request_bytes(key, rng.choice([1, 5, 10]), rng.choice([10, 100]), 60, rng.choice([0, 1, 1, 2, -1]))
        out += call(sid, block, msg, ping=extras and k == n_calls // 2, split=extras and k % 7 == 3)
        sid += 2
    return bytes(out)
