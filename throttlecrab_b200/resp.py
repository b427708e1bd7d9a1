"""RESP ingest for the batched engine (SURVEY §8f "next" row #3).

Mirrors the reference's RESP value model, parser limits and serializer
(throttlecrab-server/src/transport/redis/resp.rs:8-232) and the command semantics of
`process_command` / `handle_throttle` (redis/mod.rs:150-295): same replies, same error strings.
What changes is the shape of the work: `process_pipeline()` parses EVERY complete frame in a read buffer,
turns all well-formed `THROTTLE key max_burst count_per_period period [quantity]` commands into request
rows and hands them to the engine as ONE batch (results as if applied in arrival order), then writes the
replies in command order.  Host-side glue only: no decision is made here.
"""
import numpy as np

from . import REQ_DTYPE, NS, hash_key, OK, NEGATIVE_QUANTITY, INVALID_RATE_LIMIT
from .metrics import Metrics

MAX_BULK_STRING_SIZE = 512 * 1024 * 1024      # resp.rs:8
MAX_ARRAY_SIZE = 1024 * 1024                  # resp.rs:9
MAX_ARRAY_DEPTH = 128                         # resp.rs:10
I64_MIN, I64_MAX = -2**63, 2**63 - 1


class RespError(ValueError):
    """protocol error: the reference's parser bails (the connection is closed)"""


# ---- value model (resp.rs:13-25): tagged tuples -----------------------------------------------------------
def SimpleString(s):
    return ("simple", s)


def Error(s):
    return ("error", s)


def Integer(n):
    return ("int", int(n))


def BulkString(s):
    return ("bulk", s)          # s is str or None (null bulk string)


def Array(items):
    return ("array", list(items))


def _parse_i64(text):
    """Rust's str::parse::<i64>: optional sign, ASCII digits only, must fit."""
    t = text[1:] if text[:1] in "+-" else text
    if not t or not t.isascii() or not t.isdigit():
        return None
    n = int(text)
    return n if I64_MIN <= n <= I64_MAX else None


class RespParser:
    """resp.rs:28-177.  parse(data) -> None (need more data) | (value, bytes_consumed); raises RespError."""

    def __init__(self):
        self.depth = 0

    def parse(self, data):
        data = bytes(data)
        if not data:
            return None
        t = data[:1]
        if t == b"+":
            return self._line(data, SimpleString)
        if t == b"-":
            return self._line(data, Error)
        if t == b":":
            return self._integer(data)
        if t == b"$":
            return self._bulk(data)
        if t == b"*":
            return self._array(data)
        raise RespError("Invalid RESP type marker: %s" % chr(data[0]))

    @staticmethod
    def _read_line(data):
        i = data.find(b"\r\n")
        return None if i < 0 else (data[:i], i + 2)

    @staticmethod
    def _utf8(b):
        try:
            return b.decode("utf-8")
        except UnicodeDecodeError as e:
            raise RespError("invalid utf-8: %s" % e)

    def _line(self, data, ctor):
        r = self._read_line(data)
        if r is None:
            return None
        return ctor(self._utf8(r[0][1:])), r[1]

    def _int_line(self, data):
        r = self._read_line(data)
        if r is None:
            return None
        n = _parse_i64(self._utf8(r[0][1:]))
        if n is None:
            raise RespError("invalid digit found in string")
        return n, r[1]

    def _integer(self, data):
        r = self._int_line(data)
        return None if r is None else (Integer(r[0]), r[1])

    def _bulk(self, data):
        r = self._int_line(data)
        if r is None:
            return None
        length, consumed = r
        if length == -1:
            return BulkString(None), consumed
        if not 0 <= length <= MAX_BULK_STRING_SIZE:
            raise RespError("Invalid bulk string length: %d" % length)
        if len(data) < consumed + length + 2:
            return None
        return BulkString(self._utf8(data[consumed:consumed + length])), consumed + length + 2

    def _array(self, data):
        if self.depth >= MAX_ARRAY_DEPTH:
            raise RespError("Maximum array nesting depth exceeded")
        r = self._int_line(data)
        if r is None:
            return None
        count, consumed = r
        if count == -1:
            return Array([]), consumed
        if not 0 <= count <= MAX_ARRAY_SIZE:
            raise RespError("Invalid array size: %d" % count)
        items = []
        self.depth += 1
        try:
            for _ in range(count):
                e = self.parse(data[consumed:])
                if e is None:
                    return None
                items.append(e[0])
                consumed += e[1]
        finally:
            self.depth -= 1
        return Array(items), consumed


class RespSerializer:
    """resp.rs:186-232"""

    @staticmethod
    def serialize(v):
        kind, x = v
        if kind == "simple":
            return b"+" + x.encode() + b"\r\n"
        if kind == "error":
            return b"-" + x.encode() + b"\r\n"
        if kind == "int":
            return b":" + str(x).encode() + b"\r\n"
        if kind == "bulk":
            if x is None:
                return b"$-1\r\n"
            b = x.encode()
            return b"$" + str(len(b)).encode() + b"\r\n" + b + b"\r\n"
        return b"*" + str(len(x)).encode() + b"\r\n" + b"".join(RespSerializer.serialize(e) for e in x)


def _arg_integer(v):                          # redis/mod.rs:289-295
    if v[0] == "bulk" and v[1] is not None:
        return _parse_i64(v[1])
    if v[0] == "int":
        return v[1]
    return None


def _plan_command(value):
    """-> ("reply", RespValue) for everything that needs no decision, or ("throttle", key, b, c, p, q)."""
    if value[0] != "array":
        return ("reply", Error("ERR expected array of commands"))              # mod.rs:158
    args = value[1]
    if not args:
        return ("reply", Error("ERR empty command"))                            # :162
    if args[0][0] != "bulk" or args[0][1] is None:
        return ("reply", Error("ERR invalid command format"))                   # :168
    command = args[0][1].upper()
    if command == "PING":                                                        # :208-218
        if len(args) == 1:
            return ("reply", SimpleString("PONG"))
        if len(args) == 2:
            return ("reply", args[1])
        return ("reply", Error("ERR wrong number of arguments for 'ping' command"))
    if command == "QUIT":
        return ("reply", SimpleString("OK"))
    if command != "THROTTLE":
        return ("reply", Error("ERR unknown command '%s'" % command))           # :186
    if len(args) < 5 or len(args) > 6:                                           # :226-230
        return ("reply", Error("ERR wrong number of arguments for 'throttle' command"))
    if args[1][0] != "bulk" or args[1][1] is None:
        return ("reply", Error("ERR invalid key"))                              # :235
    nums = []
    for a, name in zip(args[2:], ("max_burst", "count_per_period", "period", "quantity")):
        n = _arg_integer(a)
        if n is None:
            return ("reply", Error("ERR invalid %s" % name))                    # :239-258
        nums.append(n)
    if len(nums) == 3:
        nums.append(1)
    return ("throttle", args[1][1], nums[0], nums[1], nums[2], nums[3])


def _is_quit(value):
    """redis/mod.rs:132-135: an array whose first element is the bulk string QUIT (any case)"""
    return (value[0] == "array" and len(value[1]) > 0 and value[1][0][0] == "bulk"
            and value[1][0][1] is not None and value[1][0][1].upper() == "QUIT")


def _counted(value):
    """whether process_command reaches its command match and records the command (redis/mod.rs:156-169,201-205): an
    array whose first element is a bulk string"""
    return value[0] == "array" and len(value[1]) > 0 and value[1][0][0] == "bulk" and value[1][0][1] is not None


def _throttle_reply(o, limit, quantity):
    st = int(o["status"])
    if st == OK:                                                                 # mod.rs:274-283, types.rs:87-97
        return Array([Integer(1 if o["allowed"] else 0), Integer(limit), Integer(int(o["remaining"])),
                      Integer(int(o["reset_after_ns"]) // NS), Integer(int(o["retry_after_ns"]) // NS)])
    # "ERR {e}" (mod.rs:285) where e = "Rate limit check failed: {CellError}" (actor.rs:252, core/mod.rs:58-65)
    if st == NEGATIVE_QUANTITY:
        return Error("ERR Rate limit check failed: negative quantity: %d" % quantity)
    if st == INVALID_RATE_LIMIT:
        return Error("ERR Rate limit check failed: invalid rate limit parameters")
    return Error("ERR Rate limit check failed: internal error")


def process_pipeline(buffer, rate_limit_batch, now_ns):
    """Parse every complete command in `buffer`, decide all THROTTLE commands in ONE engine batch
    (`rate_limit_batch(REQ_DTYPE array) -> RES_DTYPE array`, e.g. RateLimiter.rate_limit_batch), and return
    (reply_bytes, bytes_consumed, n_throttle, close).  `now_ns` may be an int (one timestamp for the whole buffer,
    like SystemTime::now() per command at mod.rs:270 read once) or a callable returning one per command.

    As in the reference's connection loop (redis/mod.rs:128-149): commands are answered in order; a protocol error
    on a LATER frame does not undo the commands before it -- they are applied and answered, then `close` is "error"
    (the reference returns the parser's error, which closes the connection); nothing after a QUIT is executed and
    `close` is "quit".  Otherwise `close` is None."""
    parser = RespParser()
    data = bytes(buffer)
    plans, consumed, close = [], 0, None
    while consumed < len(data):
        try:
            r = parser.parse(data[consumed:])
        except RespError:
            close = "error"
            break
        if r is None:
            break
        plans.append(_plan_command(r[0]))
        consumed += r[1]
        if _is_quit(r[0]):
            close = "quit"
            break
    rows = [p for p in plans if p[0] == "throttle"]
    res = None
    if rows:
        req = np.empty(len(rows), REQ_DTYPE)
        for i, (_, key, b, c, p, q) in enumerate(rows):
            req[i] = (hash_key(key), b, c, p, q, now_ns() if callable(now_ns) else now_ns)
        res = rate_limit_batch(req)
    out, j = [], 0
    for p in plans:
        if p[0] == "reply":
            out.append(RespSerializer.serialize(p[1]))
            continue
        out.append(RespSerializer.serialize(_throttle_reply(res[j], p[2], p[5])))
        j += 1
    return b"".join(out), consumed, len(rows), close


def process_pipeline_native(buffer, limiter, now_ns, ring=None, slot=0):
    """The same contract as process_pipeline, with the hot command on the native path: gcra_resp_parse_throttle
    (csrc/gcra_resp.inc) walks the buffer once and writes one request row per plain THROTTLE frame straight into the
    request array -- the pinned ring slot `ring.req[slot]` when a Ring is given -- and gcra_resp_format_replies
    writes the replies; only frames that are not plain THROTTLE commands (PING, QUIT, RESP-integer arguments, ...)
    go through the general parser above.  All THROTTLE commands of the buffer are ONE engine batch (the ring's
    submit / wait when a ring is given, else rate_limit_batch); replies come back in command order.
    A keyed ring (Ring(..., key_capacity=...)) takes gcra_resp_parse_throttle_keyed instead: keys are copied into
    the slot's key arena and hashed on the GPU, not on this thread; a key that no longer fits ends the batch there,
    unconsumed, like a full slot.  A key longer than the whole arena can never fit: when it comes first, its frame
    is hashed on this thread and decided alone, as a batch of host-hashed rows, so every frame is answered.
    Returns (reply_bytes, bytes_consumed, n_throttle, close)."""
    import ctypes as C
    from . import RES_DTYPE, _kb, key_ref
    L, h = limiter._L, limiter._h
    data = bytes(buffer)
    cap = ring.cap if ring is not None else max(len(data) // 32 + 1, 16)
    req = ring.req[slot] if ring is not None else np.empty(cap, REQ_DTYPE)
    arena = ring.keys[slot] if ring is not None and ring.keys is not None else None
    kused = C.c_uint64(0)
    host_hashed = arena is None                           # (the batch's rows hold key hashes, not key references)
    parser = RespParser()
    segs, n, consumed, close = [], 0, 0, None            # segs: ("rows", first, count) | ("reply", value) | ("row", index, limit, qty)
    now = int(now_ns() if callable(now_ns) else now_ns)
    while consumed < len(data) and n < cap:
        used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
        view = data[consumed:]
        rows = req.ctypes.data + n * REQ_DTYPE.itemsize
        if arena is None:
            limiter.store._check(L.gcra_resp_parse_throttle(h, view, len(view), now, cap - n, rows,
                                                            C.byref(used), C.byref(cnt), C.byref(stop)))
        else:
            limiter.store._check(L.gcra_resp_parse_throttle_keyed(h, view, len(view), now, cap - n, rows,
                                                                  arena.ctypes.data, len(arena), C.byref(kused),
                                                                  C.byref(used), C.byref(cnt), C.byref(stop)))
        if arena is not None and stop.value == 3 and n == 0 and cnt.value == 0:
            # the first frame's key is longer than the arena: this one frame, hashed here, is the batch
            limiter.store._check(L.gcra_resp_parse_throttle(h, view, len(view), now, 1, rows, C.byref(used),
                                                            C.byref(cnt), C.byref(stop)))
            host_hashed = True
        if cnt.value:
            segs.append(("rows", n, cnt.value))
            n += cnt.value
            consumed += used.value
        if host_hashed and arena is not None:
            break
        if stop.value != 2:
            break                                         # end of buffer, incomplete frame, or the slot is full
        try:                                              # one frame for the general parser
            r = parser.parse(data[consumed:])
        except RespError:
            close = "error"
            break
        if r is None:
            break
        consumed += r[1]
        plan = _plan_command(r[0])
        if plan[0] == "throttle":
            if n >= cap:
                consumed -= r[1]
                break
            kb = _kb(plan[1])
            if arena is not None and len(kb) > len(arena) - kused.value:
                if n:
                    consumed -= r[1]
                    break
                host_hashed = True                        # longer than the whole arena: decided alone (see above)
            if host_hashed:
                kh = hash_key(kb) if not any(limiter.store.hash_seed()) else limiter.store.hash_key(kb)
            else:
                at = kused.value
                arena[at:at + len(kb)] = np.frombuffer(kb, np.uint8)
                kused.value = at + len(kb)
                kh = key_ref(at, len(kb))
            req[n] = (kh, plan[2], plan[3], plan[4], plan[5], now)
            segs.append(("row", n, plan[2], plan[5]))
            n += 1
            if host_hashed and arena is not None:
                break
        else:
            segs.append(("reply", plan[1]))
        if _is_quit(r[0]):
            close = "quit"
            break
    res = None
    if n:
        if ring is not None:
            ring.submit(slot, n, now, keys_len=None if host_hashed else kused.value)
            ring.wait(slot)
            res = ring.res[slot]
        else:
            res = limiter.rate_limit_batch(req[:n])
    out = []
    scratch = C.create_string_buffer(max(n, 1) * 160)
    for sg in segs:
        if sg[0] == "reply":
            out.append(RespSerializer.serialize(sg[1]))
        elif sg[0] == "row":
            out.append(RespSerializer.serialize(_throttle_reply(res[sg[1]], sg[2], sg[3])))
        else:
            first, cnt = sg[1], sg[2]
            w = L.gcra_resp_format_replies(req.ctypes.data + first * REQ_DTYPE.itemsize,
                                           res.ctypes.data + first * RES_DTYPE.itemsize, cnt, scratch, len(scratch))
            out.append(scratch.raw[:w])
    return b"".join(out), consumed, n, close


def process_connections(buffers, limiter, now_ns, ring, slot=0, metrics=None):
    """process_pipeline for many connections at once, with the parsing and the reply formatting of plain THROTTLE
    frames on the GPU: `ring` is a RespRing of `limiter`'s engine.  Returns one (reply_bytes, bytes_consumed,
    n_throttle, close) per buffer, with process_pipeline's meaning; an error or a QUIT closes only its own connection.
    Each buffer holds at most 65,536 bytes (the reference's MAX_BUFFER_SIZE) and fits in the ring's input.

    Rounds run until every connection has ended at the end of its bytes, at an incomplete frame, or closed.  In a
    round, the GPU takes every open connection's plain-THROTTLE prefix: one batch per submit, rows in list order of the
    connections and frame order within each (a full slot leaves the rest to the next round, or to the next submit of
    the same round when the connections do not fit one).  Then each connection that stopped at a frame that is not a
    plain THROTTLE hands that one frame to the general parser, in list order; a THROTTLE among them is decided there
    and then, on its own.  That is the order in which decisions are made, so connections that share keys see each
    other's requests in that order.  `metrics` (a metrics.Metrics of `limiter`'s engine) records the commands of the
    general path as the reference's Redis transport does; the GPU counts the ring's rows."""
    now = int(now_ns)
    return ring_rounds(buffers, ring, slot, now, lambda data: general(data, limiter, now, metrics))


def general(data, limiter, now, metrics=None):
    """The general path of a connection that the batch walk stopped at a frame that is not a plain THROTTLE (stop 2):
    that one frame, at the start of `data`, parsed by RespParser and answered; a THROTTLE among them is decided there
    and then, on its own, with the key hashed by limiter.store.hash_key.  Returns None (the frame is incomplete) or
    (bytes consumed, reply bytes, THROTTLE decisions, close), close being None, "quit" or "error".  A Metrics as
    `metrics` records the command as redis/mod.rs:193-205 does: every command that reaches the command match, allowed
    unless its THROTTLE reply is an array that starts with 0 (an -ERR reply counts as allowed)."""
    try:
        r = RespParser().parse(data)
    except RespError:
        return 0, b"", 0, "error"
    if r is None:
        return None
    plan = _plan_command(r[0])
    if plan[0] == "throttle":
        kb = plan[1].encode()
        req = np.empty(1, REQ_DTYPE)
        req[0] = (limiter.store.hash_key(kb), plan[2], plan[3], plan[4], plan[5], now)
        res = limiter.rate_limit_batch(req)
        if isinstance(metrics, Metrics):
            metrics.record_request("redis", not (int(res[0]["status"]) == OK and not res[0]["allowed"]), plan[1])
        return r[1], RespSerializer.serialize(_throttle_reply(res[0], plan[2], plan[5])), 1, \
            "quit" if _is_quit(r[0]) else None
    if isinstance(metrics, Metrics) and _counted(r[0]):
        metrics.record_request("redis", True)
    return r[1], RespSerializer.serialize(plan[1]), 0, "quit" if _is_quit(r[0]) else None


def ring_rounds(buffers, ring, slot, now, general):
    """The round loop of process_connections, shared by the RESP and HTTP rings: GPU prefixes, then one call of
    `general(bytes from the connection's position)` per connection that stopped at 2, in list order.  `general`
    returns None (the frame is incomplete: the connection waits for more bytes) or (bytes consumed, reply bytes,
    THROTTLE decisions, close), where a close other than None ends the connection."""
    from . import RESP_MAX_CONN_BYTES
    datas = [bytes(b) for b in buffers]
    n = len(datas)
    for d in datas:
        if len(d) > min(RESP_MAX_CONN_BYTES, ring.in_capacity):
            raise ValueError("a connection buffer of %d bytes: at most %d" % (len(d), min(RESP_MAX_CONN_BYTES,
                                                                                       ring.in_capacity)))
    pos, n_thr, close = [0] * n, [0] * n, [None] * n
    out = [[] for _ in range(n)]
    live = [c for c in range(n) if datas[c]]
    while live:
        stops, i = {}, 0
        while i < len(live):                               # as many submits as the ring's capacity needs
            group, used = [], 0
            while i < len(live) and len(group) < ring.max_conns:
                c = live[i]
                rest = len(datas[c]) - pos[c]
                if used + rest > ring.in_capacity:
                    break
                ring.input[slot][used:used + rest] = np.frombuffer(datas[c], np.uint8, rest, pos[c])
                ring.conns[slot][len(group)] = (used, rest)
                group.append(c)
                used += rest
                i += 1
            ring.submit(slot, len(group), now)
            ring.wait(slot)
            for j, c in enumerate(group):
                o = ring.outcome[slot][j]
                off, ln = int(o["reply_off"]), int(o["reply_len"])
                out[c].append(ring.replies[slot][off:off + ln].tobytes())
                pos[c] += int(o["consumed"])
                n_thr[c] += int(o["n_frames"])
                stops[c] = int(o["stop"])
        nxt = []
        for c in live:
            if stops[c] == 3:
                nxt.append(c)
                continue
            if stops[c] != 2:
                continue                                   # the end of its bytes, or an incomplete frame
            g = general(datas[c][pos[c]:])
            if g is None:
                continue
            used, reply, k, close[c] = g
            pos[c] += used
            out[c].append(reply)
            n_thr[c] += k
            if close[c] is None and pos[c] < len(datas[c]):
                nxt.append(c)
        live = nxt
    return [(b"".join(out[c]), pos[c], n_thr[c], close[c]) for c in range(n)]
