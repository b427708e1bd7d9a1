"""HTTP ingest for the batched engine: the general path beside the GPU's fast path.

Mirrors the reference's HTTP transport (throttlecrab-server/src/transport/http.rs:60-73,103-159): the routes
POST /throttle (a JSON `HttpThrottleRequest`), GET /health and GET /metrics, the status codes its stack (axum 0.8,
hyper 1.x, httparse, serde_json) gives, and the response bytes of gcra_http_format_replies for a decision.

- `parse_request(data)` reads one request off a connection's bytes the way httparse and hyper's HTTP/1 server do
  where it matters here: CRLF or bare LF line ends, token header names, a malformed head answered with 400 and the
  connection closed, Content-Length or chunked Transfer-Encoding bodies, HTTP/1.0 and `Connection: close` closing
  after the response.
- `handle_request(req, limiter, now_ns)` answers it: 404 for an unknown path (empty body), 405 with `allow` for a
  wrong method, 415 without a JSON content type (axum's rule: application/json or a +json suffix), 400 for a JSON
  syntax error, 422 for a JSON data error (missing or duplicate field, wrong type, an integer outside i64), else a
  THROTTLE decision.  The JSON rules are serde_json's, not Python's: no NaN or Infinity, no lone surrogate escapes,
  integers only within i64 (and `-0` is a float), unknown fields ignored, escapes decoded.  The rejection bodies start
  with axum's prefixes ("Failed to parse the request body as JSON: ", "Failed to deserialize the JSON body into the
  target type: "); the detail after the prefix is this module's own text, not serde_json's.
- `process_connections(buffers, limiter, now_ns, ring)` is resp.process_connections for HTTP: plain requests are
  parsed, decided and answered on the GPU (an HttpRing); every other request comes through here.

The status line is always HTTP/1.1; response headers follow hyper's encoder as read from its source (the handler's
headers, then `connection: close` when the connection closes, `content-length`, `date`), not as observed.
"""
import ctypes as C

import numpy as np

from . import REQ_DTYPE, RES_DTYPE, HTTP_REPLY_MAX, OK, _native
from .metrics import Metrics
from .resp import ring_rounds

I64_MIN, I64_MAX = -2**63, 2**63 - 1
MAX_HEADERS = 100                       # hyper's default header limit (more: 431)
REASONS = {200: "OK", 400: "Bad Request", 404: "Not Found", 405: "Method Not Allowed", 415: "Unsupported Media Type",
           422: "Unprocessable Entity", 431: "Request Header Fields Too Large", 500: "Internal Server Error"}
TEXT = "text/plain; charset=utf-8"
FIELDS = ("key", "max_burst", "count_per_period", "period", "quantity")
_TCHAR = frozenset(b"!#$%&'*+-.^_`|~0123456789abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ")


class Request:
    """One request read off a connection.  `bad` is a status (400, 431) when the head is malformed; the connection
    then closes after the response."""

    def __init__(self, consumed, method=b"", target=b"", version=1, headers=(), body=b"", bad=None):
        self.consumed, self.method, self.target, self.version = consumed, method, target, version
        self.headers, self.body, self.bad = list(headers), body, bad

    def header(self, name):
        """the first value of header `name` (lower case), or None"""
        for n, v in self.headers:
            if n == name:
                return v
        return None

    def header_tokens(self, name):
        return [t.strip().lower() for n, v in self.headers if n == name for t in v.split(b",") if t.strip()]

    @property
    def close(self):
        conn = self.header_tokens(b"connection")
        if self.bad is not None or b"close" in conn:
            return True
        return self.version == 0 and b"keep-alive" not in conn

    @property
    def path(self):
        return self.target.split(b"?", 1)[0]


def _lines(data, pos):
    """the line at pos (CRLF or bare LF) -> (line, next pos), or None if it has not ended yet"""
    i = data.find(b"\n", pos)
    if i < 0:
        return None
    end = i - 1 if i > pos and data[i - 1] == 13 else i
    return data[pos:end], i + 1


def _chunked(data, pos):
    """a chunked body from pos -> (decoded body, next pos), None if incomplete; ValueError if malformed"""
    out = bytearray()
    while True:
        r = _lines(data, pos)
        if r is None:
            return None
        line, pos = r
        size = line.split(b";", 1)[0].strip()
        if not size or any(c not in b"0123456789abcdefABCDEF" for c in size) or len(size) > 16:
            raise ValueError("invalid chunk size")
        n = int(size, 16)
        if n == 0:
            while True:                                   # trailers, up to the empty line
                r = _lines(data, pos)
                if r is None:
                    return None
                line, pos = r
                if not line:
                    return bytes(out), pos
        if len(data) < pos + n + 1:
            return None
        out += data[pos:pos + n]
        pos += n
        if data[pos:pos + 2] == b"\r\n":
            pos += 2
        elif data[pos:pos + 1] == b"\n":
            pos += 1
        elif data[pos:pos + 1] == b"\r" and len(data) == pos + 1:
            return None
        else:
            raise ValueError("invalid chunk end")


def parse_request(data):
    """The request at the start of `data` -> a Request, or None when its bytes have not all arrived."""
    data = bytes(data)
    pos = 0
    while data[pos:pos + 2] == b"\r\n" or data[pos:pos + 1] == b"\n":  # empty lines before a request are skipped
        pos += 2 if data[pos] == 13 else 1
    r = _lines(data, pos)
    if r is None:
        return None
    line, pos = r
    parts = line.split(b" ")
    if (len(parts) != 3 or not parts[0] or any(c not in _TCHAR for c in parts[0]) or not parts[1]
            or any(c < 0x21 or c > 0x7e for c in parts[1]) or parts[2] not in (b"HTTP/1.0", b"HTTP/1.1")):
        return Request(pos, bad=400)
    method, target, version = parts[0], parts[1], int(parts[2] == b"HTTP/1.1")
    headers = []
    while True:
        r = _lines(data, pos)
        if r is None:
            return None
        line, pos = r
        if not line:
            break
        name, colon, value = line.partition(b":")
        if (not colon or not name or any(c not in _TCHAR for c in name)
                or any(c != 9 and (c < 0x20 or c == 0x7f) for c in value)):
            return Request(pos, bad=400)                   # obs-fold, no colon, a control byte, ...
        headers.append((name.lower(), value.strip(b" \t")))
        if len(headers) > MAX_HEADERS:
            return Request(pos, bad=431)
    req = Request(pos, method, target, version, headers)
    te = req.header_tokens(b"transfer-encoding")
    if te:
        if te[-1] != b"chunked" or version == 0:
            return Request(pos, bad=400)
        try:
            r = _chunked(data, pos)
        except ValueError:
            return Request(pos, bad=400)
        if r is None:
            return None
        req.body, req.consumed = r
        return req
    lens = set()
    for n, v in headers:
        if n == b"content-length":
            for t in v.split(b","):
                t = t.strip(b" \t")
                if not t or not t.isdigit() or len(t) > 19:
                    return Request(pos, bad=400)
                lens.add(int(t))
    if len(lens) > 1:
        return Request(pos, bad=400)
    n = lens.pop() if lens else 0
    if len(data) < pos + n:
        return None
    req.body, req.consumed = data[pos:pos + n], pos + n
    return req


# ---- JSON as serde_json reads HttpThrottleRequest ---------------------------------------------------------------
class JsonError(ValueError):
    def __init__(self, status, detail):
        super().__init__(detail)
        self.status = status


def _syntax(msg, pos):
    return JsonError(400, "%s at byte %d" % (msg, pos))


def _data(msg):
    return JsonError(422, msg)


class _Json:
    WS = b" \t\n\r"

    def __init__(self, b):
        self.b, self.i, self.depth = b, 0, 0

    def peek(self):
        self.ws()
        return self.b[self.i] if self.i < len(self.b) else None

    def ws(self):
        while self.i < len(self.b) and self.b[self.i] in self.WS:
            self.i += 1

    def expect(self, ch, what):
        c = self.peek()
        if c is None:
            raise _syntax("EOF while parsing %s" % what, self.i)
        if c != ch:
            raise _syntax("expected %s" % chr(ch), self.i)
        self.i += 1

    def ident(self, word):
        if self.b[self.i:self.i + len(word)] != word:
            if word.startswith(self.b[self.i:]):
                raise _syntax("EOF while parsing a value", self.i)
            raise _syntax("expected ident", self.i)
        self.i += len(word)

    def string(self):
        """the string at i (after its opening quote was seen) -> str"""
        self.i += 1
        out, b = [], self.b
        while True:
            j = self.i
            while j < len(b) and b[j] not in b'"\\' and b[j] >= 0x20:
                j += 1
            try:
                out.append(b[self.i:j].decode("utf-8"))
            except UnicodeDecodeError:
                raise _syntax("invalid unicode code point", self.i)
            self.i = j
            if j >= len(b):
                raise _syntax("EOF while parsing a string", j)
            c = b[j]
            if c == 0x22:
                self.i += 1
                return "".join(out)
            if c < 0x20:
                raise _syntax("control character (\\u0000-\\u001F) found while parsing a string", j)
            self.i += 1                                       # a backslash
            if self.i >= len(b):
                raise _syntax("EOF while parsing a string", self.i)
            e = b[self.i]
            self.i += 1
            simple = {0x22: '"', 0x5c: "\\", 0x2f: "/", 0x62: "\b", 0x66: "\f", 0x6e: "\n", 0x72: "\r", 0x74: "\t"}
            if e in simple:
                out.append(simple[e])
                continue
            if e != 0x75:
                raise _syntax("invalid escape", self.i - 1)
            u = self.hex4()
            if 0xDC00 <= u <= 0xDFFF:
                raise _syntax("lone leading surrogate in hex escape", self.i)
            if 0xD800 <= u <= 0xDBFF:
                if b[self.i:self.i + 2] != b"\\u":
                    raise _syntax("unexpected end of hex escape", self.i)
                self.i += 2
                lo = self.hex4()
                if not 0xDC00 <= lo <= 0xDFFF:
                    raise _syntax("lone leading surrogate in hex escape", self.i)
                u = 0x10000 + ((u - 0xD800) << 10) + (lo - 0xDC00)
            out.append(chr(u))

    def hex4(self):
        h = self.b[self.i:self.i + 4]
        if len(h) < 4:
            raise _syntax("EOF while parsing a string", len(self.b))
        if any(c not in b"0123456789abcdefABCDEF" for c in h):
            raise _syntax("invalid escape", self.i)
        self.i += 4
        return int(h, 16)

    def number(self):
        """-> ("int", value) or ("float", text), serde_json's grammar and its integer/float split"""
        b, s = self.b, self.i
        if self.i < len(b) and b[self.i] == 0x2d:
            self.i += 1
        if self.i >= len(b):
            raise _syntax("EOF while parsing a value", self.i)
        if not 0x30 <= b[self.i] <= 0x39:
            raise _syntax("invalid number", self.i)
        if b[self.i] == 0x30 and self.i + 1 < len(b) and 0x30 <= b[self.i + 1] <= 0x39:
            raise _syntax("invalid number", self.i + 1)
        while self.i < len(b) and 0x30 <= b[self.i] <= 0x39:
            self.i += 1
        is_float = False
        if self.i < len(b) and b[self.i] == 0x2e:
            self.i += 1
            is_float = True
            if not (self.i < len(b) and 0x30 <= b[self.i] <= 0x39):
                raise _syntax("invalid number", self.i)
            while self.i < len(b) and 0x30 <= b[self.i] <= 0x39:
                self.i += 1
        if self.i < len(b) and b[self.i] in b"eE":
            self.i += 1
            is_float = True
            if self.i < len(b) and b[self.i] in b"+-":
                self.i += 1
            if not (self.i < len(b) and 0x30 <= b[self.i] <= 0x39):
                raise _syntax("invalid number", self.i)
            while self.i < len(b) and 0x30 <= b[self.i] <= 0x39:
                self.i += 1
        text = b[s:self.i].decode()
        if is_float:
            if float(text) in (float("inf"), float("-inf")):
                raise _syntax("number out of range", s)
            return ("float", text)
        v = int(text)
        if v == 0 and text.startswith("-"):
            return ("float", "-0.0")                          # serde_json reads -0 as a float
        if v < I64_MIN or v > 2**64 - 1:
            return ("float", text)                            # beyond u64 / i64: serde_json falls back to f64
        return ("int", v)

    def any(self):
        """a value of any type (an ignored field's), checked for syntax only"""
        c = self.peek()
        if c is None:
            raise _syntax("EOF while parsing a value", self.i)
        if c in b"[{":
            self.depth += 1
            if self.depth > 128:
                raise _syntax("recursion limit exceeded", self.i)
            close = 0x5d if c == 0x5b else 0x7d
            self.i += 1
            if self.peek() == close:
                self.i += 1
            else:
                while True:
                    if c == 0x7b:
                        if self.peek() != 0x22:
                            raise _syntax("key must be a string", self.i)
                        self.string()
                        self.expect(0x3a, "an object")
                    self.any()
                    n = self.peek()
                    if n == 0x2c:
                        self.i += 1
                        continue
                    if n == close:
                        self.i += 1
                        break
                    raise _syntax("EOF while parsing a list" if n is None else "expected `,` or end", self.i)
            self.depth -= 1
            return ("seq" if c == 0x5b else "map", None)
        if c == 0x22:
            return ("str", self.string())
        if c == 0x74:
            self.ident(b"true")
            return ("bool", True)
        if c == 0x66:
            self.ident(b"false")
            return ("bool", False)
        if c == 0x6e:
            self.ident(b"null")
            return ("null", None)
        if c == 0x2d or 0x30 <= c <= 0x39:
            return self.number()
        raise _syntax("expected value", self.i)

    def field(self, name):
        """the value of a known field, type-checked as serde's derive for HttpThrottleRequest does"""
        c = self.peek()
        if c is None:
            raise _syntax("EOF while parsing a value", self.i)
        if name == "quantity" and c == 0x6e:
            self.ident(b"null")
            return None
        if name == "key":
            if c == 0x22:
                return self.string()
            raise _data("invalid type: %s, expected a string" % self.scalar()[0])
        kind, v = self.scalar()
        if kind == "int" and I64_MIN <= v <= I64_MAX:
            return v
        if kind == "int":
            raise _data("invalid value: integer `%d`, expected i64" % v)
        raise _data("invalid type: %s, expected i64" % ("floating point `%s`" % v if kind == "float" else kind))

    def scalar(self):
        """a value whose type is all that is asked: an array or object is not read past its bracket (serde reports
        the type at once)"""
        c = self.peek()
        if c is not None and c in b"[{":
            self.i += 1
            return ("seq" if c == 0x5b else "map", None)
        return self.any()


def decode_throttle(body):
    """the body of POST /throttle -> (key: str, max_burst, count_per_period, period, quantity); JsonError(status)"""
    j = _Json(bytes(body))
    c = j.peek()
    vals = {}
    if c == 0x7b:
        j.i += 1
        if j.peek() != 0x7d:
            while True:
                if j.peek() is None:
                    raise _syntax("EOF while parsing an object", j.i)
                if j.peek() != 0x22:
                    raise _syntax("key must be a string", j.i)
                name = j.string()
                j.expect(0x3a, "an object")
                if name in FIELDS:
                    if name in vals:
                        raise _data("duplicate field `%s`" % name)
                    vals[name] = j.field(name)
                else:
                    j.any()
                n = j.peek()
                if n == 0x2c:
                    j.i += 1
                    continue
                if n == 0x7d:
                    break
                raise _syntax("EOF while parsing an object" if n is None else "expected `,` or `}`", j.i)
        j.i += 1
        for f in FIELDS[:4]:
            if f not in vals:
                raise _data("missing field `%s`" % f)
    elif c == 0x5b:                                        # a struct from a sequence: the fields in order
        j.i += 1
        for k, f in enumerate(FIELDS):
            if j.peek() == 0x5d:
                raise _data("invalid length %d, expected struct HttpThrottleRequest with 5 elements" % k)
            if k:
                j.expect(0x2c, "a list")
            vals[f] = j.field(f)
        if j.peek() != 0x5d:
            raise _syntax("trailing characters" if j.peek() == 0x2c else "expected `,` or `]`", j.i)
        j.i += 1
    elif c is None:
        raise _syntax("EOF while parsing a value", j.i)
    else:
        kind, _ = j.scalar()
        raise _data("invalid type: %s, expected struct HttpThrottleRequest" % kind)
    j.ws()
    if j.i < len(j.b):
        raise _syntax("trailing characters", j.i)
    q = vals.get("quantity")
    return (vals["key"], vals["max_burst"], vals["count_per_period"], vals["period"], 1 if q is None else q)


def json_content_type(value):
    """axum's rule: a mime type application/json or application/<subtype>+json, parameters allowed"""
    if value is None:
        return False
    try:
        v = value.decode("ascii")
    except UnicodeDecodeError:
        return False
    essence, *params = v.split(";")
    t, slash, sub = essence.strip().lower().partition("/")
    if not slash or not t or not sub or any(c not in _TCHAR for c in (t + sub).encode()):
        return False
    for p in params:
        name, eq, _ = p.strip().partition("=")
        if not eq or not name or any(c not in _TCHAR for c in name.encode()):
            return False
    return t == "application" and (sub == "json" or sub.endswith("+json"))


# ---- responses ---------------------------------------------------------------------------------------------------
def _date(now_ns):
    import email.utils
    return email.utils.formatdate(now_ns // 10**9, usegmt=True)


def response(status, body, now_ns, content_type=None, extra=(), close=False, head=False):
    """a response as hyper writes it: status line, the handler's headers, connection, content-length, date"""
    h = ["HTTP/1.1 %d %s" % (status, REASONS[status])]
    if content_type:
        h.append("content-type: " + content_type)
    h += ["%s: %s" % kv for kv in extra]
    if close:
        h.append("connection: close")
    h += ["content-length: %d" % len(body), "date: " + _date(now_ns)]
    return ("\r\n".join(h) + "\r\n\r\n").encode() + (b"" if head else body)


def format_replies(req, res):
    """gcra_http_format_replies of REQ_DTYPE rows and their RES_DTYPE results"""
    req = np.ascontiguousarray(req, REQ_DTYPE)
    res = np.ascontiguousarray(res, RES_DTYPE)
    buf = C.create_string_buffer(max(len(req), 1) * HTTP_REPLY_MAX)
    w = _native.lib().gcra_http_format_replies(req.ctypes.data, res.ctypes.data, len(req), buf, len(buf))
    return buf.raw[:w]


def handle_request(req, limiter, now_ns, metrics=None):
    """Answer one Request -> (response bytes, n_throttle, close).  A THROTTLE is decided on its own through
    limiter.rate_limit_batch with the key hashed by limiter.store.hash_key; `metrics` (a callable returning text)
    serves GET /metrics, which is 404 without it.  A metrics.Metrics also records the THROTTLE: an error when the
    engine returns a status other than OK (the 500 response), else allowed or denied with its key."""
    now = int(now_ns)
    close = req.close
    if req.bad is not None:
        return response(req.bad, b"", now, close=True), 0, True
    path, method = req.path, req.method
    routes = {b"/throttle": (b"POST",), b"/health": (b"GET", b"HEAD")}
    if metrics is not None:
        routes[b"/metrics"] = (b"GET", b"HEAD")
    if path not in routes:
        return response(404, b"", now, close=close), 0, close
    if method not in routes[path]:
        return response(405, b"", now, extra=[("allow", ",".join(m.decode() for m in routes[path]))],
                        close=close), 0, close
    if path != b"/throttle":
        body = b"OK" if path == b"/health" else metrics().encode()
        return response(200, body, now, TEXT, close=close, head=method == b"HEAD"), 0, close
    if not json_content_type(req.header(b"content-type")):
        return response(415, b"Expected request with `Content-Type: application/json`", now, TEXT,
                        close=close), 0, close
    try:
        key, b, c, p, q = decode_throttle(req.body)
    except JsonError as e:
        prefix = ("Failed to parse the request body as JSON: " if e.status == 400
                  else "Failed to deserialize the JSON body into the target type: ")
        return response(e.status, (prefix + str(e)).encode(), now, TEXT, close=close), 0, close
    row = np.zeros(1, REQ_DTYPE)
    row[0] = (limiter.store.hash_key(key.encode()), b, c, p, q, now)
    res = limiter.rate_limit_batch(row)
    if isinstance(metrics, Metrics):                       # (http.rs:146-160)
        if int(res[0]["status"]) != OK:
            metrics.record_error("http")
        else:
            metrics.record_request("http", bool(res[0]["allowed"]), key)
    out = format_replies(row, res)
    if close:                                              # hyper's connection header, after the handler's
        i = out.index(b"\r\n", out.index(b"\r\n") + 2) + 2
        out = out[:i] + b"connection: close\r\n" + out[i:]
    return out, 1, close


def process_connections(buffers, limiter, now_ns, ring, slot=0, metrics=None):
    """resp.process_connections for HTTP: `ring` is an HttpRing of `limiter`'s engine.  Returns one
    (reply_bytes, bytes_consumed, n_throttle, close) per buffer; close is None, "close" (the request asked for it, or
    was HTTP/1.0) or "error" (a malformed head, answered with 400 or 431).  Rounds as in resp.process_connections: the
    GPU takes every open connection's plain prefix, then each connection stopped at a request that is not plain hands
    that one request to parse_request / handle_request, in list order."""
    now = int(now_ns)
    return ring_rounds(buffers, ring, slot, now, lambda data: general(data, limiter, now, metrics))


def general(data, limiter, now, metrics=None):
    """The general path of a connection stopped at a request that is not plain (stop 2): that one request, at the start
    of `data`, parsed by parse_request and answered by handle_request.  Returns None (the request is incomplete) or
    (bytes consumed, response bytes, THROTTLE decisions, close), close being None, "close" or "error"."""
    req = parse_request(data)
    if req is None:
        return None
    out, n, close = handle_request(req, limiter, now, metrics)
    return req.consumed, out, n, ("error" if req.bad is not None else "close") if close else None
