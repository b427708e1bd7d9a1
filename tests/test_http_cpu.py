"""The HTTP fast path's host side (gcra_http_parse_throttle, gcra_http_format_replies; csrc/gcra_http.cuh) against a
Python model of the plain grammar, against the general path (throttlecrab_b200.http), and byte for byte against a
Python writer of the responses.  No device work."""
import ctypes as C
import email.utils
import json
import re

import numpy as np
import pytest

import throttlecrab_b200 as tc
from throttlecrab_b200 import _native, http

NOW = 1_700_000_000 * 10**9
NS = 10**9
I64_MIN, I64_MAX = -2**63, 2**63 - 1
L = _native.lib()


def request(body, headers=None, line=b"POST /throttle HTTP/1.1"):
    """a request in curl's header layout (Host, User-Agent, Accept, Content-Type, Content-Length) unless `headers`"""
    if isinstance(body, dict):
        body = json.dumps(body).encode()
    if headers is None:
        headers = [(b"Host", b"localhost:8080"), (b"User-Agent", b"curl/8.5.0"), (b"Accept", b"*/*"),
                   (b"Content-Type", b"application/json"), (b"Content-Length", str(len(body)).encode())]
    return line + b"\r\n" + b"".join(n + b": " + v + b"\r\n" for n, v in headers) + b"\r\n" + body


def body_of(key="k", b=3, c=10, p=60, q=None, order=None, sep=(", ", ": ")):
    m = {"key": key, "max_burst": b, "count_per_period": c, "period": p}
    if q is not None:
        m["quantity"] = q
    names = order or list(m)
    return ("{" + sep[0].join(json.dumps(n) + sep[1] + (json.dumps(m[n], ensure_ascii=False)) for n in names)
            + "}").encode()


def walk(buf, cap=1 << 12, h=None):
    """gcra_http_parse_throttle -> (rows, consumed, n, stop)"""
    req = np.zeros(max(cap, 1), tc.REQ_DTYPE)
    used, cnt, stop = C.c_uint64(), C.c_uint32(), C.c_int32()
    assert L.gcra_http_parse_throttle(h, buf, len(buf), NOW, cap, req.ctypes.data, C.byref(used), C.byref(cnt),
                                      C.byref(stop)) == 0
    return req[:cnt.value], used.value, cnt.value, stop.value


# ---- a model of the plain grammar: the head line by line, the body by regular expressions ------------------------
RL = b"POST /throttle HTTP/1.1\r\n"
TOKEN = rb"[!#$%&'*+\-.^_`|~0-9A-Za-z]*"
VALUE = rb"[\t\x20-\x7e\x80-\xff]*"
WS = rb"[ \t\n\r]*"
INT = rb"-?(?:0|[1-9][0-9]{0,18})"
MEMBER = re.compile(WS + rb'"([^"\\\x00-\x1f]*)"' + WS + b":" + WS + rb'("[^"\\\x00-\x1f]*"|' + INT + rb"|null)" + WS)


def model_body(body):
    """a whole body -> (key bytes, b, c, p, q), or None if it is not plain"""
    m = re.match(WS + b"{", body)
    if not m:
        return None
    pos, vals = m.end(), {}
    while True:
        m = MEMBER.match(body, pos)
        if not m:
            return None
        name, v = m.group(1).decode("latin-1"), m.group(2)
        if name not in http.FIELDS or name in vals:
            return None
        if name == "key":
            if not v.startswith(b'"'):
                return None
            try:
                v[1:-1].decode("utf-8")
            except UnicodeDecodeError:
                return None
            vals[name] = v[1:-1]
        elif v == b"null" and name == "quantity":
            vals[name] = 1
        else:
            if v.startswith(b'"') or v == b"null" or v == b"-0" or int(v) > I64_MAX or int(v) < -I64_MAX:
                return None
            vals[name] = int(v)
        pos = m.end()
        if body[pos:pos + 1] == b",":
            pos += 1
            continue
        if body[pos:pos + 1] != b"}":
            return None
        pos += 1
        break
    if any(f not in vals for f in http.FIELDS[:4]) or not re.fullmatch(WS, body[pos:]):
        return None
    return (vals["key"], vals["max_burst"], vals["count_per_period"], vals["period"], vals.get("quantity", 1))


def model(buf):
    """the request at buf's start -> (0, its length, fields) | (1, 0, None) | (2, 0, None); a body that has not all
    arrived is not modelled (None)"""
    n = len(buf)
    if buf[:len(RL)] != RL[:n]:
        return 2, 0, None
    if n < len(RL):
        return 1, 0, None
    pos, count, clen, ctype = len(RL), 0, None, False
    while True:
        if pos >= n:
            return 1, 0, None
        if buf[pos] == 13:
            if pos + 1 >= n:
                return 1, 0, None
            if buf[pos + 1] != 10:
                return 2, 0, None
            pos += 2
            break
        if count == 64:
            return 2, 0, None
        name = re.match(TOKEN, buf[pos:]).group(0)
        colon = pos + len(name)
        if colon >= n:
            return 1, 0, None
        if buf[colon] != 58 or not name:
            return 2, 0, None
        vend = colon + 1 + len(re.match(VALUE, buf[colon + 1:]).group(0))
        if vend >= n:
            return 1, 0, None
        if buf[vend] != 13:
            return 2, 0, None
        if vend + 1 >= n:
            return 1, 0, None
        if buf[vend + 1] != 10:
            return 2, 0, None
        value, pos, count = buf[colon + 1:vend].strip(b" \t"), vend + 2, count + 1
        lname = name.lower()
        if lname == b"content-length":
            if clen is not None or not re.fullmatch(rb"[0-9]{1,5}", value) or int(value) > 65536:
                return 2, 0, None
            clen = int(value)
        elif lname == b"content-type":
            if ctype or value.lower() != b"application/json":
                return 2, 0, None
            ctype = True
        elif lname in (b"transfer-encoding", b"connection", b"expect", b"upgrade"):
            return 2, 0, None
    if clen is None or not ctype:
        return 2, 0, None
    if n - pos < clen:
        return None
    f = model_body(buf[pos:pos + clen])
    return (2, 0, None) if f is None else (0, pos + clen, f)


def check_one(buf):
    """the host walk, the model and (where plain) the general path agree on the request at buf's start"""
    rows, used, n, stop = walk(buf, cap=1)
    want = model(buf)
    if want is None:
        assert stop in (1, 2) and n == 0
        return stop
    rc, end, f = want
    if rc == 0:
        assert (n, used) == (1, end), buf
        assert stop == (0 if end == len(buf) else 3), buf
        key, b, c, p, q = f
        r = rows[0]
        assert int(r["key_hash"]) == tc.hash_key(key)
        assert [int(r[x]) for x in ("max_burst", "count_per_period", "period", "quantity", "now_ns")] == [b, c, p, q, NOW]
        g = http.parse_request(buf)                          # the general path reads the same request
        assert g is not None and g.bad is None and g.consumed == end and not g.close
        assert (g.method, g.path) == (b"POST", b"/throttle") and http.json_content_type(g.header(b"content-type"))
        assert http.decode_throttle(g.body) == (key.decode(), b, c, p, q)
        return 0
    assert (n, used, stop) == (0, 0, rc), (buf, stop, rc)
    return rc


# ---- the reference's own example ---------------------------------------------------------------------------------
README = b'{"key": "test", "max_burst": 3, "count_per_period": 10, "period": 60}'
RLEN = b"%d" % len(README)


def test_readme_curl_request_parses_to_its_row():
    buf = request(README)
    assert buf.startswith(b"POST /throttle HTTP/1.1\r\nHost: localhost:8080\r\nUser-Agent: curl/")
    rows, used, n, stop = walk(buf)
    assert (used, n, stop) == (len(buf), 1, 0)
    assert tuple(int(rows[0][f]) for f in tc.REQ_DTYPE.names) == (tc.hash_key("test"), 3, 10, 60, 1, NOW)
    assert check_one(buf) == 0
    # a fresh key: allowed, limit 3, remaining 2 (the result a fresh GCRA entry gives; the oracle decides it here)
    import oracle
    st = oracle.OracleStore(oracle.PERIODIC, capacity=10, created_ns=NOW, p0=NS)
    s, a, rem, reset, retry = st.rate_limit("test", 3, 10, 60, 1, NOW)
    res = np.zeros(1, tc.RES_DTYPE)
    res[0] = (rem, reset, retry, s, a, [0, 0, 0])
    out = http.format_replies(rows, res)
    body = out.split(b"\r\n\r\n", 1)[1]
    assert json.loads(body) == {"allowed": True, "limit": 3, "remaining": 2, "reset_after": reset // NS,
                                "retry_after": 0}
    assert body.startswith(b'{"allowed":true,"limit":3,"remaining":2,"reset_after":')


# ---- the grammar -------------------------------------------------------------------------------------------------
def test_minimal_request_is_min_frame_bytes():
    body = b'{"key":"","max_burst":0,"count_per_period":0,"period":0}'
    buf = request(body, [(b"content-length", b"56"), (b"content-type", b"application/json")]).replace(b": ", b":")
    assert len(body) == 56 and len(buf) == 133       # gcra_http::MIN_FRAME_BYTES
    assert walk(buf)[1:] == (133, 1, 0)


def test_header_case_order_and_extra_headers():
    body = body_of()
    base = [(b"Content-Type", b"application/json"), (b"Content-Length", str(len(body)).encode())]
    extra = [(b"Host", b"x"), (b"Accept", b"*/*"), (b"X-Trace", b"\x80\xff opaque"), (b"Accept-Encoding", b"gzip")]
    rng = np.random.default_rng(3)
    for _ in range(200):
        hs = base + [extra[int(i)] for i in rng.choice(len(extra), int(rng.integers(0, 5)))]
        hs = [hs[int(i)] for i in rng.permutation(len(hs))]
        hs = [(bytes(c ^ 0x20 if 0x61 <= (c | 0x20) <= 0x7a and rng.random() < 0.5 else c for c in n),
               v if n.lower() != b"content-type" else bytes(c ^ 0x20 if 0x61 <= c <= 0x7a and rng.random() < 0.3
                                                            else c for c in v))
              for n, v in hs]
        sep = [b": ", b":", b":\t ", b" :"][int(rng.integers(0, 4))]
        buf = RL[:-2] + b"\r\n" + b"".join(n + sep + v + (b" \t" if rng.random() < 0.3 else b"") + b"\r\n"
                                           for n, v in hs) + b"\r\n" + body
        rc = check_one(buf)
        assert rc == (2 if sep == b" :" else 0), buf
    # 64 header lines is the most the fast path takes
    many = base + [(b"X-%d" % i, b"v") for i in range(62)]
    assert check_one(request(body, many)) == 0
    assert check_one(request(body, many + [(b"X-last", b"v")])) == 2


def test_member_order_whitespace_and_quantity():
    for order in (None, ["period", "key", "count_per_period", "max_burst"], ["max_burst", "period", "count_per_period", "key"]):
        for sep in ((",", ":"), (" , ", " : "), (",\n\t", ":\r\n ")):
            for q in (None, 1, 7, -3):
                names = (order or ["key", "max_burst", "count_per_period", "period"]) + (["quantity"] if q is not None else [])
                b = b" \n" + body_of("k:%s" % q, 5, 10, 60, q, names, sep) + b"\t\r\n"
                assert check_one(request(b)) == 0
    null = b'{"key":"n","max_burst":1,"count_per_period":2,"period":3,"quantity" : null }'
    assert check_one(request(null)) == 0
    assert walk(request(null))[0][0]["quantity"] == 1


def test_utf8_keys_and_post_inside_keys():
    for key in ["kéy", "ключ", "键", "😀x", "POST /throttle HTTP/1.1", "a" * 3000, ""]:
        buf = request(body_of(key))
        assert check_one(buf) == 0
        assert int(walk(buf)[0][0]["key_hash"]) == tc.hash_key(key.encode())
    for bad in [b"\xff", b"\xc0\xaf", b"\xed\xa0\x80", b"\xf4\x90\x80\x80"]:     # not UTF-8: the general path
        buf = request(b'{"key":"' + bad + b'","max_burst":1,"count_per_period":1,"period":1}')
        assert check_one(buf) == 2
        assert http.handle_request(http.parse_request(buf), None, NOW)[0].startswith(b"HTTP/1.1 400 ")


def test_every_truncation_of_a_valid_request_is_stop_1():
    for buf in [request(README), request(body_of("kéy", 1, 2, 3, None, None, (" ,", ": ")) + b"  "),
                request(b'{"key":"n","max_burst":-12,"count_per_period":2,"period":3,"quantity":null}')]:
        for cut in range(1, len(buf)):
            rows, used, n, stop = walk(buf[:cut])
            assert (used, n, stop) == (0, 0, 1), (cut, buf[:cut])
        assert walk(buf)[1:] == (len(buf), 1, 0)
        two = buf + buf
        for cut in range(len(buf) + 1, len(two)):
            assert walk(two[:cut])[1:] == (len(buf), 1, 1)


NEAR_MISSES = {
    "chunked": request(b"%x\r\n" % len(README) + README + b"\r\n0\r\n\r\n", [(b"Content-Type", b"application/json"),
                                                                (b"Transfer-Encoding", b"chunked")]),
    "connection close": request(README, [(b"Content-Type", b"application/json"), (b"Content-Length", RLEN),
                                         (b"Connection", b"close")]),
    "keep-alive": request(README, [(b"Connection", b"keep-alive"), (b"Content-Type", b"application/json"),
                                   (b"Content-Length", RLEN)]),
    "expect": request(README, [(b"Content-Type", b"application/json"), (b"Content-Length", RLEN),
                               (b"Expect", b"100-continue")]),
    "upgrade": request(README, [(b"Content-Type", b"application/json"), (b"Content-Length", RLEN),
                                (b"Upgrade", b"h2c")]),
    "duplicate length": request(README, [(b"Content-Type", b"application/json"), (b"Content-Length", RLEN),
                                         (b"Content-Length", RLEN)]),
    "short length": request(README, [(b"Content-Type", b"application/json"), (b"Content-Length", b"%d" % (len(README) - 1))]),
    "long length": request(README + b"}", [(b"Content-Type", b"application/json"), (b"Content-Length", b"%d" % (len(README) + 1))]),
    "signed length": request(README, [(b"Content-Type", b"application/json"), (b"Content-Length", b"+" + RLEN)]),
    "no length": request(README, [(b"Content-Type", b"application/json")]),
    "no type": request(README, [(b"Content-Length", RLEN)]),
    "type with charset": request(README, [(b"Content-Type", b"application/json; charset=utf-8"),
                                          (b"Content-Length", RLEN)]),
    "duplicate type": request(README, [(b"Content-Type", b"application/json"), (b"Content-Type", b"application/json"),
                                       (b"Content-Length", RLEN)]),
    "escape": request(b'{"key": "te\\u0073t", "max_burst": 3, "count_per_period": 10, "period": 60}'),
    "float": request(b'{"key": "test", "max_burst": 3.0, "count_per_period": 10, "period": 60}'),
    "exponent": request(b'{"key": "test", "max_burst": 3e0, "count_per_period": 10, "period": 60}'),
    "minus zero": request(b'{"key": "test", "max_burst": -0, "count_per_period": 10, "period": 60}'),
    "leading zero": request(b'{"key": "test", "max_burst": 03, "count_per_period": 10, "period": 60}'),
    "unknown member": request(b'{"key": "test", "max_burst": 3, "count_per_period": 10, "period": 60, "x": 1}'),
    "duplicate member": request(b'{"key": "test", "max_burst": 3, "max_burst": 3, "count_per_period": 10, "period": 60}'),
    "missing member": request(b'{"key": "test", "max_burst": 3, "count_per_period": 10}'),
    "20 digits": request(b'{"key": "test", "max_burst": 10000000000000000000, "count_per_period": 10, "period": 60}'),
    "i64 max + 1": request(b'{"key": "test", "max_burst": 9223372036854775808, "count_per_period": 10, "period": 60}'),
    "i64 min": request(b'{"key": "test", "max_burst": -9223372036854775808, "count_per_period": 10, "period": 60}'),
    "string number": request(b'{"key": "test", "max_burst": "3", "count_per_period": 10, "period": 60}'),
    "array body": request(b'["test", 3, 10, 60, null]'),
    "trailing comma": request(b'{"key": "test", "max_burst": 3, "count_per_period": 10, "period": 60,}'),
    "http/1.0": request(README, line=b"POST /throttle HTTP/1.0"),
    "query": request(README, line=b"POST /throttle?x HTTP/1.1"),
    "get": request(README, line=b"GET /throttle HTTP/1.1"),
    "bare lf": request(README).replace(b"\r\n", b"\n", 2),
    "obs-fold": request(README).replace(b"Accept: */*\r\n", b"Accept: */*\r\n  folded\r\n"),
    "no colon": request(README).replace(b"Accept: */*", b"Accept */*"),
    "control byte": request(README).replace(b"Accept: */*", b"Accept: *\x01*"),
}


@pytest.mark.parametrize("name", sorted(NEAR_MISSES))
def test_near_misses_are_stop_2(name):
    buf = NEAR_MISSES[name]
    assert walk(buf)[1:] == (0, 0, 2)
    assert check_one(buf) == 2
    g = http.parse_request(buf)                            # the general path answers every one of them
    assert g is not None


def _fuzz_request(rng):
    keys = ["a", "user:1", "kéy", "", "x" * 70, "POST ", "with\"quote", "back\\slash", "tab\there", "é" * 5]
    nums = [0, 1, 3, 60, -1, -5, 2**31, I64_MAX, -I64_MAX, I64_MIN, 2**63, "1.5", "1e3", "-0", "007", "null", '"5"']
    def num():
        return nums[int(rng.integers(0, len(nums)))] if rng.random() < 0.15 else int(rng.integers(1, 200))
    m = {"key": keys[int(rng.integers(0, len(keys)))], "max_burst": num(), "count_per_period": num(), "period": num()}
    if rng.random() < 0.4:
        m["quantity"] = num() if rng.random() < 0.8 else None
    if rng.random() < 0.05:
        m["extra"] = [1, 2]
    names = list(m)
    rng.shuffle(names)
    if rng.random() < 0.05 and names:
        names.pop()
    ws = [b"", b" ", b"\n", b"\t "]
    w = lambda: ws[int(rng.integers(0, len(ws)))]
    parts = [json.dumps(n).encode() + w() + b":" + w() + (v.encode() if isinstance(v, str) and n != "key" else
                                                         json.dumps(v, ensure_ascii=False).encode())
             for n, v in ((n, m[n]) for n in names)]
    body = w() + b"{" + w() + (w() + b"," + w()).join(parts) + w() + b"}" + w()
    buf = request(body)
    if rng.random() < 0.1:
        f = bytearray(buf)
        for _ in range(int(rng.integers(1, 3))):
            pos = int(rng.integers(0, len(f)))
            f[pos] = int(rng.choice([0x0d, 0x0a, 0x22, 0x3a, 0x2c, 0x7b, 0x7d, 0x30, 0x20, 0x5c, 0xff, 0x41]))
        buf = bytes(f)
    return buf


def test_fuzz_host_walk_against_the_model_and_the_general_path():
    rng = np.random.default_rng(20261017)
    kinds = {0: 0, 1: 0, 2: 0}
    for _ in range(4000):
        buf = _fuzz_request(rng)
        kinds[check_one(buf)] += 1
        if rng.random() < 0.2:                                  # a cut: stop 1 when the whole request was plain
            cut = int(rng.integers(1, len(buf)))
            if model(buf)[0] == 0 and model(buf)[1] == len(buf):
                assert walk(buf[:cut])[1:] == (0, 0, 1)
    assert kinds[0] > 1500 and kinds[2] > 300, kinds
    # pipelines: the walk takes the plain prefix, request by request
    for _ in range(300):
        reqs = [_fuzz_request(rng) for _ in range(int(rng.integers(1, 8)))]
        buf = b"".join(reqs)
        rows, used, n, stop = walk(buf)
        at, k = 0, 0
        while at < len(buf):
            m = model(buf[at:])
            if m is None or m[0] != 0:
                break
            at += m[1]
            k += 1
        assert (used, n) == (at, k)
        if at < len(buf) and m is not None:
            assert stop == m[0]


def test_row_cap_is_stop_3():
    one = request(README)
    assert walk(one * 5, cap=3)[1:] == (3 * len(one), 3, 3)
    assert walk(one * 3, cap=3)[1:] == (3 * len(one), 3, 0)


# ---- responses ---------------------------------------------------------------------------------------------------
def py_reply(q, r):
    """the response as a Python writer sees it: json.dumps for the body, email.utils.formatdate for the date"""
    def secs(ns):
        return -(-ns // NS) if ns < 0 else ns // NS         # toward zero, as the engine's i64 division
    st = int(r["status"])
    if st == tc.OK:
        body = {"allowed": bool(r["allowed"]), "limit": int(q["max_burst"]), "remaining": int(r["remaining"]),
                "reset_after": secs(int(r["reset_after_ns"])), "retry_after": secs(int(r["retry_after_ns"]))}
        line = "HTTP/1.1 200 OK"
    else:
        why = {tc.NEGATIVE_QUANTITY: "negative quantity: %d" % int(q["quantity"]),
               tc.INVALID_RATE_LIMIT: "invalid rate limit parameters"}.get(st, "internal error")
        body = {"error": "Internal server error: Rate limit check failed: " + why}
        line = "HTTP/1.1 500 Internal Server Error"
    b = json.dumps(body, separators=(",", ":")).encode()
    date = email.utils.formatdate(int(q["now_ns"]) // NS, usegmt=True)
    return ("%s\r\ncontent-type: application/json\r\ncontent-length: %d\r\ndate: %s\r\n\r\n" % (line, len(b), date)
            ).encode() + b


def _rows(cases):
    req = np.zeros(len(cases), tc.REQ_DTYPE)
    res = np.zeros(len(cases), tc.RES_DTYPE)
    for i, (qq, rr) in enumerate(cases):
        req[i] = (1, qq.get("b", 3), 10, 60, qq.get("q", 1), qq.get("now", NOW))
        res[i] = (rr.get("rem", 2), rr.get("reset", 6 * NS), rr.get("retry", 0), rr.get("st", tc.OK),
                  rr.get("a", 1), [0, 0, 0])
    return req, res


def test_format_replies_bytes_statuses_and_dates():
    dates = [0, -1, -NS, NS - 1, 951782400 * NS, 951868799 * NS + 5, 1709164800 * NS, 1709251199 * NS,
             -2203891200 * NS, 4107542400 * NS, I64_MIN, I64_MAX, I64_MIN + NS, I64_MAX - NS, NOW]
    cases = []
    for d in dates:
        cases.append(({"now": d}, {}))
    for st in (tc.OK, tc.NEGATIVE_QUANTITY, tc.INVALID_RATE_LIMIT, tc.INTERNAL, 77):
        for a in (0, 1):
            cases.append(({"q": -5 if st == tc.NEGATIVE_QUANTITY else 1}, {"st": st, "a": a}))
    rng = np.random.default_rng(9)
    for _ in range(2000):
        cases.append(({"b": int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64)),
                       "q": int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64)),
                       "now": int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64))},
                      {"rem": int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64)),
                       "reset": int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64)),
                       "retry": int(rng.integers(-10**12, 10**12)), "st": int(rng.integers(0, 4)),
                       "a": int(rng.integers(0, 2))}))
    req, res = _rows(cases)
    want = b"".join(py_reply(q, r) for q, r in zip(req, res))
    assert http.format_replies(req, res) == want
    # the dates named in the issue of the format: the epoch, one second before, leap days, the ends of the i64 range
    got = [http.format_replies(req[i:i + 1], res[i:i + 1]).split(b"date: ")[1][:29] for i in range(len(dates))]
    assert got[0] == b"Thu, 01 Jan 1970 00:00:00 GMT" and got[1] == got[2] == b"Wed, 31 Dec 1969 23:59:59 GMT"
    assert got[4] == b"Tue, 29 Feb 2000 00:00:00 GMT" and got[6] == b"Thu, 29 Feb 2024 00:00:00 GMT"
    assert got[8] == b"Thu, 01 Mar 1900 00:00:00 GMT"
    assert got[10] == b"Tue, 21 Sep 1677 00:12:43 GMT" and got[11] == b"Fri, 11 Apr 2262 23:47:16 GMT"
    # too little room: nothing written
    buf = C.create_string_buffer(tc.HTTP_REPLY_MAX * 2 - 1)
    assert L.gcra_http_format_replies(req.ctypes.data, res.ctypes.data, 2, buf, len(buf)) == 0


def test_longest_reply_is_pinned():
    ext = [I64_MIN, I64_MAX, -1, 0]
    cases = []
    for b in ext:
        for rem in ext:
            for t in ext:
                for now in (I64_MIN, I64_MAX, 0):
                    cases.append(({"b": b, "now": now}, {"rem": rem, "reset": t, "retry": t, "a": 0}))
    for q in ext:
        for st in (1, 2, 3):
            for now in (I64_MIN, 0):
                cases.append(({"q": q, "now": now}, {"st": st}))
    req, res = _rows(cases)
    lens = [len(http.format_replies(req[i:i + 1], res[i:i + 1])) for i in range(len(req))]
    ok = max(n for n, r in zip(lens, res) if r["status"] == tc.OK)
    err = max(n for n, r in zip(lens, res) if r["status"] != tc.OK)
    assert (ok, err) == (240, 226)
    assert max(ok, err) <= tc.HTTP_REPLY_MAX == 256


# ---- the general path ----------------------------------------------------------------------------------------------
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


def _status(buf, metrics=None):
    g = http.parse_request(buf)
    out, n, close = http.handle_request(g, _Decider(), NOW, metrics)
    return int(out.split(b" ", 2)[1]), out, n, close


def test_general_path_statuses():
    ct = (b"Content-Type", b"application/json")
    def post(body, headers=None, **kw):
        return request(body, headers or [ct, (b"Content-Length", str(len(body)).encode())], **kw)
    assert _status(request(README))[0] == 200
    s, out, n, close = _status(b"GET /health HTTP/1.1\r\nHost: x\r\n\r\n")
    assert (s, n, close) == (200, 0, False) and out.endswith(b"\r\n\r\nOK")
    assert b"content-type: text/plain; charset=utf-8\r\ncontent-length: 2\r\ndate: " in out
    assert _status(b"GET /nope HTTP/1.1\r\n\r\n")[1].split(b"\r\n")[1:3] == [b"content-length: 0",
                                                                           _status(b"GET / HTTP/1.1\r\n\r\n")[1].split(b"\r\n")[2]]
    assert _status(b"GET /metrics HTTP/1.1\r\n\r\n")[0] == 404
    assert _status(b"GET /metrics HTTP/1.1\r\n\r\n", metrics=lambda: "m 1\n")[1].endswith(b"m 1\n")
    s, out, _, _ = _status(b"GET /throttle HTTP/1.1\r\n\r\n")
    assert s == 405 and b"\r\nallow: POST\r\n" in out
    assert b"\r\nallow: GET,HEAD\r\n" in _status(b"POST /health HTTP/1.1\r\ncontent-length: 0\r\n\r\n")[1]
    assert _status(post(README, [(b"Content-Length", RLEN)]))[0] == 415
    assert _status(post(README, [(b"Content-Type", b"text/json"), (b"Content-Length", RLEN)]))[0] == 415
    for good_ct in (b"application/json; charset=utf-8", b"application/vnd.api+json", b"Application/JSON"):
        assert _status(post(README, [(b"Content-Type", good_ct), (b"Content-Length", RLEN)]))[0] == 200, good_ct
    for body, want in [(b'{"key": "a", "max_burst": NaN, "count_per_period": 1, "period": 1}', 400),
                       (b'{"key": "a", "max_burst": Infinity, "count_per_period": 1, "period": 1}', 400),
                       (b'{"key": "\\ud800", "max_burst": 1, "count_per_period": 1, "period": 1}', 400),
                       (b'{"key": "\\udc00x", "max_burst": 1, "count_per_period": 1, "period": 1}', 400),
                       (b'{"key": "a", "max_burst": 1, "count_per_period": 1, "period": 1', 400),
                       (b'{"key": "a", "max_burst": 1, "count_per_period": 1, "period": 1} x', 400),
                       (b'', 400),
                       (b'{"key": "a", "max_burst": 9223372036854775808, "count_per_period": 1, "period": 1}', 422),
                       (b'{"key": "a", "max_burst": -9223372036854775809, "count_per_period": 1, "period": 1}', 422),
                       (b'{"key": "a", "max_burst": 1.0, "count_per_period": 1, "period": 1}', 422),
                       (b'{"key": "a", "max_burst": -0, "count_per_period": 1, "period": 1}', 422),
                       (b'{"key": "a", "key": "b", "max_burst": 1, "count_per_period": 1, "period": 1}', 422),
                       (b'{"key": "a", "count_per_period": 1, "period": 1}', 422),
                       (b'{"key": 5, "max_burst": 1, "count_per_period": 1, "period": 1}', 422),
                       (b'{"key": "a", "max_burst": "1", "count_per_period": 1, "period": 1}', 422),
                       (b'5', 422),
                       (b'{"key": "a", "max_burst": -9223372036854775808, "count_per_period": 1, "period": 1}', 500),
                       (b'{"key": "\\u00e9\\n", "max_burst": 1, "count_per_period": 1, "period": 1, "quantity": null,'
                        b' "other": {"deep": [1, 2.5e3, null, true]}}', 200),
                       (b'["a", 1, 1, 1, null]', 200)]:
        s, out, n, _ = _status(post(body))
        assert (s, n) == (want, int(want in (200, 500))), (body, out)
        if want == 400:
            assert out.split(b"\r\n\r\n", 1)[1].startswith(b"Failed to parse the request body as JSON: ")
        if want == 422:
            assert out.split(b"\r\n\r\n", 1)[1].startswith(b"Failed to deserialize the JSON body into the target type: ")
    # escapes are decoded before hashing: the same key as its plain spelling
    esc = post(b'{"key": "te\\u0073t", "max_burst": 3, "count_per_period": 10, "period": 60}')
    assert _status(esc)[1].split(b"\r\n\r\n")[1] == _status(request(README))[1].split(b"\r\n\r\n")[1]


def test_general_path_connections():
    assert http.parse_request(request(README)[:-1]) is None
    assert http.parse_request(b"POST /throttle HTTP/1.1\r\nContent-Type: application/json\r\n") is None
    bad = http.parse_request(b"POST /throttle HTTP/1.1\r\n folded: x\r\n\r\n")
    s, out, _, close = _status(b"NOT A REQUEST\r\n\r\n")
    assert bad.bad == 400 and (s, close) == (400, True) and b"connection: close" in out
    lf = request(README).replace(b"\r\n", b"\n")                 # bare LF is allowed by httparse
    assert _status(lf)[0] == 200
    s, out, _, close = _status(NEAR_MISSES["connection close"])
    assert (s, close) == (200, True) and out.split(b"\r\n")[2] == b"connection: close"
    assert _status(NEAR_MISSES["http/1.0"])[3] is True
    chunked = (b"POST /throttle HTTP/1.1\r\nContent-Type: application/json\r\nTransfer-Encoding: chunked\r\n\r\n"
               b"10\r\n" + README[:16] + b"\r\n" + b"%x;ext=1\r\n" % (len(README) - 16) + README[16:] + b"\r\n0\r\n\r\n")
    g = http.parse_request(chunked + b"next")
    assert g.body == README and g.consumed == len(chunked)
    assert http.parse_request(chunked[:-3]) is None
    assert _status(chunked)[0] == 200
