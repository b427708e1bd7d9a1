// gcra_http.cuh -- the grammar of a plain POST /throttle request and the text of its response, ONE definition for the
// host (gcra_http_parse_throttle, gcra_http_format_replies in gcra_resp.inc) and the HTTP ring's kernels
// (gcra_resp_ring.cu).  The cursor, the UTF-8 rule, the byte sinks, the number writer and the error texts are
// gcra_resp.cuh's.
//
// The fast path only accepts the plain shape (the reference's transport/http.rs route, as curl and most clients send
// it):
//     POST /throttle HTTP/1.1 CRLF
//     (name ":" OWS value OWS CRLF) x 0..64     Content-Length (1-5 digits, <= 65536) and
//                                                Content-Type: application/json exactly once each; no
//                                                Transfer-Encoding, Connection, Expect or Upgrade
//     CRLF
//     <Content-Length bytes>: ws { "key": "<string>", "max_burst": i, "count_per_period": i, "period": i
//                             [, "quantity": i | null] } ws   (members in any order, each once)
// with no escape and no control byte in the key (so its bytes are the decoded String), UTF-8 keys, and integers
// -?(0|[1-9][0-9]*) of at most 19 digits within (-2^63, 2^63) other than -0 (which serde_json reads as a float).
// Everything else -- another route, other headers' combinations, escapes, floats, unknown members -- is "not plain"
// and left to the general path (throttlecrab_b200/http.py).
#pragma once
#include "gcra_resp.cuh"

namespace gcra_http {

#define GCRA_HTTP_HD __host__ __device__ __forceinline__

using gcra_resp::Count;
using gcra_resp::Cursor;
using gcra_resp::Frame;
using gcra_resp::Write;

constexpr uint32_t MAX_HEADERS = 64;
constexpr uint32_t MAX_BODY = 65536;

GCRA_HTTP_HD unsigned char lower(unsigned char c) { return c >= 'A' && c <= 'Z' ? (unsigned char)(c - 'A' + 'a') : c; }

// `s[0, n)` equals the lower-case `lit` in any ASCII case
GCRA_HTTP_HD bool iequals(const unsigned char *s, uint32_t n, const char *lit) {
    uint32_t i = 0;
    for (; i < n && lit[i]; i++)
        if (lower(s[i]) != (unsigned char)lit[i]) return false;
    return i == n && !lit[i];
}

// `s[0, n)` equals `lit` exactly
GCRA_HTTP_HD bool equals(const unsigned char *s, uint32_t n, const char *lit) {
    uint32_t i = 0;
    for (; i < n && lit[i]; i++)
        if (s[i] != (unsigned char)lit[i]) return false;
    return i == n && !lit[i];
}

// RFC 9110 tchar
GCRA_HTTP_HD bool is_tchar(unsigned char c) {
    if ((c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z')) return true;
    switch (c) {
    case '!': case '#': case '$': case '%': case '&': case '\'': case '*': case '+': case '-': case '.': case '^':
    case '_': case '`': case '|': case '~': return true;
    default: return false;
    }
}

// a field value byte: HTAB, SP, VCHAR, obs-text
GCRA_HTTP_HD bool is_vbyte(unsigned char c) { return c == '\t' || (c >= 0x20 && c != 0x7f); }

GCRA_HTTP_HD bool is_ws(unsigned char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }

// ---- body -------------------------------------------------------------------------------------------------------
// Every reader returns 0 (done, the cursor moves), 1 (the bytes end first) or 2 (not plain).  The body cursor ends
// where the bytes at hand end; parse_frame turns a 1 into a 2 when the whole body was at hand.
GCRA_HTTP_HD void skip_ws(Cursor &c) {
    while (c.p < c.end && is_ws(*c.p)) c.p++;
}

// -?(0|[1-9][0-9]*), at most 19 digits, within (-2^63, 2^63), not -0, followed by a byte that is not part of a number
GCRA_HTTP_HD int read_json_int(Cursor &c, int64_t &out) {
    const unsigned char *p = c.p;
    const bool neg = p < c.end && *p == '-';
    if (neg) p++;
    if (p >= c.end) return 1;
    if (*p < '0' || *p > '9') return 2;
    uint64_t v = 0;
    int digits = 0;
    while (p < c.end && *p >= '0' && *p <= '9') {
        if (digits == 19 || (digits == 1 && v == 0)) return 2;     // 20 digits, or a leading zero
        v = v * 10 + (uint64_t)(*p - '0');
        p++; digits++;
    }
    if (p >= c.end) return 1;
    if (*p == '.' || *p == 'e' || *p == 'E') return 2;
    if (v > (uint64_t)INT64_MAX || (neg && v == 0)) return 2;
    out = neg ? -(int64_t)v : (int64_t)v;
    c.p = p;
    return 0;
}

// a string with no escape and no control byte: its bytes
GCRA_HTTP_HD int read_plain_string(Cursor &c, const unsigned char *&s, uint32_t &n) {
    const unsigned char *p = c.p;
    if (p >= c.end) return 1;
    if (*p != '"') return 2;
    s = ++p;
    while (p < c.end && *p != '"') {
        if (*p == '\\' || *p < 0x20) return 2;
        p++;
    }
    if (p >= c.end) return 1;
    n = (uint32_t)(p - s);
    c.p = p + 1;
    return 0;
}

// the body { members } with its surrounding whitespace, exactly up to c.end
GCRA_HTTP_HD int read_body(Cursor &c, Frame &fr) {
    int rc;
    skip_ws(c);
    if (c.p >= c.end) return 1;
    if (*c.p != '{') return 2;
    c.p++;
    uint32_t seen = 0;                                  // members read: bit 0 key, 1..4 the numbers
    fr.a[3] = 1;                                        // a missing or null quantity is 1 (transport/http.rs)
    for (;;) {
        skip_ws(c);
        const unsigned char *name;
        uint32_t nl;
        if ((rc = read_plain_string(c, name, nl))) return rc;
        int m;
        if (equals(name, nl, "key")) m = 0;
        else if (equals(name, nl, "max_burst")) m = 1;
        else if (equals(name, nl, "count_per_period")) m = 2;
        else if (equals(name, nl, "period")) m = 3;
        else if (equals(name, nl, "quantity")) m = 4;
        else return 2;                                  // an unknown member: serde ignores it, the general path
        if (seen >> m & 1) return 2;                    // a duplicate member: serde's error
        seen |= 1u << m;
        skip_ws(c);
        if (c.p >= c.end) return 1;
        if (*c.p != ':') return 2;
        c.p++;
        skip_ws(c);
        if (m == 0) {
            uint32_t kl;
            if ((rc = read_plain_string(c, fr.key, kl))) return rc;
            if (!gcra_resp::valid_utf8(fr.key, kl)) return 2;
            fr.klen = kl;
        } else if (m == 4 && c.p < c.end && *c.p == 'n') {
            for (int i = 0; i < 4; i++, c.p++) {
                if (c.p >= c.end) return 1;
                if (*c.p != (unsigned char)"null"[i]) return 2;
            }
            fr.a[3] = 1;
        } else if ((rc = read_json_int(c, fr.a[m - 1]))) {
            return rc;
        }
        skip_ws(c);
        if (c.p >= c.end) return 1;
        if (*c.p == ',') { c.p++; continue; }
        if (*c.p != '}') return 2;
        c.p++;
        break;
    }
    if ((seen & 15) != 15) return 2;                    // a missing member: serde's error
    skip_ws(c);
    return c.p < c.end ? 2 : 0;
}

// ---- head -------------------------------------------------------------------------------------------------------
// The request at c.p (c.p < c.end): 0 a plain request (c.p moves past its body, `fr` is filled), 1 it is incomplete
// (read more), 2 it is anything else (the general path).  A request is consumed completely or not at all.
GCRA_HTTP_HD int parse_frame(Cursor &c, Frame &fr) {
    const unsigned char *p = c.p;
    const char *line = "POST /throttle HTTP/1.1\r\n";
    for (int i = 0; line[i]; i++, p++) {
        if (p >= c.end) return 1;
        if (*p != (unsigned char)line[i]) return 2;
    }
    uint32_t headers = 0, clen = 0;
    bool has_len = false, has_type = false;
    for (;;) {
        if (p >= c.end) return 1;
        if (*p == '\r') {                               // the empty line
            if (p + 1 >= c.end) return 1;
            if (p[1] != '\n') return 2;
            p += 2;
            break;
        }
        if (headers == MAX_HEADERS) return 2;
        const unsigned char *name = p;
        while (p < c.end && *p != ':') {
            if (!is_tchar(*p)) return 2;                // obs-fold, a line without a colon, bare LF, ...
            p++;
        }
        if (p >= c.end) return 1;
        const uint32_t nl = (uint32_t)(p - name);
        if (nl == 0) return 2;
        p++;
        const unsigned char *v = p;
        while (p < c.end && *p != '\r') {
            if (!is_vbyte(*p)) return 2;
            p++;
        }
        if (p + 1 >= c.end) return 1;
        if (p[1] != '\n') return 2;
        const unsigned char *ve = p;
        p += 2;
        while (v < ve && (*v == ' ' || *v == '\t')) v++;
        while (ve > v && (ve[-1] == ' ' || ve[-1] == '\t')) ve--;
        const uint32_t vl = (uint32_t)(ve - v);
        headers++;
        if (iequals(name, nl, "content-length")) {
            if (has_len || vl == 0 || vl > 5) return 2;
            uint32_t n = 0;
            for (uint32_t i = 0; i < vl; i++) {
                if (v[i] < '0' || v[i] > '9') return 2;
                n = n * 10 + (v[i] - '0');
            }
            if (n > MAX_BODY) return 2;
            clen = n;
            has_len = true;
        } else if (iequals(name, nl, "content-type")) {
            if (has_type || !iequals(v, vl, "application/json")) return 2;
            has_type = true;
        } else if (iequals(name, nl, "transfer-encoding") || iequals(name, nl, "connection") ||
                   iequals(name, nl, "expect") || iequals(name, nl, "upgrade")) {
            return 2;
        }
    }
    if (!has_len || !has_type) return 2;
    const bool whole = (uint64_t)(c.end - p) >= clen;
    Cursor b = {p, whole ? p + clen : c.end};
    const int rc = read_body(b, fr);
    if (rc == 1) return whole ? 2 : 1;
    if (rc) return rc;
    if (!whole) return 1;                               // (the rest of the body can only be whitespace: read it)
    c.p = p + clen;
    return 0;
}

// the smallest plain request: the request line, "content-length:56\r\n", "content-type:application/json\r\n", the
// empty line and the 56-byte body {"key":"","max_burst":0,"count_per_period":0,"period":0}
constexpr uint32_t MIN_FRAME_BYTES = 25 + 19 + 31 + 2 + 56;

// ---- responses (transport/http.rs:103-159, types.rs:73-97, hyper's encoder) -------------------------------------
// IMF-fixdate of floor(ns / 1e9) seconds, proleptic Gregorian (days-from-civil inverted, as in Hinnant's algorithm)
template <class Out>
GCRA_HTTP_HD void put_date(Out &o, int64_t ns) {
    int64_t s = ns / 1000000000LL;
    if (ns % 1000000000LL < 0) s--;
    int64_t days = s / 86400, sod = s % 86400;
    if (sod < 0) { sod += 86400; days--; }
    const int wday = (int)(((days % 7) + 11) % 7);      // 1970-01-01 was a Thursday (4)
    const int64_t z = days + 719468;
    const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
    const int64_t doe = z - era * 146097;
    const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const int64_t mp = (5 * doy + 2) / 153;
    const int d = (int)(doy - (153 * mp + 2) / 5 + 1);
    const int m = (int)(mp < 10 ? mp + 3 : mp - 9);
    const int64_t y = yoe + era * 400 + (m <= 2);
    const char *wd = "SunMonTueWedThuFriSat";
    const char *mn = "JanFebMarAprMayJunJulAugSepOctNovDec";
    o.put(wd[3 * wday]); o.put(wd[3 * wday + 1]); o.put(wd[3 * wday + 2]);
    o.put(','); o.put(' ');
    o.put((char)('0' + d / 10)); o.put((char)('0' + d % 10));
    o.put(' ');
    o.put(mn[3 * (m - 1)]); o.put(mn[3 * (m - 1) + 1]); o.put(mn[3 * (m - 1) + 2]);
    o.put(' ');
    o.put((char)('0' + y / 1000)); o.put((char)('0' + y / 100 % 10)); o.put((char)('0' + y / 10 % 10));
    o.put((char)('0' + y % 10));
    o.put(' ');
    const int hh = (int)(sod / 3600), mm = (int)(sod / 60 % 60), ss = (int)(sod % 60);
    o.put((char)('0' + hh / 10)); o.put((char)('0' + hh % 10)); o.put(':');
    o.put((char)('0' + mm / 10)); o.put((char)('0' + mm % 10)); o.put(':');
    o.put((char)('0' + ss / 10)); o.put((char)('0' + ss % 10));
    gcra_resp::put_str(o, " GMT");
}

// the JSON body: ThrottleResponse as serde_json writes it, or axum's 500 text
template <class Out>
GCRA_HTTP_HD void put_body(Out &o, const gcra_request &q, const gcra_result &r) {
    using gcra_resp::put_i64;
    using gcra_resp::put_str;
    if (r.status == GCRA_OK) {
        put_str(o, r.allowed ? "{\"allowed\":true" : "{\"allowed\":false");
        put_str(o, ",\"limit\":"); put_i64(o, q.max_burst);
        put_str(o, ",\"remaining\":"); put_i64(o, r.remaining);
        put_str(o, ",\"reset_after\":"); put_i64(o, r.reset_after_ns / 1000000000LL);   // types.rs as_secs()
        put_str(o, ",\"retry_after\":"); put_i64(o, r.retry_after_ns / 1000000000LL);
        o.put('}');
    } else {
        put_str(o, "{\"error\":\"Internal server error: ");
        gcra_resp::put_check_failed(o, q, r);
        put_str(o, "\"}");
    }
}

// the response to one decided request: status line, content-type, content-length, date, the empty line, the body.
// At most REPLY_MAX bytes.
template <class Out>
GCRA_HTTP_HD void put_reply(Out &o, const gcra_request &q, const gcra_result &r) {
    using gcra_resp::put_str;
    Count body;
    put_body(body, q, r);
    put_str(o, r.status == GCRA_OK ? "HTTP/1.1 200 OK\r\n" : "HTTP/1.1 500 Internal Server Error\r\n");
    put_str(o, "content-type: application/json\r\ncontent-length: ");
    gcra_resp::put_i64(o, (int64_t)body.n);
    put_str(o, "\r\ndate: ");
    put_date(o, q.now_ns);
    put_str(o, "\r\n\r\n");
    put_body(o, q, r);
}
constexpr uint32_t REPLY_MAX = 256;

#undef GCRA_HTTP_HD
}  // namespace gcra_http
