// gcra_resp.cuh -- the grammar of a plain THROTTLE frame and the text of its reply, ONE definition for the host
// (gcra_resp_parse_throttle, gcra_resp_format_replies in gcra_resp.inc) and the RESP ring's kernels
// (gcra_resp_kernels.cuh).
//
// The fast path only accepts the plain shape
//     *5|*6 CRLF $8 CRLF THROTTLE CRLF $<n> CRLF <key, n bytes> CRLF ($<m> CRLF <decimal> CRLF) x 3|4
// (command name in any case; bulk-string arguments; UTF-8 key; optional sign; i64 range).  Everything else -- another
// command, RESP integers as arguments, a malformed or oversized frame -- is reported as "not plain" and left to the
// general parser (throttlecrab_b200/resp.py, a mirror of resp.rs with its limits and error strings).
#pragma once
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#include "../../include/gcra_b200.h"

namespace gcra_resp {

#define GCRA_RESP_HD __host__ __device__ __forceinline__

struct Cursor {
    const unsigned char *p, *end;
};

// "<digits>\r\n" with optional sign -> value; 0 ok, 1 need more data, 2 not a plain integer line
GCRA_RESP_HD int read_int_line(Cursor &c, int64_t &out, bool allow_sign) {
    const unsigned char *p = c.p;
    if (p >= c.end) return 1;
    bool neg = false;
    if (allow_sign && (*p == '-' || *p == '+')) { neg = *p == '-'; p++; }
    uint64_t v = 0;
    int digits = 0;
    while (p < c.end && *p >= '0' && *p <= '9') {
        if (digits >= 19) return 2;                     // may not fit an i64: the general parser decides
        v = v * 10 + (uint64_t)(*p - '0');
        p++; digits++;
    }
    if (p >= c.end) return 1;
    if (digits == 0 || *p != '\r') return 2;
    if (p + 1 >= c.end) return 1;
    if (p[1] != '\n') return 2;
    if (v > (uint64_t)INT64_MAX) return 2;
    out = neg ? -(int64_t)v : (int64_t)v;
    c.p = p + 2;
    return 0;
}

// "$<n>\r\n<n bytes>\r\n" -> span; same return codes
GCRA_RESP_HD int read_bulk(Cursor &c, const unsigned char *&s, uint64_t &n) {
    if (c.p >= c.end) return 1;
    if (*c.p != '$') return 2;
    Cursor t = {c.p + 1, c.end};
    int64_t len;
    int rc = read_int_line(t, len, false);
    if (rc) return rc;
    if (len > 512 * 1024 * 1024) return 2;             // MAX_BULK_STRING_SIZE (resp.rs:8): the general parser's error
    if ((uint64_t)(t.end - t.p) < (uint64_t)len + 2) return 1;
    if (t.p[len] != '\r' || t.p[len + 1] != '\n') return 2;
    s = t.p;
    n = (uint64_t)len;
    c.p = t.p + len + 2;
    return 0;
}

GCRA_RESP_HD int bulk_to_i64(const unsigned char *s, uint64_t n, int64_t &out) {
    if (n == 0 || n > 20) return 2;
    unsigned char tmp[24];
    memcpy(tmp, s, n);
    tmp[n] = '\r'; tmp[n + 1] = '\n';
    Cursor t = {tmp, tmp + n + 2};
    return read_int_line(t, out, true) == 0 && t.p == tmp + n + 2 ? 0 : 2;
}

// well-formed UTF-8 as str::from_utf8 defines it (resp.rs:110 turns every bulk string into a String and fails the
// frame otherwise): no overlong forms, no surrogates, nothing above U+10FFFF
GCRA_RESP_HD bool valid_utf8(const unsigned char *s, uint64_t n) {
    uint64_t i = 0;
    while (i < n) {
        const unsigned char c = s[i];
        if (c < 0x80) { i++; continue; }
        int more;
        unsigned char lo = 0x80, hi = 0xBF;             // allowed range of the first continuation byte
        if (c >= 0xC2 && c <= 0xDF) more = 1;
        else if (c == 0xE0) { more = 2; lo = 0xA0; }
        else if (c == 0xED) { more = 2; hi = 0x9F; }
        else if (c >= 0xE1 && c <= 0xEF) more = 2;
        else if (c == 0xF0) { more = 3; lo = 0x90; }
        else if (c == 0xF4) { more = 3; hi = 0x8F; }
        else if (c >= 0xF1 && c <= 0xF3) more = 3;
        else return false;
        if (n - i <= (uint64_t)more) return false;
        if (s[i + 1] < lo || s[i + 1] > hi) return false;
        for (int k = 2; k <= more; k++)
            if ((s[i + k] & 0xC0) != 0x80) return false;
        i += (uint64_t)more + 1;
    }
    return true;
}

// The command name in any case.  This is what toupper from <cctype> did before: the library never calls setlocale,
// so it runs in the C locale, where toupper maps exactly a-z to A-Z and leaves every other byte as it is.
GCRA_RESP_HD bool is_throttle_name(const unsigned char *s) {
    bool eq = true;
    for (int i = 0; i < 8; i++) {
        const unsigned char c = s[i] >= 'a' && s[i] <= 'z' ? (unsigned char)(s[i] - 'a' + 'A') : s[i];
        eq &= c == (unsigned char)"THROTTLE"[i];
    }
    return eq;
}

// a plain THROTTLE frame: its key bytes and max_burst, count_per_period, period, quantity
struct Frame {
    const unsigned char *key;
    uint64_t klen;
    int64_t a[4];
};

// the request row of a plain frame whose key hashes to key_hash (or is the reference key_hash)
GCRA_RESP_HD gcra_request request_row(const Frame &fr, uint64_t key_hash, int64_t now_ns) {
    gcra_request r;
    r.key_hash = key_hash;
    r.max_burst = fr.a[0];
    r.count_per_period = fr.a[1];
    r.period = fr.a[2];
    r.quantity = fr.a[3];
    r.now_ns = now_ns;
    return r;
}

// The frame at c.p (c.p < c.end): 0 a plain THROTTLE frame (c.p moves past it, `fr` is filled), 1 it is incomplete
// (read more), 2 it is anything else (the general parser).  A frame is consumed completely or not at all.
GCRA_RESP_HD int parse_frame(Cursor &c, Frame &fr) {
    Cursor f = c;
    int rc;
    if (*f.p != '*') return 2;
    f.p++;
    int64_t arity;
    if ((rc = read_int_line(f, arity, false))) return rc;
    if (arity != 5 && arity != 6) return 2;
    const unsigned char *s;
    uint64_t sl;
    if ((rc = read_bulk(f, s, sl))) return rc;
    if (sl != 8 || !is_throttle_name(s)) return 2;
    if ((rc = read_bulk(f, fr.key, fr.klen))) return rc;
    if (!valid_utf8(fr.key, fr.klen)) return 2;         // the general parser produces resp.rs's error
    fr.a[0] = fr.a[1] = fr.a[2] = 0;
    fr.a[3] = 1;                                        // quantity defaults to 1 (mod.rs:261-266)
    for (int i = 0; i < (int)arity - 2; i++) {
        if ((rc = read_bulk(f, s, sl))) return rc;
        if (bulk_to_i64(s, sl, fr.a[i])) return 2;
    }
    c = f;
    return 0;
}

// the smallest plain THROTTLE frame: "*5\r\n" "$8\r\nTHROTTLE\r\n" "$0\r\n\r\n" and three of "$1\r\n5\r\n"
constexpr uint32_t MIN_FRAME_BYTES = 4 + 14 + 6 + 3 * 7;

// ---- replies (mod.rs:274-285, types.rs:87-97) written through a byte sink: Count measures, Write writes ----
struct Count {
    uint32_t n = 0;
    GCRA_RESP_HD void put(char) { n++; }
};
struct Write {
    char *p;
    GCRA_RESP_HD void put(char c) { *p++ = c; }
};

template <class Out>
GCRA_RESP_HD void put_str(Out &o, const char *s) {
    while (*s) o.put(*s++);
}

// decimal, most significant digit first (no digit buffer: on the device that would live in local memory)
template <class Out>
GCRA_RESP_HD void put_i64(Out &o, int64_t v) {
    const uint64_t u = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    if (v < 0) o.put('-');
    uint64_t p = 1;
    while (u / p >= 10) p *= 10;
    for (; p; p /= 10) o.put((char)('0' + u / p % 10));
}

// the actor's error for a row that was not decided: "Rate limit check failed: {CellError}" (actor.rs:252,
// core/mod.rs:58-65), which every transport wraps in its own way.  (Literals, so that each reply below is written
// from one string.)
#define GCRA_CHECK_FAILED_NEGATIVE "Rate limit check failed: negative quantity: "
#define GCRA_CHECK_FAILED_INVALID "Rate limit check failed: invalid rate limit parameters"
#define GCRA_CHECK_FAILED_INTERNAL "Rate limit check failed: internal error"

template <class Out>
GCRA_RESP_HD void put_check_failed(Out &o, const gcra_request &q, const gcra_result &r) {
    if (r.status == GCRA_NEGATIVE_QUANTITY) {
        put_str(o, GCRA_CHECK_FAILED_NEGATIVE);
        put_i64(o, q.quantity);
    } else if (r.status == GCRA_INVALID_RATE_LIMIT) {
        put_str(o, GCRA_CHECK_FAILED_INVALID);
    } else {
        put_str(o, GCRA_CHECK_FAILED_INTERNAL);
    }
}

// the reply to one decided THROTTLE command: *5 :allowed :limit :remaining :reset_after_s :retry_after_s, or the
// reference's error line.  At most REPLY_MAX bytes.
template <class Out>
GCRA_RESP_HD void put_reply(Out &o, const gcra_request &q, const gcra_result &r) {
    if (r.status == GCRA_OK) {
        put_str(o, "*5\r\n:");
        o.put(r.allowed ? '1' : '0');
        put_str(o, "\r\n:"); put_i64(o, q.max_burst);
        put_str(o, "\r\n:"); put_i64(o, r.remaining);
        put_str(o, "\r\n:"); put_i64(o, r.reset_after_ns / 1000000000LL);      // types.rs:93 as_secs()
        put_str(o, "\r\n:"); put_i64(o, r.retry_after_ns / 1000000000LL);
        put_str(o, "\r\n");
    } else if (r.status == GCRA_NEGATIVE_QUANTITY) {
        put_str(o, "-ERR " GCRA_CHECK_FAILED_NEGATIVE);
        put_i64(o, q.quantity);
        put_str(o, "\r\n");
    } else if (r.status == GCRA_INVALID_RATE_LIMIT) {
        put_str(o, "-ERR " GCRA_CHECK_FAILED_INVALID "\r\n");
    } else {
        put_str(o, "-ERR " GCRA_CHECK_FAILED_INTERNAL "\r\n");
    }
}
constexpr uint32_t REPLY_MAX = 160;

#undef GCRA_RESP_HD
}  // namespace gcra_resp
