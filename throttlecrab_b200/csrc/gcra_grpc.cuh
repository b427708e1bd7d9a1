// gcra_grpc.cuh -- the grammar of a plain gRPC Throttle call and the bytes of its response, ONE definition for the
// host (gcra_grpc_parse_throttle, gcra_grpc_format_replies, gcra_grpc_header_class in gcra_resp.inc) and the gRPC
// ring's kernels (gcra_resp_ring.cu).  The cursor, the UTF-8 rule, the byte sinks and the error texts are
// gcra_resp.cuh's.
//
// HTTP/2 keeps state per connection, so the walk takes it as input: the highest stream id used so far, the connection's
// send window, the peer's initial stream window and one class byte per HPACK dynamic-table entry (the host's decoder
// owns the table; nothing here changes it).  A plain call is
//     HEADERS(END_HEADERS, not END_STREAM, not PADDED) on a new odd stream id above last_stream, whose header block
//         holds only indexed fields (static, or dynamic below n_dyn) and literals without indexing / never indexed
//         with an indexed or raw name and a raw value (or any value of a name whose value does not matter), with
//         :method POST, :path /throttlecrab.RateLimiter/Throttle and content-type application/grpc[+proto] exactly
//         once each and pseudo-headers first;
//     DATA on the same stream holding one uncompressed gRPC message (flag 0, length = payload - 5) that prost reads
//         as a ThrottleRequest, with END_STREAM, or followed by an empty DATA(END_STREAM);
//     in between only WINDOW_UPDATE and at most one PING per walk.
// WINDOW_UPDATE and PING frames between calls are taken on their own.  Anything else -- a dynamic-table change
// (literal with incremental indexing, size update), a Huffman string whose bytes decide the class, SETTINGS,
// RST_STREAM, GOAWAY, CONTINUATION, PUSH_PROMISE, PRIORITY, a PING ACK, padding, interleaved streams, a frame above
// 16,384 octets, a window that cannot take the largest response -- is "not plain" (stop 2) and left to the general
// path (throttlecrab_b200/grpc_transport.py).
#pragma once
#include "gcra_resp.cuh"

namespace gcra_grpc {

#define GCRA_GRPC_HD __host__ __device__ __forceinline__

using gcra_resp::Count;
using gcra_resp::Frame;
using gcra_resp::Write;

// ---- header classes --------------------------------------------------------------------------------------------
// The class of a decoded header field (name and value), and the class of a name alone: a name alone is IGNORE,
// SCHEME, AUTHORITY or NOT_PLAIN when its value does not matter, else one of the NAME_* classes.
enum : uint32_t {
    H_IGNORE = 0, H_METHOD_POST = 1, H_PATH = 2, H_SCHEME = 3, H_AUTHORITY = 4, H_CTYPE = 5, H_ENCODING = 6,
    H_NOT_PLAIN = 7, H_NAME_METHOD = 8, H_NAME_PATH = 9, H_NAME_CTYPE = 10, H_NAME_ENCODING = 11, H_NAME_TE = 12,
};

GCRA_GRPC_HD bool equals(const unsigned char *s, uint32_t n, const char *lit) {
    uint32_t i = 0;
    for (; i < n && lit[i]; i++)
        if (s[i] != (unsigned char)lit[i]) return false;
    return i == n && !lit[i];
}

// a lower-case field name (RFC 9113 8.2.1: no upper case; tchar, and ':' only to start a pseudo-header)
GCRA_GRPC_HD uint32_t name_class(const unsigned char *s, uint32_t n) {
    if (n == 0) return H_NOT_PLAIN;
    for (uint32_t i = 0; i < n; i++) {
        const unsigned char c = s[i];
        const bool ok = (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '-' || c == '_' || c == '.' ||
                        c == '!' || c == '#' || c == '$' || c == '%' || c == '&' || c == '\'' || c == '*' ||
                        c == '+' || c == '^' || c == '`' || c == '|' || c == '~' || (c == ':' && i == 0);
        if (!ok) return H_NOT_PLAIN;
    }
    if (s[0] == ':') {
        if (equals(s, n, ":method")) return H_NAME_METHOD;
        if (equals(s, n, ":path")) return H_NAME_PATH;
        if (equals(s, n, ":scheme")) return H_SCHEME;
        if (equals(s, n, ":authority")) return H_AUTHORITY;
        return H_NOT_PLAIN;                                 // :status, :protocol, unknown pseudo-headers
    }
    if (equals(s, n, "content-type")) return H_NAME_CTYPE;
    if (equals(s, n, "grpc-encoding")) return H_NAME_ENCODING;
    if (equals(s, n, "te")) return H_NAME_TE;
    if (equals(s, n, "connection") || equals(s, n, "keep-alive") || equals(s, n, "proxy-connection") ||
        equals(s, n, "transfer-encoding") || equals(s, n, "upgrade") || equals(s, n, "content-length"))
        return H_NOT_PLAIN;
    return H_IGNORE;
}

// the class of a field whose name has class `nc` and whose value is s[0, n)
GCRA_GRPC_HD uint32_t value_class(uint32_t nc, const unsigned char *s, uint32_t n) {
    for (uint32_t i = 0; i < n; i++)
        if ((s[i] < 0x20 && s[i] != '\t') || s[i] == 0x7f) return H_NOT_PLAIN;   // not a field value (h2 refuses it)
    switch (nc) {
    case H_NAME_METHOD: return equals(s, n, "POST") ? H_METHOD_POST : H_NOT_PLAIN;
    case H_NAME_PATH: return equals(s, n, "/throttlecrab.RateLimiter/Throttle") ? H_PATH : H_NOT_PLAIN;
    case H_NAME_CTYPE:
        return equals(s, n, "application/grpc") || equals(s, n, "application/grpc+proto") ? H_CTYPE : H_NOT_PLAIN;
    case H_NAME_ENCODING: return equals(s, n, "identity") ? H_ENCODING : H_NOT_PLAIN;
    case H_NAME_TE: return equals(s, n, "trailers") ? H_IGNORE : H_NOT_PLAIN;
    default: return nc;
    }
}

GCRA_GRPC_HD uint32_t header_class(const unsigned char *name, uint32_t nl, const unsigned char *value, uint32_t vl) {
    return value_class(name_class(name, nl), value, vl);
}

// The RFC 7541 static table's entries 1..61 as class bytes: the entry's class | its name's class << 4
// (tests/test_grpc_cpu.py checks every entry against header_class of the table's strings).
#define GCRA_GRPC_STATIC_CLASSES                                                                                   \
    {0x00, 0x44, 0x87, 0x81, 0x97, 0x97, 0x33, 0x33, 0x77, 0x77, 0x77, 0x77, 0x77, 0x77, 0x77, 0x00, 0x00,       \
     0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x77, 0x00, 0x00, 0xa7, 0x00, 0x00,       \
     0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00,       \
     0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x77, 0x00, 0x00, 0x00, 0x00}
GCRA_GRPC_HD unsigned char static_class(uint32_t i) {
    const unsigned char t[62] = GCRA_GRPC_STATIC_CLASSES;
    return t[i];
}

// ---- HPACK header block ------------------------------------------------------------------------------------------
// an HPACK integer with an N-bit prefix (RFC 7541 5.1), bounded to 2^21 (a longer one is not plain)
GCRA_GRPC_HD bool read_hpack_int(const unsigned char *&p, const unsigned char *end, uint32_t bits, uint32_t &v) {
    if (p >= end) return false;
    const uint32_t mask = (1u << bits) - 1;
    v = *p++ & mask;
    if (v < mask) return true;
    for (uint32_t m = 0; m <= 14; m += 7) {
        if (p >= end) return false;
        const unsigned char b = *p++;
        v += (uint32_t)(b & 0x7f) << m;
        if (!(b & 0x80)) return true;
    }
    return false;
}

// a string literal: its bytes and whether they are Huffman-coded
GCRA_GRPC_HD bool read_hpack_str(const unsigned char *&p, const unsigned char *end, const unsigned char *&s,
                                 uint32_t &n, bool &huff) {
    if (p >= end) return false;
    huff = *p & 0x80;
    if (!read_hpack_int(p, end, 7, n) || n > (uint32_t)(end - p)) return false;
    s = p;
    p += n;
    return true;
}

// A HEADERS block: plain (true) or not.  dyn[k] is the class byte of dynamic index 62 + k, k < n_dyn.
GCRA_GRPC_HD bool header_block_plain(const unsigned char *p, const unsigned char *end, const unsigned char *dyn,
                                     uint32_t n_dyn) {
    uint32_t method = 0, path = 0, ctype = 0, scheme = 0, authority = 0;
    bool regular = false;
    while (p < end) {
        const unsigned char c = *p;
        uint32_t cls;
        if (c & 0x80) {                                     // indexed field
            uint32_t i;
            if (!read_hpack_int(p, end, 7, i) || i == 0) return false;
            if (i <= 61) cls = static_class(i) & 15;
            else if (i - 62 < n_dyn) cls = dyn[i - 62] & 15;
            else return false;
        } else if (c & 0x60) {                              // incremental indexing, or a dynamic table size update
            return false;
        } else {                                            // literal without indexing (0000) or never indexed (0001)
            uint32_t i;
            if (!read_hpack_int(p, end, 4, i)) return false;
            const unsigned char *ns = nullptr, *vs;
            uint32_t nl = 0, vl, nc;
            bool nh, vh;
            if (i == 0) {
                if (!read_hpack_str(p, end, ns, nl, nh) || nh) return false;
                nc = name_class(ns, nl);
            } else if (i <= 61) {
                nc = static_class(i) >> 4;
            } else if (i - 62 < n_dyn) {
                nc = dyn[i - 62] >> 4;
            } else {
                return false;
            }
            if (!read_hpack_str(p, end, vs, vl, vh)) return false;
            // A Huffman value is taken unread only when its name's class does not depend on it.  Its coding is not
            // checked either: a malformed string there (bad padding, EOS) gets its call answered, where the general
            // path would end the connection with COMPRESSION_ERROR.  The header's value is ignored by the server in
            // both cases; decoding it here would cost the walk a Huffman table for a field that carries nothing.
            cls = vh ? (nc >= H_NAME_METHOD ? H_NOT_PLAIN : nc) : value_class(nc, vs, vl);
        }
        switch (cls) {
        case H_METHOD_POST: method++; break;
        case H_PATH: path++; break;
        case H_SCHEME: scheme++; break;
        case H_AUTHORITY: authority++; break;
        case H_CTYPE: ctype++; break;
        case H_IGNORE: case H_ENCODING: break;
        default: return false;
        }
        const bool pseudo = cls >= H_METHOD_POST && cls <= H_AUTHORITY;
        if (pseudo && regular) return false;
        regular |= !pseudo;
    }
    return method == 1 && path == 1 && ctype == 1 && scheme <= 1 && authority <= 1;
}

// ---- the ThrottleRequest message, as prost decodes it ---------------------------------------------------------
// a varint of at most 10 bytes whose 10th byte is 0 or 1 (prost's decode_varint)
GCRA_GRPC_HD bool read_varint(const unsigned char *&p, const unsigned char *end, uint64_t &v) {
    v = 0;
    for (uint32_t k = 0; k < 10; k++) {
        if (p >= end) return false;
        const unsigned char b = *p++;
        if (k == 9 && b > 1) return false;
        v |= (uint64_t)(b & 0x7f) << (7 * k);
        if (!(b & 0x80)) return true;
    }
    return false;
}

// fields 1..5 (key, max_burst, count_per_period, period, quantity) into fr: an absent field is 0 (an empty key),
// int32 is the varint's low 32 bits, the last of duplicates wins; unknown fields of wire types 0, 1, 2 and 5 are
// skipped.  Groups and everything prost refuses are not plain.
GCRA_GRPC_HD bool decode_message(const unsigned char *p, const unsigned char *end, Frame &fr) {
    fr.key = p;
    fr.klen = 0;
    fr.a[0] = fr.a[1] = fr.a[2] = fr.a[3] = 0;
    while (p < end) {
        uint64_t key, v;
        if (!read_varint(p, end, key) || key > 0xffffffffULL) return false;
        const uint32_t wt = (uint32_t)key & 7, tag = (uint32_t)(key >> 3);
        if (tag == 0) return false;
        if (tag == 1) {
            if (wt != 2 || !read_varint(p, end, v) || v > (uint64_t)(end - p)) return false;
            if (!gcra_resp::valid_utf8(p, v)) return false;
            fr.key = p;
            fr.klen = v;
            p += v;
        } else if (tag <= 5) {
            if (wt != 0 || !read_varint(p, end, v)) return false;
            fr.a[tag - 2] = (int64_t)(int32_t)(uint32_t)v;
        } else if (wt == 0) {
            if (!read_varint(p, end, v)) return false;
        } else if (wt == 1 || wt == 5) {
            const uint32_t k = wt == 1 ? 8 : 4;
            if ((uint32_t)(end - p) < k) return false;
            p += k;
        } else if (wt == 2) {
            if (!read_varint(p, end, v) || v > (uint64_t)(end - p)) return false;
            p += v;
        } else {
            return false;
        }
    }
    return true;
}

// ---- frames ------------------------------------------------------------------------------------------------------
enum : uint32_t { F_DATA = 0, F_HEADERS = 1, F_PING = 6, F_WINDOW_UPDATE = 8 };
enum : uint32_t { END_STREAM = 0x1, ACK = 0x1, END_HEADERS = 0x4, PADDED = 0x8, PRIORITY = 0x20 };
constexpr uint32_t MAX_FRAME = 16384;                      // SETTINGS_MAX_FRAME_SIZE's initial value
constexpr int64_t MAX_WINDOW = 0x7fffffff;

struct Hdr {
    uint32_t len, type, flags, sid;
};

// the frame header at s[p]: 0 the whole frame is at hand, 1 it is not, 2 its payload is above MAX_FRAME
GCRA_GRPC_HD int read_frame(const unsigned char *s, uint32_t p, uint32_t len, Hdr &h) {
    if (len - p < 9) return 1;
    h.len = (uint32_t)s[p] << 16 | (uint32_t)s[p + 1] << 8 | s[p + 2];
    h.type = s[p + 3];
    h.flags = s[p + 4];
    h.sid = ((uint32_t)s[p + 5] & 0x7f) << 24 | (uint32_t)s[p + 6] << 16 | (uint32_t)s[p + 7] << 8 | s[p + 8];
    if (h.len > MAX_FRAME) return 2;
    return h.len > len - p - 9 ? 1 : 0;
}

// whether the HEADERS frame at s[p] carries a plain header block, and whether the DATA frame at s[p] carries one
// plain message (both stateless beyond the dynamic table's classes: the ring kernel decides them in parallel)
GCRA_GRPC_HD bool headers_plain(const unsigned char *s, uint32_t p, const Hdr &h, const unsigned char *dyn,
                                uint32_t n_dyn) {
    uint32_t skip = h.flags & PRIORITY ? 5 : 0;
    if (h.len < skip) return false;
    return header_block_plain(s + p + 9 + skip, s + p + 9 + h.len, dyn, n_dyn);
}
GCRA_GRPC_HD bool data_plain(const unsigned char *s, uint32_t p, const Hdr &h, Frame &fr) {
    const unsigned char *d = s + p + 9;
    if (h.len < 5 || d[0] != 0) return false;
    const uint32_t m = (uint32_t)d[1] << 24 | (uint32_t)d[2] << 16 | (uint32_t)d[3] << 8 | d[4];
    return m == h.len - 5 && decode_message(d + 5, d + h.len, fr);
}

// the largest response DATA payload: the 5-byte prefix and ThrottleResponse with every field present, the four
// int32 fields negative (1 + 10 bytes each): what a call's windows must hold
constexpr uint32_t RESPONSE_DATA_MAX = 5 + 2 + 4 * 11;

// the connection state a walk starts from (gcra_grpc_conn) and where it ends (gcra_grpc_outcome)
struct State {
    uint32_t last_stream;
    int64_t send_window;
    uint32_t data_octets;
    uint32_t ping;
    unsigned char opaque[8];
};

// A WINDOW_UPDATE or PING frame at s[p] (header h) within the walk, `open` the call's stream (0 between calls) and
// *swin its window: false if it is not plain.
GCRA_GRPC_HD bool control(const unsigned char *s, uint32_t p, const Hdr &h, uint32_t open, int64_t &swin, State &st) {
    const unsigned char *d = s + p + 9;
    if (h.type == F_PING) {
        if (h.len != 8 || h.sid != 0 || (h.flags & ACK) || st.ping) return false;
        st.ping = 1;
        for (int i = 0; i < 8; i++) st.opaque[i] = d[i];
        return true;
    }
    if (h.len != 4) return false;
    const uint32_t inc = ((uint32_t)d[0] & 0x7f) << 24 | (uint32_t)d[1] << 16 | (uint32_t)d[2] << 8 | d[3];
    if (inc == 0) return false;
    // (an update that would pass 2^31 - 1 is not taken: the state handed to the general path stays as it was, and
    // the general path answers it with FLOW_CONTROL_ERROR)
    if (h.sid == 0) {
        if (st.send_window + inc > MAX_WINDOW) return false;
        st.send_window += inc;
        return true;
    }
    if (h.sid == open) {
        if (swin + inc > MAX_WINDOW) return false;
        swin += inc;
        return true;
    }
    return (h.sid & 1) && h.sid <= st.last_stream;          // a closed stream: ignored; an idle one is an error
}

struct Conn {
    uint32_t last_stream;
    int32_t send_window, init_window;
    uint32_t n_dyn;
    const unsigned char *dyn;
};

struct WalkEnd {
    uint32_t consumed, n, stop;
};

// The walk over s[0, len) from connection state `cn`: at most max_calls calls.  Plain(i, p, h) says whether frame i
// (counted from 0 at s[0]), a HEADERS or DATA frame at s[p], is plain as headers_plain / data_plain define it;
// Call(k, data_at) receives call k's message frame (its DATA frame starts at data_at).  Stop: 0 the bytes ended on a
// frame boundary, 1 an incomplete frame or call follows, 2 a frame that is not plain follows, 3 a call follows and
// max_calls were taken.  A call is taken whole or not at all; the WINDOW_UPDATE and PING frames before it are taken
// on their own.  (Plain and Call are host lambdas in gcra_grpc_parse_throttle and device lambdas in the ring kernel.)
#pragma nv_exec_check_disable
template <class Plain, class Call>
GCRA_GRPC_HD WalkEnd walk(const unsigned char *s, uint32_t len, const Conn &cn, uint32_t max_calls, Plain plain,
                          Call call, State &st) {
    st.last_stream = cn.last_stream;
    st.send_window = cn.send_window;
    st.data_octets = 0;
    st.ping = 0;
    uint32_t p = 0, i = 0, n = 0, why = 0;
    while (p < len) {
        Hdr h;
        int rc = read_frame(s, p, len, h);
        if (rc) { why = rc; break; }
        if (h.type == F_WINDOW_UPDATE || h.type == F_PING) {
            int64_t none = 0;
            if (!control(s, p, h, 0, none, st)) { why = 2; break; }
            p += 9 + h.len; i++;
            continue;
        }
        if (h.type != F_HEADERS) { why = 2; break; }
        if (n >= max_calls) { why = 3; break; }
        const uint32_t sid = h.sid;
        if (!(sid & 1) || sid <= st.last_stream || !(h.flags & END_HEADERS) || (h.flags & (END_STREAM | PADDED)) ||
            !plain(i, p, h)) { why = 2; break; }
        State t = st;
        int64_t swin = cn.init_window;
        uint32_t q = p + 9 + h.len, j = i + 1, data_at = 0;
        int crc = 0;
        for (bool msg = false;;) {
            if (q >= len) { crc = 1; break; }
            Hdr g;
            if ((crc = read_frame(s, q, len, g))) break;
            if (g.type == F_WINDOW_UPDATE || g.type == F_PING) {
                if (!control(s, q, g, sid, swin, t)) { crc = 2; break; }
                q += 9 + g.len; j++;
                continue;
            }
            if (g.type != F_DATA || g.sid != sid || (g.flags & PADDED)) { crc = 2; break; }
            if (msg) {                                      // after the message: only an empty DATA(END_STREAM)
                if (g.len != 0 || !(g.flags & END_STREAM)) crc = 2;
                else { q += 9; j++; }
                break;
            }
            if (!plain(j, q, g)) { crc = 2; break; }
            msg = true;
            data_at = q;
            t.data_octets += g.len;
            q += 9 + g.len; j++;
            if (g.flags & END_STREAM) break;
        }
        if (crc) { why = (uint32_t)crc; break; }
        // the responses go out after the walk: the stream's window and what the connection's window holds after
        // this call's updates must take the largest response of every call so far
        if (swin < (int64_t)RESPONSE_DATA_MAX ||
            t.send_window < (int64_t)(n + 1) * RESPONSE_DATA_MAX) { why = 2; break; }
        t.last_stream = sid;
        st = t;
        call(n, data_at);
        n++;
        p = q; i = j;
    }
    return {p, n, why};
}

// the smallest plain call: HEADERS with a 3-byte block (:method POST static, :path and content-type dynamic), then
// DATA(END_STREAM) with the prefix of an empty message
constexpr uint32_t MIN_CALL_BYTES = 9 + 3 + 9 + 5;

// ---- responses (grpc.rs:148-193, tonic's encoder; an encoder without HPACK state) ---------------------------------
template <class Out>
GCRA_GRPC_HD void put_frame_header(Out &o, uint32_t len, uint32_t type, uint32_t flags, uint32_t sid) {
    o.put((char)(len >> 16)); o.put((char)(len >> 8)); o.put((char)len);
    o.put((char)type); o.put((char)flags);
    o.put((char)(sid >> 24)); o.put((char)(sid >> 16)); o.put((char)(sid >> 8)); o.put((char)sid);
}

template <class Out>
GCRA_GRPC_HD void put_varint(Out &o, uint64_t v) {
    while (v >= 0x80) { o.put((char)(v | 0x80)); v >>= 7; }
    o.put((char)v);
}

// an int32 field as prost writes it: omitted when 0, negative values as 10-byte varints
template <class Out>
GCRA_GRPC_HD void put_i32_field(Out &o, uint32_t tag, int64_t v) {
    const int32_t x = (int32_t)(uint32_t)(uint64_t)v;
    if (x == 0) return;
    o.put((char)(tag << 3));
    put_varint(o, (uint64_t)(int64_t)x);
}

// ThrottleResponse { allowed = 1, limit = 2, remaining = 3, retry_after = 4, reset_after = 5 }, each `as i32`
template <class Out>
GCRA_GRPC_HD void put_message(Out &o, const gcra_request &q, const gcra_result &r) {
    if (r.allowed) { o.put(0x08); o.put(0x01); }
    put_i32_field(o, 2, q.max_burst);
    put_i32_field(o, 3, r.remaining);
    put_i32_field(o, 4, r.retry_after_ns / 1000000000LL);  // types.rs as_secs()
    put_i32_field(o, 5, r.reset_after_ns / 1000000000LL);
}

// an HPACK string literal without Huffman coding
template <class Out>
GCRA_GRPC_HD void put_hpack_len(Out &o, uint32_t n) {
    if (n < 127) { o.put((char)n); return; }
    o.put(127);
    n -= 127;
    while (n >= 128) { o.put((char)(n | 0x80)); n >>= 7; }
    o.put((char)n);
}

// a byte that grpc-message carries percent-encoded: the gRPC spec's rule (outside 0x20..0x7E, and '%'), plus the
// characters tonic also encodes (space " # < > ` ? { })
GCRA_GRPC_HD bool pct(unsigned char c) {
    return c < 0x20 || c > 0x7e || c == '%' || c == ' ' || c == '"' || c == '#' || c == '<' || c == '>' ||
           c == '`' || c == '?' || c == '{' || c == '}';
}

template <class Out>
struct PctOut {                                            // a sink that percent-encodes into another
    Out &o;
    GCRA_GRPC_HD void put(char ch) {
        const unsigned char c = (unsigned char)ch;
        if (!pct(c)) { o.put(ch); return; }
        o.put('%'); o.put("0123456789ABCDEF"[c >> 4]); o.put("0123456789ABCDEF"[c & 15]);
    }
};

// "Rate limiter error: " + the actor's error (grpc.rs:179), percent-encoded
template <class Out>
GCRA_GRPC_HD void put_grpc_message(Out &o, const gcra_request &q, const gcra_result &r) {
    PctOut<Out> e{o};
    gcra_resp::put_str(e, "Rate limiter error: ");
    gcra_resp::put_check_failed(e, q, r);
}

// ":status 200" (static 8) and "content-type: application/grpc" as a literal without indexing (static name 31)
#define GCRA_GRPC_STATUS_CTYPE "\x88\x0f\x10\x10" "application/grpc"
#define GCRA_GRPC_STATUS_CTYPE_LEN 20u

// The response to one decided call on stream `sid`: HEADERS(:status 200, content-type), DATA(the message) and
// trailers HEADERS(END_STREAM, grpc-status: 0); or, for a decide error, one trailers-only HEADERS(END_STREAM) with
// grpc-status: 13 and grpc-message.  At most REPLY_MAX bytes.
template <class Out>
GCRA_GRPC_HD void put_reply(Out &o, const gcra_request &q, const gcra_result &r, uint32_t sid) {
    using gcra_resp::put_str;
    if (r.status == GCRA_OK) {
        Count m;
        put_message(m, q, r);
        put_frame_header(o, GCRA_GRPC_STATUS_CTYPE_LEN, F_HEADERS, END_HEADERS, sid);
        put_str(o, GCRA_GRPC_STATUS_CTYPE);
        put_frame_header(o, 5 + m.n, F_DATA, 0, sid);
        o.put(0); o.put(0); o.put(0); o.put(0); o.put((char)m.n);
        put_message(o, q, r);
        put_frame_header(o, 15, F_HEADERS, END_STREAM | END_HEADERS, sid);
        o.put(0); o.put(11); put_str(o, "grpc-status"); o.put(1); o.put('0');
    } else {
        Count t;
        put_grpc_message(t, q, r);
        Count l;
        put_hpack_len(l, t.n);
        put_frame_header(o, GCRA_GRPC_STATUS_CTYPE_LEN + 16 + 14 + l.n + t.n, F_HEADERS, END_STREAM | END_HEADERS, sid);
        put_str(o, GCRA_GRPC_STATUS_CTYPE);
        o.put(0); o.put(11); put_str(o, "grpc-status"); o.put(2); put_str(o, "13");
        o.put(0); o.put(12); put_str(o, "grpc-message"); put_hpack_len(o, t.n);
        put_grpc_message(o, q, r);
    }
}
constexpr uint32_t REPLY_MAX = 168;

// the octets of a reply's DATA payload (what it takes of the send windows)
GCRA_GRPC_HD uint32_t data_len(const gcra_request &q, const gcra_result &r) {
    if (r.status != GCRA_OK) return 0;
    Count m;
    put_message(m, q, r);
    return 5 + m.n;
}

#undef GCRA_GRPC_HD
}  // namespace gcra_grpc
