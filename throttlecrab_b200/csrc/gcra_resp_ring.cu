// gcra_resp_ring.cu -- the rings' kernels (gcra_resp_ring_*): connections' read buffers -> request rows, and results
// -> reply bytes.  The frame grammar and the reply text are the host parser's own: gcra_resp.cuh for RESP,
// gcra_http.cuh for HTTP, gcra_grpc.cuh for gRPC.  A translation unit of its own: the parse kernel's dynamic shared
// memory would pad every kernel's static shared memory in gcra_b200.cu to 16 bytes.  gcra_b200.cu launches these
// kernels through the functions at the end.
//
//   ring_parse_kernel<K>    one CTA per connection: rows of the connection's plain prefix, exactly what its
//                           protocol's host walk (gcra_resp_parse_throttle, gcra_http_parse_throttle,
//                           gcra_grpc_parse_throttle) writes for it at the row cap that connections before it leave
//   ring_reply_kernel<K>    one thread per row: the reply bytes, packed in row order
//   ring_outcome_kernel<K>  one warp per connection: where its replies lie (and a gRPC connection's DATA octets)
// Every ring kind -- RespTraits, HttpTraits, GrpcTraits, MixedTraits -- is an instantiation of these three templates.
// A mixed ring takes connections of all three protocols in one slot: its parse kernel picks each connection's parse
// body, its reply kernel each row's reply writer.  ring_metrics_kernel counts a finished slot's rows per transport and
// names its denied keys (gcra_ring_metrics).
#include "gcra_resp_ring.cuh"

namespace gcra {

// A ring kind: its protocol, and the parse kernel's CTAs per SM (its min-blocks bound).  Everything else the kernels
// take of a kind follows from the protocol: the reply tile and bound (reply_tile_rows, reply_max), each connection's
// parse body (ring_conn: constant but for a mixed ring), each row's reply writer (put_reply: constant but for a mixed
// ring), and whether the outcome kernel sums DATA octets (where gRPC rows can occur).  RESP and HTTP also carry the
// grammar of their parse body: where a frame may start (`candidate`: every position the parse kernel parses
// speculatively; `chain_start`: whether the frame that follows the previous one can start here) and the frame's parse.
struct RespTraits {
    // (3 CTAs per SM: the key_ref store would take the parse kernel from 80 to 84 registers, and 2 CTAs per SM, for
    // short connections; bounded, it fits 80 with no spills)
    static constexpr RingProto PROTO = PROTO_RESP;
    static constexpr u32 PARSE_CTAS = 3;
    __device__ static bool candidate(const unsigned char *s, u32 p, u32) { return s[p] == '*' && (p == 0 || s[p - 1] == '\n'); }
    // (a frame ends with "\r\n", so the next one starts at a candidate exactly when its first byte is '*')
    __device__ static bool chain_start(const unsigned char *s, u32 p, u32) { return s[p] == '*'; }
    __device__ static int parse(gcra_resp::Cursor &c, gcra_resp::Frame &f) { return gcra_resp::parse_frame(c, f); }
};

struct HttpTraits {
    static constexpr RingProto PROTO = PROTO_HTTP;
    static constexpr u32 PARSE_CTAS = 3;
    // "POST ", or the part of it that fits before the segment's end (a body ends in '}' or whitespace, so there is no
    // line-start rule as for RESP)
    __device__ static bool candidate(const unsigned char *s, u32 p, u32 len) {
        const char *w = "POST ";
        for (u32 i = 0; i < 5 && p + i < len; i++)
            if (s[p + i] != (unsigned char)w[i]) return false;
        return true;
    }
    __device__ static bool chain_start(const unsigned char *s, u32 p, u32 len) { return candidate(s, p, len); }
    __device__ static int parse(gcra_resp::Cursor &c, gcra_resp::Frame &f) { return gcra_http::parse_frame(c, f); }
};

struct GrpcTraits {
    static constexpr RingProto PROTO = PROTO_GRPC;
    static constexpr u32 PARSE_CTAS = 1;
};

// (3 CTAs per SM: the RESP parse kernel's, so that short connections keep its occupancy)
struct MixedTraits {
    static constexpr RingProto PROTO = PROTO_MIXED;
    static constexpr u32 PARSE_CTAS = 3;
};

constexpr u32 RESP_KIND_SHIFT = 17;            // a candidate's word: frame end (0 .. 65536) | kind << 17
constexpr u64 RESP_AGG = 1ULL << 62, RESP_INC = 1ULL << 63, RESP_VAL = RESP_AGG - 1;   // look-back status words

__device__ __forceinline__ u64 ld_volatile_u64(const u64 *p) {
    u64 v;
    asm volatile("ld.volatile.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile_u64(u64 *p, u64 v) {
    asm volatile("st.volatile.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// exclusive scan of one value per thread over a CTA of THREADS threads; *sum receives the total
template <u32 THREADS>
__device__ __forceinline__ u64 resp_block_scan(u64 v, u64 *warp_sums, u64 *sum) {
    const u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    u64 inc = v;
#pragma unroll
    for (u32 o = 1; o < 32; o <<= 1) {
        const u64 y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) warp_sums[w] = inc;
    __syncthreads();
    u64 before = 0, all = 0;
    for (u32 i = 0; i < THREADS / 32; i++) {
        if (i < w) before += warp_sums[i];
        all += warp_sums[i];
    }
    *sum = all;
    __syncthreads();                               // warp_sums may be reused
    return before + inc - v;
}

// Decoupled look-back: publish this item's `value`, then add those of the items before it, taken by ticket, until
// one that has published its inclusive prefix; publish this item's.  Returns the exclusive prefix.  Every earlier
// item was handed to a CTA that runs already, so the wait ends.  (One thread.)
__device__ __forceinline__ u64 resp_look_back(u64 *status, u32 item, u64 value) {
    if (item == 0) { st_volatile_u64(&status[0], RESP_INC | value); return 0; }
    st_volatile_u64(&status[item], RESP_AGG | value);
    u64 excl = 0;
    for (u32 j = item - 1;; j--) {
        u64 st;
        do { st = ld_volatile_u64(&status[j]); } while (!(st & (RESP_AGG | RESP_INC)));
        excl += st & RESP_VAL;
        if (st & RESP_INC) break;
    }
    st_volatile_u64(&status[item], RESP_INC | (excl + value));
    return excl;
}

__device__ __forceinline__ u32 resp_rank(const u32 *bits, const u32 *before, u32 p) {
    return before[p >> 5] + __popc(bits[p >> 5] & ((1u << (p & 31)) - 1));
}

// ---- the parse bodies: connection c = in[off, + len), taken by ticket, so in table order ----
// Its rows go to rows[base_c ...], base_c = the rows of the connections before it, whatever their protocols; at most
// row_cap rows in all, cut exactly where its protocol's host walk with max_frames = row_cap - base_c stops (stop 3).
// A body writes the connection's end state to its outcome rows, {base_c, n_frames} to
// conn_rows[c]; the CTA of the last connection writes the row count to *total and the segments' row counts of the
// batch view (segment s holds rows [s << cap_shift, (s + 1) << cap_shift)).  status[0 .. n_conns) and *ticket are zero
// at launch.  smem is the dynamic shared memory rounded up to 16 bytes.  A body returns {base_c, the rows taken} to
// every thread.  key_ref (null: not written) receives each row's key as {its offset in `in`, its length}: a plain key
// is raw contiguous bytes (a RESP bulk string, a JSON string without escapes, a protobuf string), which
// ring_metrics_kernel names denied keys from.

// the connection's bytes into smem: 16-byte loads of the chunks wholly inside it, single bytes at its ends (nothing
// outside it); returns where its first byte lands
__device__ __forceinline__ const unsigned char *stage_conn(unsigned char *smem, const unsigned char *in, u32 off, u32 len) {
    const uintptr_t seg = reinterpret_cast<uintptr_t>(in) + off;
    stage_key_span(seg, len, 0, len, threadIdx.x, RESP_THREADS,
                   [&](uintptr_t g, u32 o) { *reinterpret_cast<uint4 *>(smem + o) = __ldg(reinterpret_cast<const uint4 *>(g)); },
                   [&](uintptr_t g, u32 o) { smem[o] = *reinterpret_cast<const unsigned char *>(g); });
    return smem + (seg & 15);
}

// (thread 0) connection c's first row, its walk having found n: the rows of the connections before it, at most row_cap
__device__ __forceinline__ u32 claim_rows(const RingParse &a, u32 c, u32 n) {
    const u64 excl = resp_look_back(a.status, c, n);
    return excl < a.row_cap ? (u32)excl : a.row_cap;
}

// (thread 0) connection c's rows [base, + n): conn_rows[c]; after the last connection's, the batch's row counts
__device__ __forceinline__ void publish_rows(const RingParse &a, u32 c, u32 base, u32 n) {
    a.conn_rows[c] = make_uint2(base, n);
    if (c == a.n_conns - 1) {
        const u32 t = base + n;
        *a.total = t;
        for (u32 s = 0; s < a.nseg; s++) {
            const u32 first = s << a.cap_shift;
            a.seg_counts[s] = t <= first ? 0 : min(t - first, 1u << a.cap_shift);
        }
    }
}

// row i: frame fr of the connection at in[off ...], staged at sb; its key hashed from shared memory with the engine's
// hash
__device__ __forceinline__ void put_row(const RingParse &a, u32 i, const gcra_resp::Frame &fr, const unsigned char *sb,
                                        u32 off) {
    a.rows[i] = gcra_resp::request_row(fr, hash_key_engine(KeyBytes{fr.key}, fr.klen, a.k0, a.k1), a.now_ns);
    if (a.key_ref) a.key_ref[i] = make_uint2(off + (u32)(fr.key - sb), (u32)fr.klen);
}

__device__ __forceinline__ gcra_resp_outcome resp_outcome(u32 consumed, u32 n_frames, int32_t stop) {
    gcra_resp_outcome o;
    o.consumed = consumed;
    o.n_frames = n_frames;
    o.stop = stop;
    o.reserved = 0;
    o.reply_off = 0;
    o.reply_len = 0;
    return o;
}

// RESP and HTTP (grammar P): the dynamic shared memory laid out as RespSmem(max_len, cand_per_word(P::PROTO)).  Every
// candidate frame start is parsed speculatively in parallel; thread 0 chains the true frames from the segment start.
// The end state goes to outcome[c].
template <class P>
__device__ __forceinline__ uint2 resp_parse_conn(unsigned char *smem, const RingParse &a, u32 c, u32 off, u32 len) {
    __shared__ u64 warp_sums[RESP_THREADS / 32];
    __shared__ u32 s_base, s_n;
    const RespSmem L(a.max_len[P::PROTO - 1], cand_per_word(P::PROTO));
    u32 *bits = reinterpret_cast<u32 *>(smem + L.bits_off);
    u32 *before = reinterpret_cast<u32 *>(smem + L.before_off);
    u32 *cand = reinterpret_cast<u32 *>(smem + L.cand_off);

    const unsigned char *sb = stage_conn(smem, a.in, off, len);
    __syncthreads();

    // candidate frame starts: one bit per byte; each thread takes a run of 32-byte words
    const u32 words = (len + 31) / 32, per = (words + RESP_THREADS - 1) / RESP_THREADS;
    const u32 w0 = min(words, threadIdx.x * per), w1 = min(words, w0 + per);
    u32 mine = 0;
    for (u32 w = w0; w < w1; w++) {
        u32 b = 0;
        for (u32 j = 0; j < 32; j++) {
            const u32 p = w * 32 + j;
            if (p < len && P::candidate(sb, p, len)) b |= 1u << j;
        }
        bits[w] = b;
        mine += __popc(b);
    }
    u64 ncand;
    u32 idx = (u32)resp_block_scan<RESP_THREADS>(mine, warp_sums, &ncand);
    for (u32 w = w0; w < w1; w++) {
        before[w] = idx;
        for (u32 b = bits[w]; b; b &= b - 1) cand[idx++] = w * 32 + __ffs(b) - 1;
    }
    __syncthreads();

    // every candidate parsed speculatively: its end, or why it is not a plain frame
    for (u32 i = threadIdx.x; i < (u32)ncand; i += RESP_THREADS) {
        gcra_resp::Cursor cu = {sb + cand[i], sb + len};
        gcra_resp::Frame fr;
        const int rc = P::parse(cu, fr);
        cand[i] = rc ? (u32)rc << RESP_KIND_SHIFT : (u32)(cu.p - sb);
    }
    __syncthreads();

    if (threadIdx.x == 0) {
        // The true frames: the chain from the segment start; a position the protocol cannot start a frame at is a
        // frame that is not plain.  cand[k] becomes the start of the k-th frame (k <= the index read, so nothing still
        // to be read is overwritten).
        u32 n = 0, p = 0, why = 0;
        while (p < len) {
            if (!P::chain_start(sb, p, len)) { why = 2; break; }
            const u32 e = cand[resp_rank(bits, before, p)];
            if (e >> RESP_KIND_SHIFT) { why = e >> RESP_KIND_SHIFT; break; }
            cand[n++] = p;
            p = e;
        }
        // the cap cuts this connection as max_frames = row_cap - base would
        const u32 base = claim_rows(a, c, n), room = a.row_cap - base;
        u32 take = n, stop_at = p;
        if (n > room || (n == room && p < len)) { take = room; why = 3; stop_at = take < n ? cand[take] : p; }
        s_base = base; s_n = take;
        a.outcome[c] = resp_outcome(stop_at, take, (int32_t)why);
        publish_rows(a, c, base, take);
    }
    __syncthreads();

    // the rows: each frame parsed again
    const u32 base = s_base, take = s_n;
    for (u32 k = threadIdx.x; k < take; k += RESP_THREADS) {
        gcra_resp::Cursor cu = {sb + cand[k], sb + len};
        gcra_resp::Frame fr;
        P::parse(cu, fr);
        put_row(a, base + k, fr, sb, off);
    }
    return make_uint2(base, take);
}

// gRPC: the HTTP/2 state gconns[gs] (whose off and len it does not read), the dynamic shared memory laid out as
// GrpcSmem(max_len).  HTTP/2 has no byte that marks a frame start: the starts are the chain of 9-byte headers from
// offset 0.  So thread 0 hops that chain over the staged bytes and lists every whole frame (one shared-memory word per
// frame); then every HEADERS and DATA frame is judged in parallel (gcra_grpc::headers_plain, data_plain: the
// stateless, costly part); then thread 0 runs the host's walk (gcra_grpc::walk) over the list with the connection's
// state, looking the judgements up instead of making them; the rows are decoded and hashed in parallel, their stream
// ids to stream_ids[base_c ...].  The end state goes to the connection's gRPC outcome row goutcome[gs], all but the
// reply fields and data_sent (the outcome kernel's); on a mixed ring (K) its consumed, n_frames and stop also go to
// outcome[c].
template <class K>
__device__ __forceinline__ uint2 grpc_parse_conn(unsigned char *smem, const RingParse &a, u32 c, u32 off, u32 len,
                                                 u32 gs) {
    __shared__ unsigned char s_dyn[GCRA_GRPC_MAX_DYN];
    __shared__ u32 s_nf, s_base, s_n;
    const GrpcSmem L(a.max_len[PROTO_GRPC - 1]);
    u32 *frames = reinterpret_cast<u32 *>(smem + L.frames_off);
    u32 *calls = reinterpret_cast<u32 *>(smem + L.calls_off);

    const gcra_grpc_conn *cn = a.gconns + gs;
    const u32 n_dyn = cn->n_dyn;
    const unsigned char *sb = stage_conn(smem, a.in, off, len);
    for (u32 i = threadIdx.x; i < n_dyn; i += RESP_THREADS) s_dyn[i] = cn->dyn_class[i];
    __syncthreads();

    if (threadIdx.x == 0) {                                    // the hop walk: every whole frame's start
        u32 p = 0, nf = 0;
        while (len - p >= 9) {
            const u32 fl = (u32)sb[p] << 16 | (u32)sb[p + 1] << 8 | sb[p + 2];
            if (fl > len - p - 9) break;
            frames[nf++] = p;
            p += 9 + fl;
        }
        s_nf = nf;
    }
    __syncthreads();
    const u32 nf = s_nf;
    for (u32 i = threadIdx.x; i < nf; i += RESP_THREADS) {   // the judgements: bit 31 of the frame's word
        const u32 p = frames[i];
        gcra_grpc::Hdr h;
        bool ok = false;
        if (!gcra_grpc::read_frame(sb, p, len, h)) {
            gcra_resp::Frame fr;
            if (h.type == gcra_grpc::F_HEADERS) ok = gcra_grpc::headers_plain(sb, p, h, s_dyn, n_dyn);
            else if (h.type == gcra_grpc::F_DATA) ok = gcra_grpc::data_plain(sb, p, h, fr);
        }
        frames[i] = p | (u32)ok << 31;
    }
    __syncthreads();

    if (threadIdx.x == 0) {
        const gcra_grpc::Conn k{cn->last_stream, cn->send_window, cn->init_window, n_dyn, s_dyn};
        auto plain = [&](u32 i, u32, const gcra_grpc::Hdr &) { return (frames[i] >> 31) != 0; };
        auto call = [&](u32 j, u32 at) { calls[j] = at; };
        gcra_grpc::State st;
        gcra_grpc::WalkEnd e = gcra_grpc::walk(sb, len, k, 0xffffffffu, plain, call, st);
        const u32 base = claim_rows(a, c, e.n), room = a.row_cap - base;
        if (e.n >= room) e = gcra_grpc::walk(sb, len, k, room, plain, call, st);   // the cap decides the stop
        s_base = base; s_n = e.n;
        gcra_grpc_outcome o;
        o.consumed = e.consumed;
        o.n_frames = e.n;
        o.stop = (int32_t)e.stop;
        o.data_octets = st.data_octets;
        o.reply_off = 0;
        o.reply_len = 0;
        o.last_stream = st.last_stream;
        o.send_window = (int32_t)st.send_window;
        o.data_sent = 0;
        o.ping = st.ping;
        for (int i = 0; i < 8; i++) o.ping_opaque[i] = st.ping ? st.opaque[i] : 0;
        a.goutcome[gs] = o;
        if (K::PROTO == PROTO_MIXED) a.outcome[c] = resp_outcome(o.consumed, o.n_frames, o.stop);
        publish_rows(a, c, base, e.n);
    }
    __syncthreads();

    const u32 base = s_base, take = s_n;
    for (u32 j = threadIdx.x; j < take; j += RESP_THREADS) {
        const u32 at = calls[j];
        gcra_grpc::Hdr h;
        gcra_grpc::read_frame(sb, at, len, h);
        gcra_resp::Frame fr;
        gcra_grpc::data_plain(sb, at, h, fr);
        put_row(a, base + j, fr, sb, off);
        a.stream_ids[base + j] = h.sid;
    }
    return make_uint2(base, take);
}

// ---- the kernels ----
// The parse kernel: connection c's protocol's body (uniform over the CTA; a compile-time choice but for a mixed ring),
// whose end state goes to outcome[c] (every ring but a gRPC one) and, for a gRPC connection, to its gRPC outcome row.
// A mixed ring's row i also gets its protocol in row_proto[i], for the reply kernel.
template <class K>
__global__ void __launch_bounds__(RESP_THREADS, K::PARSE_CTAS) ring_parse_kernel(const __grid_constant__ RingParse a) {
    // (no alignment is declared for the dynamic shared memory: that would pad every kernel's; RespSmem and GrpcSmem
    // leave room to round its start up to 16 bytes)
    extern __shared__ unsigned char ring_dyn[];
    unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(ring_dyn) + 15) & ~(uintptr_t)15);
    __shared__ u32 s_conn;
    if (threadIdx.x == 0) s_conn = atomicAdd(a.ticket, 1u);
    __syncthreads();
    const u32 c = s_conn;
    const RingConn cn = ring_conn(K::PROTO, a.conns, a.gconns, a.mconns, c);
    uint2 br;
    if (cn.proto == PROTO_GRPC)
        br = grpc_parse_conn<K>(smem, a, c, cn.off, cn.len, cn.grpc_state);
    else if (cn.proto == PROTO_HTTP)
        br = resp_parse_conn<HttpTraits>(smem, a, c, cn.off, cn.len);
    else
        br = resp_parse_conn<RespTraits>(smem, a, c, cn.off, cn.len);
    if (K::PROTO == PROTO_MIXED)
        for (u32 k = threadIdx.x; k < br.y; k += RESP_THREADS) a.row_proto[br.x + k] = (unsigned char)cn.proto;
}

// row i's reply in its protocol: gcra_resp::put_reply, gcra_http::put_reply, or gcra_grpc::put_reply on its stream
template <class Out>
__device__ __forceinline__ void put_reply(Out &o, u32 proto, const gcra_request &q, const gcra_result &r, u32 sid) {
    if (proto == PROTO_GRPC) gcra_grpc::put_reply(o, q, r, sid);
    else if (proto == PROTO_HTTP) gcra_http::put_reply(o, q, r);
    else gcra_resp::put_reply(o, q, r);
}

// The replies of rows [0, *total) in row order, straight into `out` (pinned host memory): each CTA takes a tile of
// rows by ticket, measures its replies, finds the tile's offset by a look-back over the tiles before it, writes the
// replies into shared memory and copies the tile's bytes out in one coalesced sweep.  row_off[i] = the offset of row
// i's reply, row_off[*total] = all the bytes.  status[] and *ticket are zero at launch.  A gRPC row's response goes on
// stream stream_ids[i]; a mixed ring's row i is in protocol row_proto[i] (a connection's rows are contiguous, so most
// warps take one branch).
template <class K>
__global__ void __launch_bounds__(reply_tile_rows(K::PROTO))
ring_reply_kernel(const gcra_request *__restrict__ rows, const gcra_result *__restrict__ res,
                  const u32 *__restrict__ stream_ids, const unsigned char *__restrict__ row_proto, const u32 *total_p,
                  u64 *status, u32 *ticket, u64 *__restrict__ row_off, unsigned char *out) {
    constexpr u32 T = reply_tile_rows(K::PROTO);
    static_assert(T * reply_max(K::PROTO) <= 48 * 1024, "the reply tile fits static shared memory");
    __shared__ __align__(16) char stage[T * reply_max(K::PROTO)];
    __shared__ u64 warp_sums[T / 32];
    __shared__ u64 s_base;
    __shared__ u32 s_tile;
    if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const u32 tile = s_tile, total = *total_p;
    if ((u64)tile * T >= total) return;                        // uniform over the CTA
    const u32 row = tile * T + threadIdx.x;
    gcra_request q{};
    gcra_result r{};
    u32 sid = 0, proto = K::PROTO;
    gcra_resp::Count cnt;
    if (row < total) {
        q = rows[row];
        r = res[row];
        if (K::PROTO == PROTO_MIXED) proto = row_proto[row];
        if (proto == PROTO_GRPC) sid = stream_ids[row];
        put_reply(cnt, proto, q, r, sid);
    }
    u64 tile_bytes;
    const u64 at = resp_block_scan<T>(cnt.n, warp_sums, &tile_bytes);
    if (threadIdx.x == 0) s_base = resp_look_back(status, tile, tile_bytes);
    if (row < total) {
        gcra_resp::Write o{stage + at};
        put_reply(o, proto, q, r, sid);
    }
    __syncthreads();
    const u64 base = s_base;
    if (row < total) row_off[row] = base + at;
    if (row + 1 == total) row_off[total] = base + at + cnt.n;
    for (u32 i = threadIdx.x; i < (u32)tile_bytes; i += T) out[base + i] = stage[i];
}

// one warp per connection: where its replies lie, in outcome[c] (every ring but a gRPC one) and in a gRPC
// connection's gRPC outcome row (on a mixed ring: row mconns[c].grpc_state), with the DATA octets of its responses
template <class K>
__global__ void ring_outcome_kernel(const uint2 *__restrict__ conn_rows, const gcra_mixed_conn *__restrict__ mconns,
                                    u32 n_conns, const gcra_request *__restrict__ rows,
                                    const gcra_result *__restrict__ res, const u32 *total_p,
                                    const u64 *__restrict__ row_off, gcra_resp_outcome *outcome,
                                    gcra_grpc_outcome *goutcome) {
    const u32 c = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x & 31;
    if (c >= n_conns) return;                                  // uniform over the warp
    const u32 total = *total_p;
    u32 proto = K::PROTO, grpc_state = c;
    if (K::PROTO == PROTO_MIXED) {
        const gcra_mixed_conn mc = mconns[c];
        proto = mc.protocol;
        grpc_state = mc.grpc_state;
    }
    const uint2 br = conn_rows[c];
    const u32 lo = min(br.x, total), hi = min(br.x + br.y, total);
    const u64 a = total ? row_off[lo] : 0, b = total ? row_off[hi] : 0;
    u32 sent = 0;
    if (proto == PROTO_GRPC) {                                 // uniform over the warp
        for (u32 i = lo + lane; i < hi; i += 32) sent += gcra_grpc::data_len(rows[i], res[i]);
#pragma unroll
        for (u32 o = 16; o; o >>= 1) sent += __shfl_xor_sync(0xffffffffu, sent, o);
    }
    if (lane) return;
    if (K::PROTO != PROTO_GRPC) {
        outcome[c].reply_off = a;
        outcome[c].reply_len = b - a;
    }
    if (proto == PROTO_GRPC) {
        gcra_grpc_outcome *go = goutcome + grpc_state;
        go->reply_off = a;
        go->reply_len = b - a;
        go->data_sent = sent;
    }
}

// ---- ring metrics: counts per transport and denied keys' names (gcra_ring_metrics) ----
// One thread per row.  A row's class follows the reference's transports: RESP counts an -ERR reply as allowed and
// never an error (redis/mod.rs:193-205); HTTP and gRPC answer status != OK with an error (http.rs:148-151,
// grpc.rs:177-179).  A warp's rows go to the CTA's 9 counters by ballot, the CTA's to HBM in at most 9 atomic adds.
// A denied row finds its key's entry in the denied table, which finish_batch counted this batch into before the reply
// stream went on: the probe of denied_tile_flush (an empty word or 64 probes: the key found the table full).  On a
// name table (gcra_ring_metrics_sharded: the denied count is on the key's owner, maybe another GPU) the row inserts its
// key instead, by a CAS of an empty word, and a key that finds the table full is counted in `full`.  The first row to
// CAS the entry's length word from GCRA_NAME_UNKNOWN copies its key bytes.
constexpr u32 RING_METRICS_THREADS = 256, DENIED_PROBES = 64;

__device__ __forceinline__ u32 name_home(u64 k, u32 mask) { return (u32)(mix64(k ^ 0x9E3779B97F4A7C15ULL)) & mask; }

__device__ __forceinline__ void ring_metrics_name(const RingMetrics &a, u32 i) {
    const NameTableView &t = a.names;
    u64 k = a.rows[i].key_hash;
    if (k == 0) k = 1;                                          // (as denied_tile_add stores it)
    u32 h = name_home(k, t.mask);
    for (u32 probe = 0; probe < DENIED_PROBES; probe++) {
        u64 cur = t.keys[h];
        if (cur == 0) {
            if (!a.full) return;
            cur = atomicCAS(reinterpret_cast<unsigned long long *>(t.keys + h), 0ULL, (unsigned long long)k);
            if (cur == 0) cur = k;                              // (claimed)
        }
        if (cur == k) {
            if (t.name_len[h] != GCRA_NAME_UNKNOWN) return;     // (most denials are of keys named already)
            const uint2 kr = a.key_ref[i];
            const u32 len = kr.y > GCRA_DENIED_NAME_MAX ? GCRA_NAME_TOO_LONG : kr.y;
            if (atomicCAS(&t.name_len[h], GCRA_NAME_UNKNOWN, len) != GCRA_NAME_UNKNOWN || len == GCRA_NAME_TOO_LONG) return;
            unsigned char *dst = t.names + (size_t)h * GCRA_DENIED_NAME_MAX;
            for (u32 b = 0; b < len; b++) dst[b] = a.in[kr.x + b];
            return;
        }
        h = (h + 1) & t.mask;
    }
    if (a.full) atomicAdd(reinterpret_cast<unsigned long long *>(a.full), 1ULL);
}

__global__ void __launch_bounds__(RING_METRICS_THREADS) ring_metrics_kernel(RingMetrics a) {
    __shared__ u32 cnt[9];
    if (threadIdx.x < 9) cnt[threadIdx.x] = 0;
    __syncthreads();
    const u32 i = blockIdx.x * RING_METRICS_THREADS + threadIdx.x, total = *a.total;
    u32 cls = 9;                                                // (no row)
    if (i < total) {
        const u32 proto = a.row_proto ? a.row_proto[i] : a.proto;
        // status | allowed << 32: the second half of the 32-byte result row
        const longlong2 tail = reinterpret_cast<const longlong2 *>(a.res + i)[1];
        const bool ok = (u32)tail.y == GCRA_OK, denied = ok && ((tail.y >> 32) & 0xff) == 0;
        cls = (proto - 1) * 3 + (denied ? 1 : ok || proto == GCRA_PROTO_RESP ? 0 : 2);
        if (denied && a.names.keys) ring_metrics_name(a, i);
    }
#pragma unroll
    for (u32 k = 0; k < 9; k++) {
        const u32 b = __ballot_sync(0xffffffffu, cls == k);
        if ((threadIdx.x & 31) == 0 && b) atomicAdd(&cnt[k], (u32)__popc(b));
    }
    __syncthreads();
    if (threadIdx.x < 9 && cnt[threadIdx.x])
        atomicAdd(reinterpret_cast<unsigned long long *>(a.counts + threadIdx.x), (unsigned long long)cnt[threadIdx.x]);
}

cudaError_t launch_ring_metrics(const RingMetrics &a, u32 max_rows, cudaStream_t st) {
    ring_metrics_kernel<<<(max_rows + RING_METRICS_THREADS - 1) / RING_METRICS_THREADS, RING_METRICS_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}

// ---- a name table's lookup and rebuild (gcra_denied_names, gcra_ring_names_keep on gcra_ring_metrics_sharded) ----
// One warp per hash.  The warp reads 32 probes of ring_metrics_name's sequence at a time; the sequence ends at the
// key's entry or an empty word (entries are never emptied: the table is rebuilt whole), or after 64 probes.
constexpr u32 NAME_WARPS = 8;

// the entry of key k (0 stored as 1) in t, or -1; warp-uniform
__device__ __forceinline__ int warp_find_name(const NameTableView &t, u64 k) {
    const u32 lane = threadIdx.x & 31, home = name_home(k, t.mask);
    for (u32 base = 0; base < DENIED_PROBES; base += 32) {
        const u64 cur = t.keys[(home + base + lane) & t.mask];
        const u32 hit = __ballot_sync(0xffffffffu, cur == k), stop = hit | __ballot_sync(0xffffffffu, cur == 0);
        if (stop) {
            const u32 f = __ffs(stop) - 1;
            return (hit >> f) & 1 ? (int)((home + base + f) & t.mask) : -1;
        }
    }
    return -1;
}

// a name's bytes, GCRA_DENIED_NAME_MAX-aligned rows: 8 bytes per lane (len <= GCRA_DENIED_NAME_MAX)
__device__ __forceinline__ void warp_copy_name(unsigned char *dst, const unsigned char *src, u32 len) {
    static_assert(GCRA_DENIED_NAME_MAX == 32 * 8, "one 8-byte word per lane");
    const u32 lane = threadIdx.x & 31;
    if (lane * 8 < len) reinterpret_cast<u64 *>(dst)[lane] = reinterpret_cast<const u64 *>(src)[lane];
}

__global__ void __launch_bounds__(NAME_WARPS * 32) ring_names_lookup_kernel(NameTableView t, const u64 *hashes, u32 n,
                                                                             u32 *out_len, unsigned char *out_names) {
    const u32 w = blockIdx.x * NAME_WARPS + (threadIdx.x >> 5);
    if (w >= n) return;
    const int e = warp_find_name(t, hashes[w] ? hashes[w] : 1);
    const u32 len = e < 0 ? GCRA_NAME_UNKNOWN : t.name_len[e];
    if ((threadIdx.x & 31) == 0) out_len[w] = len;
    if (len <= GCRA_DENIED_NAME_MAX)
        warp_copy_name(out_names + (size_t)w * GCRA_DENIED_NAME_MAX, t.names + (size_t)e * GCRA_DENIED_NAME_MAX, len);
}

__global__ void __launch_bounds__(NAME_WARPS * 32) ring_names_keep_kernel(NameTableView from, NameTableView to,
                                                                           const u64 *hashes, u32 n, u64 *full) {
    const u32 w = blockIdx.x * NAME_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (w >= n) return;
    const u64 k = hashes[w] ? hashes[w] : 1;
    const int e = warp_find_name(from, k);
    if (e < 0) return;
    int d = -1;                                                 // the entry in `to` (-2: a repeated hash)
    if (lane == 0) {
        u32 s = name_home(k, to.mask);
        for (u32 probe = 0; probe < DENIED_PROBES && d == -1; probe++, s = (s + 1) & to.mask) {
            const u64 cur = atomicCAS(reinterpret_cast<unsigned long long *>(to.keys + s), 0ULL, (unsigned long long)k);
            if (cur == 0) d = (int)s;
            else if (cur == k) d = -2;
        }
        if (d == -1) atomicAdd(reinterpret_cast<unsigned long long *>(full), 1ULL);
    }
    d = __shfl_sync(0xffffffffu, d, 0);
    if (d < 0) return;
    const u32 len = from.name_len[e];
    if (lane == 0) to.name_len[d] = len;
    if (len <= GCRA_DENIED_NAME_MAX)
        warp_copy_name(to.names + (size_t)d * GCRA_DENIED_NAME_MAX, from.names + (size_t)e * GCRA_DENIED_NAME_MAX, len);
}

cudaError_t launch_ring_names_lookup(const NameTableView &t, const u64 *hashes, u32 n, u32 *out_len,
                                     unsigned char *out_names, cudaStream_t st) {
    ring_names_lookup_kernel<<<(n + NAME_WARPS - 1) / NAME_WARPS, NAME_WARPS * 32, 0, st>>>(t, hashes, n, out_len,
                                                                                           out_names);
    return cudaGetLastError();
}

cudaError_t launch_ring_names_keep(const NameTableView &from, const NameTableView &to, const u64 *hashes, u32 n,
                                   u64 *full, cudaStream_t st) {
    ring_names_keep_kernel<<<(n + NAME_WARPS - 1) / NAME_WARPS, NAME_WARPS * 32, 0, st>>>(from, to, hashes, n, full);
    return cudaGetLastError();
}

// ---- launches (gcra_resp.inc) ----
// f(K()) for the ring kind K of `proto`
template <class F>
static cudaError_t for_kind(RingProto proto, F f) {
    switch (proto) {
    case PROTO_RESP: return f(RespTraits());
    case PROTO_HTTP: return f(HttpTraits());
    case PROTO_GRPC: return f(GrpcTraits());
    case PROTO_MIXED: return f(MixedTraits());
    default: return cudaErrorInvalidValue;
    }
}

cudaError_t resp_ring_setup() {
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, ring_metrics_kernel);  // (loads the code now: see preload in gcra_b200.cu)
    for (RingProto p : {PROTO_RESP, PROTO_HTTP, PROTO_GRPC, PROTO_MIXED}) {
        if (!e) e = for_kind(p, [&](auto k) {
            using K = decltype(k);
            for (const void *f : {(const void *)ring_parse_kernel<K>, (const void *)ring_reply_kernel<K>,
                                  (const void *)ring_outcome_kernel<K>}) {
                const cudaError_t r = cudaFuncGetAttributes(&fa, f);
                if (r) return r;
            }
            const u32 max_len[3] = {RESP_MAX_CONN_BYTES, RESP_MAX_CONN_BYTES, RESP_MAX_CONN_BYTES};
            return cudaFuncSetAttribute(ring_parse_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)parse_smem(K::PROTO, max_len));
        });
    }
    return e;
}

cudaError_t launch_ring_parse(RingProto proto, const RingParse &a, cudaStream_t st) {
    return for_kind(proto, [&](auto k) {
        ring_parse_kernel<decltype(k)><<<a.n_conns, RESP_THREADS, parse_smem(proto, a.max_len), st>>>(a);
        return cudaGetLastError();
    });
}

cudaError_t launch_ring_reply(RingProto proto, u32 tiles, const gcra_request *rows, const gcra_result *res,
                              const u32 *stream_ids, const unsigned char *row_proto, const u32 *total, u64 *ctrl,
                              u64 *row_off, unsigned char *out, cudaStream_t st) {
    return for_kind(proto, [&](auto k) {
        ring_reply_kernel<decltype(k)><<<tiles, reply_tile_rows(proto), 0, st>>>(
            rows, res, stream_ids, row_proto, total, ctrl + 1, reinterpret_cast<u32 *>(ctrl), row_off, out);
        return cudaGetLastError();
    });
}

cudaError_t launch_ring_outcome(RingProto proto, u32 n_conns, const uint2 *conn_rows, const gcra_mixed_conn *mconns,
                                const gcra_request *rows, const gcra_result *res, const u32 *total,
                                const u64 *row_off, gcra_resp_outcome *outcome, gcra_grpc_outcome *goutcome,
                                cudaStream_t st) {
    return for_kind(proto, [&](auto k) {
        ring_outcome_kernel<decltype(k)><<<(n_conns + 7) / 8, 256, 0, st>>>(conn_rows, mconns, n_conns, rows, res,
                                                                             total, row_off, outcome, goutcome);
        return cudaGetLastError();
    });
}

}  // namespace gcra
