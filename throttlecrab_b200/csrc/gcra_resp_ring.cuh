// gcra_resp_ring.cuh -- what gcra_b200.cu needs of the rings' kernels (gcra_resp_ring.cu, a translation unit of its
// own): the protocols' bounds, the kernels' shared-memory layout, their arguments and their launches.
#pragma once
#include <cuda_runtime.h>

#include "gcra_device.cuh"
#include "gcra_http.cuh"
#include "gcra_grpc.cuh"
#include "../../include/gcra_b200.h"

namespace gcra {

constexpr u32 RESP_THREADS = 256;
constexpr u32 RESP_MAX_CONN_BYTES = 65536;     // MAX_BUFFER_SIZE of the reference's Redis transport (redis/mod.rs:83)

// The ring's protocol: which grammar its parse kernel takes and which replies its reply kernel writes
// (gcra_resp.cuh for RESP, gcra_http.cuh for HTTP, gcra_grpc.cuh for gRPC); everything else about a ring slot is
// shared.  A gRPC ring has its own connection and outcome tables (gcra_grpc_conn, gcra_grpc_outcome).  A mixed ring
// takes all three in one slot: its connection table (gcra_mixed_conn) names each connection's protocol, and its
// gRPC connections' state and outcome rows are the gRPC ring's tables.
enum RingProto : u32 { PROTO_NONE = 0, PROTO_RESP = 1, PROTO_HTTP = 2, PROTO_GRPC = 3, PROTO_MIXED = 4 };
static_assert(PROTO_RESP == GCRA_PROTO_RESP && PROTO_HTTP == GCRA_PROTO_HTTP && PROTO_GRPC == GCRA_PROTO_GRPC,
              "a ring's protocol is a mixed connection's protocol");

// What the host and the kernels both need of a protocol (a ring's kind for the reply room and tile): the reply bound
// (a mixed ring's is HTTP's, the longest), the rows of a reply tile (the reply kernel stages a tile's replies in shared
// memory, at most 48 KiB), and the smallest plain frame (a connection of len bytes holds at most len / that).
__host__ __device__ constexpr u32 reply_max(RingProto p) {
    return p == PROTO_HTTP || p == PROTO_MIXED ? gcra_http::REPLY_MAX : p == PROTO_GRPC ? gcra_grpc::REPLY_MAX
                                                                                         : gcra_resp::REPLY_MAX;
}
__host__ __device__ constexpr u32 reply_tile_rows(RingProto p) { return p == PROTO_HTTP || p == PROTO_MIXED ? 128 : RESP_THREADS; }
static_assert(gcra_http::REPLY_MAX >= gcra_resp::REPLY_MAX && gcra_http::REPLY_MAX >= gcra_grpc::REPLY_MAX,
              "HTTP's replies are the longest");
__host__ __device__ constexpr u32 min_frame_bytes(RingProto p) {
    return p == PROTO_HTTP ? gcra_http::MIN_FRAME_BYTES : p == PROTO_GRPC ? gcra_grpc::MIN_CALL_BYTES
                                                                          : gcra_resp::MIN_FRAME_BYTES;
}
// The RESP and HTTP parse body's candidate room: candidates per 32 bytes.  A RESP candidate is a '*' that starts the
// segment or follows a '\n', so at most every other byte (16); an HTTP candidate starts "POST ", which cannot overlap
// itself, or a prefix of it at the segment's end, so at most len / 5 + 1 (7 per 32 bytes covers that for every len).
__host__ __device__ constexpr u32 cand_per_word(RingProto p) { return p == PROTO_HTTP ? 7 : 16; }

// The RESP and HTTP parse body's dynamic shared memory for connections of up to `max_len` bytes: the staged bytes (16
// more for the segment's misalignment), one candidate bit per byte, the candidates before each 32-byte word, and one
// word per candidate, `cand_per_word` per 32 bytes.
struct RespSmem {
    u32 words, bytes_off, bits_off, before_off, cand_off, total;
    __host__ __device__ RespSmem(u32 max_len, u32 cand_per_word) {
        words = (max_len + 31) / 32;
        bytes_off = 0;
        bits_off = (words * 32 + 16 + 15) & ~15u;
        before_off = bits_off + 4 * words;
        cand_off = before_off + 4 * words;
        total = cand_off + 4 * (words * cand_per_word) + 16;   // (+16: the start rounded up to 16 bytes)
    }
};

// The gRPC parse body's dynamic shared memory for connections of up to `max_len` bytes: the staged bytes (16 more
// for the segment's misalignment), one word per frame (a frame has at least 9 bytes) and one per call (a call has at
// least gcra_grpc::MIN_CALL_BYTES = 26).
struct GrpcSmem {
    u32 frames_off, calls_off, total;
    __host__ __device__ explicit GrpcSmem(u32 max_len) {
        frames_off = (max_len + 16 + 15) & ~15u;
        calls_off = frames_off + 4 * (max_len / 9 + 1);
        total = calls_off + 4 * (max_len / 26 + 1) + 16;        // (+16: the start rounded up to 16 bytes)
    }
};

// The parse kernel's dynamic shared memory for a ring of kind `ring`: the largest layout of its protocols, for the
// longest connection of each (max_len[p - 1] for protocol p, 0 where none)
inline u32 parse_smem(RingProto ring, const u32 max_len[3]) {
    u32 b = 0;
    for (u32 p = PROTO_RESP; p <= PROTO_GRPC; p++) {
        if (ring != PROTO_MIXED && ring != p) continue;
        const u32 t = p == PROTO_GRPC ? GrpcSmem(max_len[p - 1]).total
                                      : RespSmem(max_len[p - 1], cand_per_word((RingProto)p)).total;
        b = b > t ? b : t;
    }
    return b;
}

// Connection c of a ring of kind `ring`, read from the kind's own table: in[off, + len), its protocol and, for a gRPC
// connection, its row in the gRPC state and outcome tables (c on a gRPC ring)
struct RingConn {
    u32 off, len, proto, grpc_state;
};
__host__ __device__ __forceinline__ RingConn ring_conn(RingProto ring, const gcra_resp_conn *conns,
                                                       const gcra_grpc_conn *gconns, const gcra_mixed_conn *mconns,
                                                       u32 c) {
    if (ring == PROTO_MIXED) {
        const gcra_mixed_conn m = mconns[c];
        return {m.off, m.len, m.protocol, m.grpc_state};
    }
    if (ring == PROTO_GRPC) return {gconns[c].off, gconns[c].len, PROTO_GRPC, c};
    const gcra_resp_conn r = conns[c];
    return {r.off, r.len, ring, 0};
}

// The parse kernel's arguments.  Only the ring kind's own connection table is set: conns (RESP, HTTP), gconns (gRPC)
// or mconns with gconns (mixed: row k of gconns is the connection whose grpc_state is k).
struct RingParse {
    const unsigned char *in;
    const gcra_resp_conn *conns;
    const gcra_grpc_conn *gconns;
    const gcra_mixed_conn *mconns;
    u32 n_conns;
    u32 max_len[3];              // the longest connection of RESP, HTTP and gRPC
    i64 now_ns;
    u32 row_cap;
    u64 k0, k1;                  // the engine's hash seed
    gcra_request *rows;          // the slot's flat row array
    u32 *stream_ids;             // [row_capacity] out: gRPC rows' stream ids
    unsigned char *row_proto;    // [row_capacity] out (mixed): each row's GCRA_PROTO_*
    u64 *status;                 // [n_conns] look-back status words, zero
    u32 *ticket;                 // zero
    uint2 *conn_rows;            // [n_conns] out: first row, rows
    gcra_resp_outcome *outcome;  // [n_conns] out (pinned host memory; not on a gRPC ring)
    gcra_grpc_outcome *goutcome; // [gRPC connections] out (pinned host memory)
    u32 *total, *seg_counts;     // out: rows of the batch, rows of each segment
    u32 nseg, cap_shift;
    uint2 *key_ref;              // [row_capacity] out, or null: each row's key {offset in `in`, length}
};

// A table of key names by key hash: the denied table's keys with their names (gcra_ring_metrics), or a name table of
// its own (gcra_ring_metrics_sharded), whose keys the rows insert.  Both probe linearly from
// mix64(k ^ 0x9E3779B97F4A7C15) & mask for at most 64 entries, with key hash 0 stored as 1.
struct NameTableView {
    u64 *keys;                       // [entries], 0: empty
    u32 mask;                        // entries - 1
    u32 *name_len;                   // [entries] GCRA_NAME_UNKNOWN, GCRA_NAME_TOO_LONG or the name's length
    unsigned char *names;            // [entries][GCRA_DENIED_NAME_MAX]
};

// ring_metrics_kernel's arguments (gcra_ring_metrics, gcra_ring_metrics_sharded): a finished slot's rows, counted per
// transport into counts[3 transports][allowed, denied, errors], and their denied keys named from the slot's input
struct RingMetrics {
    const gcra_request *rows;
    const gcra_result *res;
    const unsigned char *row_proto;  // each row's GCRA_PROTO_* (mixed ring), or null: every row is `proto`'s
    u32 proto;
    const u32 *total;                // rows of the batch
    const uint2 *key_ref;            // each row's key {offset in `in`, length} (the parse kernel's key_ref)
    const unsigned char *in;         // the slot's device input
    u64 *counts;                     // [9]
    NameTableView names;             // keys null: no names
    u64 *full;                       // null: names' keys are the denied table's (looked up, never inserted); else the
                                     // name table's, and the denied rows whose key found it full are counted here
};
// one thread per row of [0, *total), max_rows >= *total
cudaError_t launch_ring_metrics(const RingMetrics &a, u32 max_rows, cudaStream_t st);
// gcra_denied_names on a name table: one warp per hash; out_len[i] its length word (GCRA_NAME_UNKNOWN when absent),
// out_names[i] its bytes (GCRA_DENIED_NAME_MAX per hash)
cudaError_t launch_ring_names_lookup(const NameTableView &t, const u64 *hashes, u32 n, u32 *out_len,
                                     unsigned char *out_names, cudaStream_t st);
// gcra_ring_names_keep: one warp per hash; each of `hashes` found in `from` is inserted with its name into `to`
// (empty); a hash that finds `to` full is counted in *full
cudaError_t launch_ring_names_keep(const NameTableView &from, const NameTableView &to, const u64 *hashes, u32 n,
                                   u64 *full, cudaStream_t st);

cudaError_t resp_ring_setup();   // once, before the first launch
// one CTA per connection of a.n_conns
cudaError_t launch_ring_parse(RingProto proto, const RingParse &a, cudaStream_t st);
// ctrl: word 0 the ticket, then one status word per tile of reply_tile_rows(proto) rows; all zero.  stream_ids: gRPC
// and mixed rings; row_proto: mixed rings.
cudaError_t launch_ring_reply(RingProto proto, u32 tiles, const gcra_request *rows, const gcra_result *res,
                              const u32 *stream_ids, const unsigned char *row_proto, const u32 *total, u64 *ctrl,
                              u64 *row_off, unsigned char *out, cudaStream_t st);
// where each connection's replies lie: outcome[c] (not on a gRPC ring), and a gRPC connection's in its gRPC outcome
// row with the DATA octets of its responses
cudaError_t launch_ring_outcome(RingProto proto, u32 n_conns, const uint2 *conn_rows, const gcra_mixed_conn *mconns,
                                const gcra_request *rows, const gcra_result *res, const u32 *total,
                                const u64 *row_off, gcra_resp_outcome *outcome, gcra_grpc_outcome *goutcome,
                                cudaStream_t st);

}  // namespace gcra
