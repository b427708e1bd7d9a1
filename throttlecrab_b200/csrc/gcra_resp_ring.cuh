// gcra_resp_ring.cuh -- what gcra_b200.cu needs of the RESP ring's kernels (gcra_resp_ring.cu, a translation unit
// of its own): their shared-memory layout and their launches.
#pragma once
#include <cuda_runtime.h>

#include "gcra_device.cuh"
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

// The dynamic shared memory of resp_parse_kernel for connections of up to `max_len` bytes: the staged bytes (16
// more for the segment's misalignment), one candidate bit per byte, the candidates before each 32-byte word, and one
// word per candidate, `cand_per_word` per 32 bytes.  A RESP candidate is a '*' that starts the segment or follows a
// '\n', so at most every other byte (16); an HTTP candidate starts "POST ", which cannot overlap itself, or a prefix
// of it at the segment's end, so at most len / 5 + 1 (7 per 32 bytes covers that for every len).
struct RespSmem {
    u32 words, bytes_off, bits_off, before_off, cand_off, total;
    __host__ __device__ explicit RespSmem(u32 max_len, u32 cand_per_word = 16) {
        words = (max_len + 31) / 32;
        bytes_off = 0;
        bits_off = (words * 32 + 16 + 15) & ~15u;
        before_off = bits_off + 4 * words;
        cand_off = before_off + 4 * words;
        total = cand_off + 4 * (words * cand_per_word) + 16;   // (+16: the start rounded up to 16 bytes)
    }
};

// resp_parse_kernel's arguments: connection c is in[conns[c].off, + conns[c].len)
struct RespParse {
    const unsigned char *in;
    const gcra_resp_conn *conns;
    u32 n_conns, max_len;
    i64 now_ns;
    u32 row_cap;
    u64 k0, k1;                  // the engine's hash seed
    gcra_request *rows;          // the slot's flat row array
    u64 *status;                 // [n_conns] look-back status words, zero
    u32 *ticket;                 // zero
    uint2 *conn_rows;            // [n_conns] out: first row, rows
    gcra_resp_outcome *outcome;  // [n_conns] out (pinned host memory)
    u32 *total, *seg_counts;     // out: rows of the batch, rows of each segment
    u32 nseg, cap_shift;
    RingProto proto;
    uint2 *key_ref;              // [row_capacity] out, or null: each row's key {offset in `in`, length}
};

// a protocol's rows per reply tile (the reply kernel stages a tile's replies in shared memory); a mixed ring's tile
// has room for HTTP's replies, the longest
constexpr u32 MIXED_REPLY_THREADS = 128;
constexpr u32 reply_tile_rows(RingProto p) {
    return p == PROTO_HTTP ? 128 : p == PROTO_MIXED ? MIXED_REPLY_THREADS : RESP_THREADS;
}

// The dynamic shared memory of grpc_parse_kernel for connections of up to `max_len` bytes: the staged bytes (16 more
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

// grpc_parse_kernel's arguments: RespParse's, with the gRPC connection and outcome tables and the rows' stream ids
struct GrpcParse {
    const unsigned char *in;
    const gcra_grpc_conn *conns;
    u32 n_conns, max_len;
    i64 now_ns;
    u32 row_cap;
    u64 k0, k1;
    gcra_request *rows;
    u32 *stream_ids;             // [row_capacity] out
    u64 *status;
    u32 *ticket;
    uint2 *conn_rows;
    gcra_grpc_outcome *outcome;  // [n_conns] out (pinned host memory)
    u32 *total, *seg_counts;
    u32 nseg, cap_shift;
    uint2 *key_ref;              // as in RespParse
};
cudaError_t launch_grpc_parse(const GrpcParse &a, cudaStream_t st);
cudaError_t launch_grpc_reply(u32 tiles, const gcra_request *rows, const gcra_result *res, const u32 *stream_ids,
                              const u32 *total, u64 *ctrl, u64 *row_off, unsigned char *out, cudaStream_t st);
cudaError_t launch_grpc_outcome(u32 n_conns, const uint2 *conn_rows, const gcra_request *rows, const gcra_result *res,
                                const u32 *total, const u64 *row_off, gcra_grpc_outcome *outcome, cudaStream_t st);

// The dynamic shared memory of mixed_parse_kernel: the largest layout that a present protocol needs, for the longest
// connection of each protocol (0 where none)
inline u32 mixed_parse_smem(u32 max_len_resp, u32 max_len_http, u32 max_len_grpc) {
    u32 b = RespSmem(max_len_resp, 16).total;
    b = b > RespSmem(max_len_http, 7).total ? b : RespSmem(max_len_http, 7).total;
    return b > GrpcSmem(max_len_grpc).total ? b : GrpcSmem(max_len_grpc).total;
}

// mixed_parse_kernel's arguments: GrpcParse's with the mixed connection table, the gRPC state table (row k: the
// connection whose grpc_state is k), the gRPC outcome table and each row's protocol
struct MixedParse {
    const unsigned char *in;
    const gcra_mixed_conn *conns;
    u32 n_conns;
    u32 max_len[3];              // the longest connection of RESP, HTTP and gRPC
    const gcra_grpc_conn *gconns;
    i64 now_ns;
    u32 row_cap;
    u64 k0, k1;
    gcra_request *rows;
    u32 *stream_ids;             // [row_capacity] out (gRPC rows)
    unsigned char *row_proto;    // [row_capacity] out: each row's GCRA_PROTO_*
    u64 *status;
    u32 *ticket;
    uint2 *conn_rows;
    gcra_resp_outcome *outcome;  // [n_conns] out (pinned host memory)
    gcra_grpc_outcome *goutcome; // [gRPC connections] out (pinned host memory)
    u32 *total, *seg_counts;
    u32 nseg, cap_shift;
    uint2 *key_ref;              // as in RespParse
};
cudaError_t launch_mixed_parse(const MixedParse &a, cudaStream_t st);
// ctrl: word 0 the ticket, then one status word per tile of MIXED_REPLY_THREADS rows; all zero
cudaError_t launch_mixed_reply(u32 tiles, const gcra_request *rows, const gcra_result *res, const u32 *stream_ids,
                               const unsigned char *row_proto, const u32 *total, u64 *ctrl, u64 *row_off,
                               unsigned char *out, cudaStream_t st);
cudaError_t launch_mixed_outcome(u32 n_conns, const uint2 *conn_rows, const gcra_mixed_conn *conns,
                                 const gcra_request *rows, const gcra_result *res, const u32 *total,
                                 const u64 *row_off, gcra_resp_outcome *outcome, gcra_grpc_outcome *goutcome,
                                 cudaStream_t st);

// ring_metrics_kernel's arguments (gcra_ring_metrics): a finished slot's rows, counted per transport into
// counts[3 transports][allowed, denied, errors], and their denied keys named from the slot's input
struct RingMetrics {
    const gcra_request *rows;
    const gcra_result *res;
    const unsigned char *row_proto;  // each row's GCRA_PROTO_* (mixed ring), or null: every row is `proto`'s
    u32 proto;
    const u32 *total;                // rows of the batch
    const uint2 *key_ref;            // each row's key {offset in `in`, length} (the parse kernel's key_ref)
    const unsigned char *in;         // the slot's device input
    u64 *counts;                     // [9]
    const u64 *denied_keys;          // the denied table's keys (DeniedTable::keys), or null: no names
    u32 denied_mask;                 // its entries - 1
    u32 *name_len;                   // [entries] GCRA_NAME_UNKNOWN, GCRA_NAME_TOO_LONG or the name's length
    unsigned char *names;            // [entries][GCRA_DENIED_NAME_MAX]
};
// one thread per row of [0, *total), max_rows >= *total
cudaError_t launch_ring_metrics(const RingMetrics &a, u32 max_rows, cudaStream_t st);

cudaError_t resp_ring_setup();   // once, before the first launch
cudaError_t launch_resp_parse(const RespParse &a, cudaStream_t st);
// ctrl: word 0 the ticket, then one status word per tile of reply_tile_rows(proto) rows; all zero
cudaError_t launch_resp_reply(RingProto proto, u32 tiles, const gcra_request *rows, const gcra_result *res,
                              const u32 *total, u64 *ctrl, u64 *row_off, unsigned char *out, cudaStream_t st);
cudaError_t launch_resp_outcome(u32 n_conns, const uint2 *conn_rows, const u32 *total, const u64 *row_off,
                                gcra_resp_outcome *outcome, cudaStream_t st);

}  // namespace gcra
