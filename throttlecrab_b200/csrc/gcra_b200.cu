// gcra_b200.cu -- host side of the engine and the C ABI declared in include/gcra_b200.h.
//
// Host responsibilities: table allocation/growth (HashMap::with_capacity / growth), the sweep
// policies of the three reference stores (adaptive_cleanup.rs:138-211, periodic.rs:128-142,
// probabilistic.rs:110-125) driving the sweep kernel, kernel sequencing on CUDA streams, and the
// pinned host ring.  All decisions are made by the kernels in gcra_kernels.cuh; there is no CPU
// decision path.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <dlfcn.h>
#include <cstring>
#include <fcntl.h>
#include <memory>
#include <string>
#include <sys/stat.h>
#include <thread>
#include <type_traits>
#include <unistd.h>
#include <vector>

#include "gcra_kernels.cuh"
#include "gcra_index_path.cuh"
#include "gcra_p2p.cuh"
#include "gcra_owned.cuh"
#include "gcra_resp_ring.cuh"

using namespace gcra;

// (reported through h->err; cudaGetLastError clears the runtime's record, so that no later launch check reports it)
#define CK(call)                                                                         \
    do {                                                                                 \
        cudaError_t e_ = (call);                                                         \
        if (e_ != cudaSuccess) {                                                         \
            h->err = std::string(#call) + ": " + cudaGetErrorString(e_);                 \
            cudaGetLastError();                                                          \
            return GCRA_INTERNAL;                                                        \
        }                                                                                \
    } while (0)

#define RC(call)                                  \
    do {                                          \
        int rc_ = (call);                         \
        if (rc_ != GCRA_OK) return rc_;           \
    } while (0)

namespace {
const __int128 NS_PER_S = 1000000000;

struct RingSlot {
    PinnedBuf<unsigned char> h_req;
    PinnedBuf<unsigned char> h_res;  // gcra_result, or gcra_result16 rows in ring mode 2
    DevBuf<unsigned char> d_req, d_res;
    PinnedBuf<unsigned char> h_keys; // keyed ring: the key arena the rows' key references point into
    DevBuf<unsigned char> d_keys;
    Event ev_in, ev_done;
    bool in_flight = false;
    // RESP or HTTP ring (gcra_resp_ring_create, gcra_http_ring_create): the rows are d_req / d_res, viewed as
    // resp_nseg segments
    PinnedBuf<unsigned char> h_in, h_replies;   // (the kernels write h_replies and h_outcome)
    PinnedBuf<gcra_resp_conn> h_conns;
    PinnedBuf<gcra_resp_outcome> h_outcome;
    DevBuf<unsigned char> d_in;
    DevBuf<gcra_resp_conn> d_conns;
    DevBuf<uint2> conn_rows;            // [max_conns] first row, rows
    DevBuf<u64> parse_ctrl, reply_ctrl; // word 0: ticket, then the look-back status words (connections | reply tiles)
    DevBuf<u64> row_off;                // [row_capacity + 1] where each row's reply starts
    DevBuf<u32> counts;                 // [0] rows of the batch, [1 + s] rows of segment s
    DevBuf<SegDesc> segs;
    // gRPC ring (gcra_grpc_ring_create): its connection and outcome tables in place of h_conns / h_outcome, and each
    // row's stream id
    PinnedBuf<gcra_grpc_conn> h_gconns;
    PinnedBuf<gcra_grpc_outcome> h_goutcome;
    DevBuf<gcra_grpc_conn> d_gconns;
    DevBuf<u32> stream_ids;
    // mixed ring (gcra_mixed_ring_create): its connection table, with h_outcome and the gRPC tables above, and each
    // row's protocol
    PinnedBuf<gcra_mixed_conn> h_mconns;
    DevBuf<gcra_mixed_conn> d_mconns;
    DevBuf<unsigned char> row_proto;
    // ring metrics (gcra_ring_metrics): each row's key {offset in d_in, length}, written by the parse kernels
    DevBuf<uint2> key_ref;
    // a peer-memory tick routed from this slot (gcra_resp_ring_submit_route): its connections and the bound of its rows
    uint32_t routed_conns = 0, routed_rows = 0;
};
}  // namespace

// ---- NCCL, resolved at run time (dlopen) so that single-GPU users do not need it ---------------------
// Minimal declarations of the public NCCL API used here (nccl.h: ncclUniqueId is 128 opaque bytes,
// ncclUint8 = 1, ncclUint32 = 3).
namespace nccl_rt {
struct UniqueId { char internal[128]; };
typedef void *Comm;
typedef int (*GetUniqueId_t)(UniqueId *);
typedef int (*CommInitRank_t)(Comm *, int, UniqueId, int);
typedef int (*CommDestroy_t)(Comm);
typedef int (*Group_t)();
typedef int (*Send_t)(const void *, size_t, int, int, Comm, cudaStream_t);
typedef int (*Recv_t)(void *, size_t, int, int, Comm, cudaStream_t);
typedef const char *(*ErrStr_t)(int);
struct Api {
    void *lib = nullptr;
    GetUniqueId_t GetUniqueId = nullptr;
    CommInitRank_t CommInitRank = nullptr;
    CommDestroy_t CommDestroy = nullptr;
    Group_t GroupStart = nullptr, GroupEnd = nullptr;
    Send_t Send = nullptr;
    Recv_t Recv = nullptr;
    ErrStr_t GetErrorString = nullptr;
};
static Api g_api;
static bool load() {
    if (g_api.lib) return true;
    void *l = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!l) l = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!l) return false;
    Api a;
    a.lib = l;
    a.GetUniqueId = (GetUniqueId_t)dlsym(l, "ncclGetUniqueId");
    a.CommInitRank = (CommInitRank_t)dlsym(l, "ncclCommInitRank");
    a.CommDestroy = (CommDestroy_t)dlsym(l, "ncclCommDestroy");
    a.GroupStart = (Group_t)dlsym(l, "ncclGroupStart");
    a.GroupEnd = (Group_t)dlsym(l, "ncclGroupEnd");
    a.Send = (Send_t)dlsym(l, "ncclSend");
    a.Recv = (Recv_t)dlsym(l, "ncclRecv");
    a.GetErrorString = (ErrStr_t)dlsym(l, "ncclGetErrorString");
    if (!a.GetUniqueId || !a.CommInitRank || !a.CommDestroy || !a.GroupStart || !a.GroupEnd || !a.Send || !a.Recv) return false;
    g_api = a;
    return true;
}
const int kUint8 = 1, kUint32 = 3;
}  // namespace nccl_rt

inline void release_comm(nccl_rt::Comm c) { nccl_rt::g_api.CommDestroy(c); }

struct NcclComm : Owned<nccl_rt::Comm, release_comm> {   // (make returns an NCCL result code)
    int make(int world, nccl_rt::UniqueId id, int rank) { reset(); return took(nccl_rt::g_api.CommInitRank(&h_, world, id, rank)); }
    nccl_rt::Comm get() const { return h_; }
};

// one tick in flight through the sharded pipeline
struct ShardSlot {
    DevBuf<gcra_request> routed, recv_req;
    DevBuf<gcra_result> recv_res, back_res;
    DevBuf<u32> src_index;
    DevBuf<u32> counts_dev;        // [2*W]: rows I send to every peer, rows every peer sends me
    PinnedBuf<u32> counts_host;    // pinned copy
    Event ev_ready, ev_counts, ev_routed, ev_done;
    bool used = false;
    uint32_t n = 0, n_recv = 0;
    gcra_result *d_res_user = nullptr;
    std::vector<size_t> send, recv, send_off, recv_off;
};

struct Shard {
    static const int DEPTH = 4;
    int rank = 0, world = 0;
    uint32_t max_rows = 0;
    Stream s_part, s_route, s_return;   // partition+counts | request all-to-all | way back
    NcclComm comm_counts, comm_req, comm_res;
    ShardSlot slots[DEPTH];
    uint32_t next = 0;
    int pending = -1;              // slot whose decide + return stages have not been issued yet
    Event ev_tmp;
};

// ---- multi-GPU over NVLink peer memory (gcra_p2p.cuh) ------------------------------------------------------
struct P2PSlot {
    DevBuf<u32> res_loc;               // [cap] where the result of my row i arrives in my outbox
    DevBuf<u32> counts_dev;            // [world] rows I routed to every owner in this tick
    DevBuf<SegDesc> segs_dev;          // [world] segment r of this inbox slot: sender r's rows, sender r's outbox
    Event ev_ready, ev_wait, ev_done;
    bool used = false;
    uint32_t n = 0;                    // rows routed, or (dev_n) a bound of them
    const u32 *dev_n = nullptr;        // a ring tick's row count on the device (gcra_resp_ring_submit_route)
    bool room_reserved = false;        // a ring tick made its room in the table before its route (p2p_room)
};

struct P2P {
    int rank = 0, world = 0;
    uint32_t cap = 0, cap_shift = 0;
    DevBuf<unsigned char> window;
    size_t window_bytes = 0, inbox_off = 0, outbox_off = 0;
    IpcMapping peer_map[P2P_MAX_WORLD];    // the windows of other processes' ranks (gcra_p2p_connect with IPC handles)
    bool connected = false, routed_pending = false;
    int ring_slot_pending = -1;            // the ring slot whose tick was routed (gcra_resp_ring_submit_route)
    P2PPeers peers_host;                   // peers_dev as this process addresses it
    DevBuf<P2PPeers> peers_dev;
    DevBuf<u32> tile_counts;
    Stream s_part, s_wait, s_sig, s_return;
    P2PSlot slots[P2P_DEPTH];
    uint64_t next_tick = 0;
    bool timed = false, timed_valid = false;
    Event ev_t[6];
};

// per-batch scratch; several sets so that the front halves of the next batches can overlap the back half of
// the current one
struct Scratch {
    DevBuf<Req> drec;
    DevBuf<u64> keys_a, keys_b;
    DevBuf<u32> sort_ws;                // enqueue_sort: tickets, digit counts, status words (sort_ws_words)
    DevBuf<LongRun> long_runs, giant_runs;
    DevBuf<u32> long_count;
    Event ev_front, ev_mid, ev_back, ev_fork, ev_join, ev_join_giant;
    bool back_recorded = false;
    // index-order pipeline (gcra_index_path.cuh)
    DevBuf<u32> slot_arr;               // [rows] slot of every row (null slot: the row failed validation)
    DevBuf<unsigned char> flags;        // [rows] pass-B verdict of rows on shared slots
    DevBuf<u32> bitmap;                 // [bm_words] 32-bit occurrence counters of the batch, hashed by slot
    DevBuf<u32> pend;                   // [pend_words] 1 bit per entry: the PREVIOUS batch's tail owns a slot of the entry
    DevBuf<u64> ctrl_block;             // word 0: {tile ticket, residue count}; then one status word per tile
    uint32_t rows_alloc = 0;
    PinnedBuf<u32> h_nres;              // pinned: residue size of the set's latest index-order batch (valid after ev_mid)
    bool mid_recorded = false, nres_counted = true;
    uint32_t nres_rows = 0;             // rows of that batch
};

// One hash table: its arrays, its counters, the view of both that the kernels take, and the capacity it was made for
// (make_table).  The engine's table is replaced only whole (install_table).
struct HostTable {
    DevBuf<u64> keys, mark;
    DevBuf<TatOff> state;
    DevBuf<i64> ei;
    DevBuf<u64> counters;            // [C_COUNT]
    Table view{};
    uint64_t capacity = 0;
    uint64_t load_limit = 0;         // claimed slots past which the table grows (table_geometry)
    uint64_t slots() const { return (uint64_t)view.null_slot + 1; }
    uint32_t lines() const { return view.null_slot / 4 + 1; }
};

// the arrays of the denied-key table: gcra_engine::denied is the view the kernels take.  names / name_len: the keys'
// names (GCRA_DENIED_NAME_MAX bytes, and a length word, per entry), while ring metrics are on
struct DeniedArrays {
    DevBuf<u64> keys, counts, dropped;
    DevBuf<unsigned char> names;
    DevBuf<u32> name_len;
};

// the name table of sharded ring metrics (gcra_ring_metrics_sharded): keys by hash, each with its name, and the
// denied rows whose key found the table full since it was made.  Replaced whole by gcra_ring_names_keep.
struct NameTable {
    DevBuf<u64> keys, full;
    DevBuf<u32> name_len;
    DevBuf<unsigned char> names;
    uint64_t cap = 0;                // entries (0: counts without names)
    NameTableView view() const { return {keys.get(), (u32)(cap - 1), name_len.get(), names.get()}; }
};

// the header of a snapshot file (gcra_snapshot_save, gcra_snapshot_begin)
namespace {
struct SnapshotHeader {
    char magic[8];
    uint32_t version, total_lines, nb_main, stash_slots;
    uint64_t capacity;
    uint64_t counters[C_COUNT];
    uint64_t hash_seed[2];           // (version 2) the identities in the table were made with this seed
};
const char SNAP_MAGIC[8] = {'G', 'C', 'R', 'A', 'B', '2', '0', '0'};
const size_t SNAP_CHUNK = 32u << 20;
}  // namespace

// What background saves (gcra_snapshot_begin) keep on the engine and reuse: made by the first save, grown by a later
// one that needs more room, released by gcra_destroy.
struct SnapshotStaging {
    Stream stream;                   // the capture, then the writer thread's copies (one thread at a time uses it)
    Event ev_store, ev_capture, ev_chunk[2];
    StreamBuf<unsigned char> dev;    // ctrl words | keys | (tat, off) pairs | ei
    size_t dev_bytes = 0;
    PinnedBuf<char> chunk[2];        // double-buffered copies on their way to the file
    PinnedBuf<u64> meta;             // [C_COUNT] the counters at the cut, then the entry count
    uint32_t grid = 0;               // persistent CTAs of snapshot_capture_kernel
};

// one background save: what its writer thread needs, and what it reports (read once `finished` is set)
struct SnapshotJob {
    std::thread writer;
    std::atomic<bool> finished{false};
    int rc = 0;
    std::string err;
    uint64_t entries = 0;
    int fd = -1;
    std::string tmp, path;
    SnapshotHeader hd{};                                       // the table at the cut; the writer adds the counters
    uint64_t cap = 0;                                          // entries the staging sections hold
    size_t keys_off = 0, state_off = 0, ei_off = 0;            // the sections in the staging
};

// Members are released in reverse declaration order, after gcra_destroy has synchronized the device: no release waits.
struct gcra_engine {
    int device = 0;
    uint32_t sms = 0;                // streaming multiprocessors of the device: sizes the grids of the streaming kernels
    Stream stream, in_stream, out_stream;
    Stream aux_stream, aux2_stream;  // hot runs beside the decide kernel: one CTA per run, one cluster per run
    HostTable tab;                   // replaced whole by grow and gcra_snapshot_load
    bool tight = false;              // GCRA_FLAG_TIGHT_TABLE: tests only, exercises stash + growth
    // scratch for one batch
    uint32_t max_batch = 0;
#ifndef GCRA_PIPE_SETS
#define GCRA_PIPE_SETS 4
#endif
    static const int N_SCR = GCRA_PIPE_SETS;
    Scratch scr[N_SCR];
    uint32_t scr_next = 0;
    // pipelined submission: three stages on three streams (front: probe | mid: decide + resolve | tail: the
    // sorted residue); the sort pipeline uses front (ingest + sort) and mid (decide)
    // (ONE front stream shared by all scratch sets: front halves run one after another; since ingest only CASes
    // the keys array they could overlap as well -- not measured yet)
    Stream front_stream, back_stream, tail_stream;
    int pend_set = -1;               // scratch set whose bitmap holds the PEND bits of the batch submitted last (-1: none)
    Event ev_ready;
    DevBuf<gcra_request> d_req;      // (16-byte rows in the compact formats)
    DevBuf<gcra_result> d_res;
    DevBuf<u32> route_counts;
    DevBuf<PolicyDerived> d_pol;
    uint32_t npol = 0;
    DevBuf<StoreOpResult> d_op;
    PinnedBuf<StoreOpResult> h_op;
    PinnedBuf<u64> h_counters;       // pinned snapshot, refreshed after every batch
    Event ev_counters;
    Event ev[4];
    Event evd[8];                    // index-order pipeline, serial timed batch: after each kernel group
    bool evd_valid = false;
    Event ev_sweep[2];
    bool sweep_timed = false;
    bool ev_valid = false;
    uint64_t launches = 0;
    uint64_t occupied_ub = 0;        // host-side upper bound of claimed slots
    // asynchronous occupancy snapshots: counters copied after every batch, read when their event is done
    static const int N_SNAP = 8;
    PinnedBuf<u64> h_snap;           // pinned [N_SNAP][C_COUNT]
    Event ev_snap[N_SNAP];
    uint64_t snap_rows_after[N_SNAP] = {};   // rows launched up to and including the snapshot's batch
    bool snap_used[N_SNAP] = {};
    uint32_t snap_next = 0;
    uint64_t rows_launched = 0;
    // store policy (mirrors the reference stores' fields)
    int kind = GCRA_STORE_ADAPTIVE;
    __int128 next_cleanup = 0, cleanup_interval = 0;
    __int128 min_interval = 0, max_interval = 0, cur_interval = 0;
    uint64_t expired_count = 0, ops_since_cleanup = 0, max_ops = 0;
    uint64_t last_removed = 0, last_total = 0;
    uint64_t ops_count = 0, cleanup_modulo = 0;
    uint64_t seen_allowed = 0, seen_expired_hits = 0;
    uint64_t n_sweeps = 0, n_grows = 0, n_purges = 0;
    std::unique_ptr<Shard> shard;    // multi-GPU: native NCCL pipeline (gcra_shard_*)
    std::unique_ptr<P2P> p2p;        // multi-GPU: NVLink peer-memory pipeline (gcra_p2p_*)
    // index-order pipeline
    uint32_t epoch = 0;              // batch epoch of the slot marks (never 0)
    uint32_t bm_mask = 0;            // bitmap entries - 1
    size_t bm_words = 0, pend_words = 0;
    uint32_t index_min = 0;          // batches of at least this many rows take the index-order pipeline (0: never)
    int prefetch_state = 0;
    uint32_t max_tiles = 0;
    uint32_t grid_probe[FMT_COUNT] = {}, grid_decide[FMT_COUNT] = {};   // resident CTAs of the persistent kernels [RowFmt]
    uint32_t grid_denied_seg = 0;    // resident CTAs of denied_count_seg_kernel
    uint32_t dbg = 0;                // timing experiments only (gcra_debug_set): skips parts of pass B
    uint32_t last_nres = 0, last_nres_rows = 0;   // newest residue size that has reached the host (and its batch's rows)
    bool adaptive = true;            // choose the pipeline from the residue feedback (off when a test / env forces one)
    uint64_t n_path_switches = 0;
    uint32_t sort_hold = 0;          // > 0: the residue was large, this many more batches take the sort pipeline
    uint32_t since_drain = 0;        // index-order batches submitted since stage 2 last waited for every tail
    uint64_t n_drains = 0, n_index_batches = 0, residue_seen = 0, residue_batches_seen = 0;
    // ring
    std::vector<RingSlot> ring;
    uint32_t ring_cap = 0;
    int ring_fmt = FMT_48_32;        // the slots' RowFmt (gcra_ring_create)
    uint64_t ring_key_cap = 0;       // bytes of every slot's key arena (0: the ring is not keyed)
    RingProto ring_proto = PROTO_NONE;   // a RESP, HTTP, gRPC or mixed ring (gcra_resp_ring_create, _http_, _grpc_, _mixed_)
    uint32_t resp_max_conns = 0, resp_nseg = 0, resp_shift = 0;
    uint64_t resp_in_cap = 0;
    DevBuf<unsigned char> d_keys;    // gcra_rate_limit_batch_keys: the caller's key arena on the device
    uint64_t d_keys_cap = 0;
    // denied requests per key (gcra_track_denied): device table, updated by a pass over every finished batch
    DeniedArrays denied_arrays;
    DeniedTable denied{};
    uint32_t denied_max = 0;
    uint64_t denied_cap = 0;
    // ring metrics (gcra_ring_metrics): ring rows per transport [3][allowed, denied, errors]
    bool ring_metrics = false;
    DevBuf<u64> ring_counts;
    // sharded ring metrics (gcra_ring_metrics_sharded): the same counts, names in a table of this rank's own
    bool ring_metrics_sharded = false;
    NameTable ring_names;
    bool ring_p2p = false;           // gcra_ring_p2p: every ring submit is a peer-memory tick
    uint64_t hash_seed[2] = {0, 0};  // SipHash key of the string-keyed entry points ((0,0): the unkeyed gcra_hash_key)
    // background saves (gcra_snapshot_begin); gcra_destroy joins the writer thread before anything is released
    std::unique_ptr<SnapshotStaging> snap;
    std::unique_ptr<SnapshotJob> job;
    bool capture_pending = false;    // launches that touch the table wait for snap->ev_capture
    std::string err;
};

// Until the capture of a background save has completed, work that may touch the table waits for it on `st`; once
// it has completed, this is one flag test.
static int after_capture(gcra_engine *h, cudaStream_t st) {
    if (!h->capture_pending) return GCRA_OK;
    if (cudaEventQuery(h->snap->ev_capture.get()) == cudaSuccess) { h->capture_pending = false; return GCRA_OK; }
    CK(cudaStreamWaitEvent(st, h->snap->ev_capture.get(), 0));
    return GCRA_OK;
}

// Whatever touches the table outside a batch comes after every batch in flight, whichever streams it was submitted
// on (the last stage of each records its scratch set's ev_back, finish_batch): on `st`, or on the host.
static int order_after_batches(gcra_engine *h, cudaStream_t st) {
    for (auto &o : h->scr) if (o.back_recorded) CK(cudaStreamWaitEvent(st, o.ev_back.get(), 0));
    return GCRA_OK;
}
static int wait_for_batches(gcra_engine *h) {
    for (auto &o : h->scr) if (o.back_recorded) CK(cudaEventSynchronize(o.ev_back.get()));
    return GCRA_OK;
}
// What reads or rewrites the denied table or the ring counts waits for the batches and for the ring slots in flight:
// a ring slot counts and names on its reply stream, after its batch's ev_back.  (The slots stay in flight for
// gcra_ring_wait.)
static int wait_for_metrics_writers(gcra_engine *h) {
    RC(wait_for_batches(h));
    for (auto &s : h->ring) if (s.in_flight) CK(cudaEventSynchronize(s.ev_done.get()));
    return GCRA_OK;
}

static uint32_t ceil_log2(uint64_t x) {
    uint32_t b = 0;
    while ((1ULL << b) < x) b++;
    return b;
}

// The shape of a table for `capacity` entries: its lines of 4 slots, the buckets the two hash choices address, the
// stash, and the claimed slots past which the table grows.
struct Geometry { uint32_t total_lines, nb_main, stash_slots; uint64_t load_limit; };

static Geometry table_geometry(uint64_t capacity, bool tight) {
    // first-fit two-choice buckets of 4 stay below ~0.4 % stash traffic up to load 0.5
    uint64_t slots = 1ULL << ceil_log2(std::max<uint64_t>(tight ? capacity : capacity * 2, tight ? 64 : 256));
    Geometry g;
    g.total_lines = (uint32_t)(slots / 4);
    uint32_t ns = std::max<uint32_t>(tight ? g.total_lines / 4 : g.total_lines / 64, 8);
    g.nb_main = g.total_lines - ns;
    g.stash_slots = (ns - 1) * 4;   // the last line is reserved (null slot)
    const uint64_t main_slots = (uint64_t)g.nb_main * 4;
    g.load_limit = tight ? main_slots * 13 / 16 : main_slots / 2;
    return g;
}

// an empty table for `capacity` entries in `t`, zeroed counters included (enqueued on h->stream)
static int make_table(gcra_engine *h, uint64_t capacity, HostTable &t) {
    const Geometry g = table_geometry(capacity, h->tight);
    const size_t slots = (size_t)g.total_lines * 4;
    CK(t.counters.make(C_COUNT));
    CK(cudaMemsetAsync(t.counters.get(), 0, C_COUNT * sizeof(u64), h->stream.get()));
    CK(t.keys.make(slots));
    CK(t.state.make(slots));
    CK(t.ei.make(slots));
    CK(t.mark.make(slots));
    Table &v = t.view;
    v.keys = t.keys.get(); v.state = t.state.get(); v.ei = t.ei.get(); v.mark = t.mark.get();
    CK(cudaMemsetAsync(v.mark, 0xff, slots * sizeof(u64), h->stream.get()));   // no batch epoch matches
    v.nb_main = g.nb_main;
    v.stash_slots = g.stash_slots;
    v.null_slot = g.total_lines * 4 - 1;
    v.slot_bits = ceil_log2((uint64_t)g.total_lines * 4);
    v.counters = t.counters.get();
    t.capacity = capacity;
    t.load_limit = g.load_limit;
    uint32_t grid = (uint32_t)std::min<size_t>((slots + TILE_THREADS - 1) / TILE_THREADS, 16 * h->sms);
    clear_slots_kernel<<<grid, TILE_THREADS, 0, h->stream.get()>>>(v, 0, slots);
    h->launches++;
    CK(cudaGetLastError());
    return GCRA_OK;
}

// `occupied` claimed slots were just read from the device: the host's bound restarts from it, and the occupancy
// snapshots taken before it are stale
static void reset_occupancy(gcra_engine *h, uint64_t occupied) {
    h->occupied_ub = occupied;
    for (bool &used : h->snap_used) used = false;
}

// The counters of a table filled from another one (growth, a version 3 load): the traffic totals `c` carries over,
// with the occupancy that the new table counted while it was filled (`fresh`).
static void take_occupancy(u64 c[C_COUNT], const u64 fresh[C_COUNT]) {
    c[C_OCCUPIED] = fresh[C_OCCUPIED];
    c[C_REAL] = fresh[C_REAL];
    c[C_STASH] = fresh[C_STASH];
}

// `t` (filled, nothing in flight on it) replaces the engine's table, with `counters` as its counter words.  The sweep
// policy's view of the counters (seen_allowed, seen_expired_hits) is the caller's to set.
static int install_table(gcra_engine *h, HostTable &&t, const u64 counters[C_COUNT]) {
    CK(cudaMemcpyAsync(t.counters.get(), counters, C_COUNT * sizeof(u64), cudaMemcpyHostToDevice, h->stream.get()));
    CK(cudaStreamSynchronize(h->stream.get()));
    h->tab = std::move(t);
    reset_occupancy(h, counters[C_OCCUPIED]);
    return GCRA_OK;
}

static int refresh_counters(gcra_engine *h, bool wait) {
    CK(cudaMemcpyAsync(h->h_counters.get(), h->tab.view.counters, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost, h->stream.get()));
    CK(cudaEventRecord(h->ev_counters.get(), h->stream.get()));
    if (wait) CK(cudaEventSynchronize(h->ev_counters.get()));
    return GCRA_OK;
}

static int do_sweep(gcra_engine *h, int64_t now_ns, uint64_t *removed) {
    CK(cudaSetDevice(h->device));
    CK(cudaDeviceSynchronize());   // the sweep is exclusive: batches may be in flight on caller streams
    RC(refresh_counters(h, true));
    uint64_t before = h->h_counters.get()[C_SWEPT];
    uint32_t grid = (uint32_t)std::min<uint64_t>((h->tab.slots() / 2 + TILE_THREADS * SWEEP_UNROLL - 1) / (TILE_THREADS * SWEEP_UNROLL), 16 * h->sms);
    CK(cudaEventRecord(h->ev_sweep[0].get(), h->stream.get()));
    static const int sweep_mode = getenv("GCRA_SWEEP_MODE") ? atoi(getenv("GCRA_SWEEP_MODE")) : 0;
    sweep_kernel<<<grid, TILE_THREADS, 0, h->stream.get()>>>(h->tab.view, h->tab.slots(), now_ns, sweep_mode);
    CK(cudaEventRecord(h->ev_sweep[1].get(), h->stream.get()));
    h->sweep_timed = true;
    h->launches++;
    CK(cudaGetLastError());
    RC(refresh_counters(h, true));
    reset_occupancy(h, h->h_counters.get()[C_OCCUPIED]);
    h->n_sweeps++;
    if (removed) *removed = h->h_counters.get()[C_SWEPT] - before;
    return GCRA_OK;
}

// reclaim the slots of keys without an entry (exclusive); returns with fresh counters
static int purge(gcra_engine *h) {
    CK(cudaDeviceSynchronize());
    const uint64_t slots = h->tab.slots();
    uint32_t grid = (uint32_t)std::min<uint64_t>((slots + TILE_THREADS - 1) / TILE_THREADS, 16 * h->sms);
    purge_kernel<<<grid, TILE_THREADS, 0, h->stream.get()>>>(h->tab.view, slots);
    h->launches++;
    CK(cudaGetLastError());
    RC(refresh_counters(h, true));
    if (h->h_counters.get()[C_STASH] == 0) {
        // no key lives in the stash any more: drop its tombstones
        uint64_t first = (uint64_t)h->tab.view.nb_main * 4, cnt = slots - first;
        clear_slots_kernel<<<(uint32_t)((cnt + TILE_THREADS - 1) / TILE_THREADS), TILE_THREADS, 0, h->stream.get()>>>(
            h->tab.view, first, cnt);
        h->launches++;
        CK(cudaGetLastError());
    }
    reset_occupancy(h, h->h_counters.get()[C_OCCUPIED]);
    h->n_purges++;
    return GCRA_OK;
}

// HashMap growth: rebuild into a table twice the size
static int grow(gcra_engine *h, uint64_t need) {
    CK(cudaStreamSynchronize(h->stream.get()));
    uint64_t newcap = std::max<uint64_t>(h->tab.capacity * 2, 256);
    while (table_geometry(newcap, h->tight).load_limit < need) newcap *= 2;
    HostTable nt;
    RC(make_table(h, newcap, nt));
    uint32_t grid = std::min<uint32_t>((h->tab.lines() + TILE_THREADS - 1) / TILE_THREADS, 8 * h->sms);
    rehash_kernel<<<grid, TILE_THREADS, 0, h->stream.get()>>>(h->tab.view, h->tab.slots(), nt.view);
    h->launches++;
    CK(cudaGetLastError());
    // carry the running totals over
    RC(refresh_counters(h, true));
    u64 keep[C_COUNT];
    memcpy(keep, h->h_counters.get(), sizeof(keep));
    u64 fresh[C_COUNT];
    CK(cudaMemcpyAsync(fresh, nt.counters.get(), sizeof(fresh), cudaMemcpyDeviceToHost, h->stream.get()));
    CK(cudaStreamSynchronize(h->stream.get()));
    if (fresh[C_INSERT_FAIL]) { h->err = "table growth lost entries"; return GCRA_INTERNAL; }
    take_occupancy(keep, fresh);
    RC(install_table(h, std::move(nt), keep));
    h->n_grows++;
    return GCRA_OK;
}

// The bound is stale (it assumes every request claimed a slot): tighten it from the newest counter snapshot that has
// already arrived, without stalling the stream.
static void tighten_occupied_ub(gcra_engine *h) {
    for (int back = 1; back <= gcra_engine::N_SNAP; back++) {
        int k = (int)((h->snap_next + gcra_engine::N_SNAP - back) % gcra_engine::N_SNAP);
        if (!h->snap_used[k]) break;
        if (cudaEventQuery(h->ev_snap[k].get()) != cudaSuccess) continue;
        uint64_t ub = h->h_snap.get()[(size_t)k * C_COUNT + C_OCCUPIED] + (h->rows_launched - h->snap_rows_after[k]);
        if (ub < h->occupied_ub) h->occupied_ub = ub;
        break;
    }
}

static int ensure_room(gcra_engine *h, uint64_t n) {
    if (h->occupied_ub + n <= h->tab.load_limit) { h->occupied_ub += n; return GCRA_OK; }
    tighten_occupied_ub(h);
    if (h->occupied_ub + n <= h->tab.load_limit) { h->occupied_ub += n; return GCRA_OK; }
    int rc = refresh_counters(h, true);
    if (rc) return rc;
    CK(cudaDeviceSynchronize());   // batches may be in flight on caller streams
    rc = refresh_counters(h, true);
    if (rc) return rc;
    h->occupied_ub = h->h_counters.get()[C_OCCUPIED];
    if (h->occupied_ub + n > h->tab.load_limit && h->h_counters.get()[C_OCCUPIED] > h->h_counters.get()[C_REAL]) {
        // crowded: first give back the slots of keys that hold no entry (swept or only ever denied)
        rc = purge(h);
        if (rc) return rc;
    }
    if (h->occupied_ub + n > h->tab.load_limit) {
        rc = grow(h, (h->occupied_ub + n));
        if (rc) return rc;
    }
    h->occupied_ub += n;
    return GCRA_OK;
}

static int snapshot_async(gcra_engine *h, uint64_t n, cudaStream_t st) {
    h->rows_launched += n;
    int k = (int)h->snap_next;
    h->snap_next = (h->snap_next + 1) % gcra_engine::N_SNAP;
    CK(cudaMemcpyAsync(h->h_snap.get() + (size_t)k * C_COUNT, h->tab.view.counters, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(h->ev_snap[k].get(), st));
    h->snap_rows_after[k] = h->rows_launched;
    h->snap_used[k] = true;
    return GCRA_OK;
}

// ---- sweep policies ------------------------------------------------------------------------
static bool adaptive_should_clean(const gcra_engine *h, __int128 now, uint64_t len) {   // adaptive_cleanup.rs:138-171
    if (now >= h->next_cleanup) return true;
    if (h->ops_since_cleanup >= h->max_ops) return true;
    if (h->expired_count > 50) {
        double ratio = (double)h->expired_count / (double)(len ? len : 1);
        double threshold = (h->last_removed > h->last_total / 4) ? 0.2 / 2.0 : 0.2 * 1.25;
        if (ratio > threshold) return true;
    }
    if (len > h->tab.load_limit * 3 / 4) return true;
    return false;
}

// called at batch boundaries with the counters of the batches finished so far
static int apply_policy(gcra_engine *h, int64_t now_ns) {
    if (h->kind == GCRA_STORE_MANUAL) return GCRA_OK;
    uint64_t allowed = h->h_counters.get()[C_ALLOWED], hits = h->h_counters.get()[C_EXPIRED_HITS];
    uint64_t d_ops = allowed - h->seen_allowed, d_hits = hits - h->seen_expired_hits;
    h->seen_allowed = allowed;
    h->seen_expired_hits = hits;
    __int128 now = now_ns;
    uint64_t removed = 0;
    if (h->kind == GCRA_STORE_PERIODIC) {                       // periodic.rs:128-142
        if (now >= h->next_cleanup) {
            int rc = do_sweep(h, now_ns, &removed);
            if (rc) return rc;
            h->expired_count = removed;
            h->next_cleanup = now + h->cleanup_interval;
        }
    } else if (h->kind == GCRA_STORE_PROBABILISTIC) {           // probabilistic.rs:110-125
        // sweep when some op count k in (ops, ops + d_ops] has k * 2654435761 % modulo == 0
        const uint64_t c = 2654435761ULL, m = h->cleanup_modulo;
        uint64_t a = h->ops_count + 1, b = h->ops_count + d_ops;
        bool hit = false;
        if (d_ops) {
            if (b < (~0ULL) / c) {
                uint64_t g = m, x = c % m;
                while (x) { uint64_t tmp = g % x; g = x; x = tmp; }
                uint64_t step = m / g;
                hit = (b / step) > ((a - 1) / step);
            } else {
                for (uint64_t k = a; k <= b && !hit; k++) hit = ((k * c) % m) == 0;
            }
        }
        h->ops_count = b;
        if (hit) { int rc = do_sweep(h, now_ns, &removed); if (rc) return rc; }
    } else {                                                    // adaptive_cleanup.rs:205-211
        h->ops_since_cleanup += d_ops;
        h->expired_count += d_hits;
        uint64_t len = h->h_counters.get()[C_REAL];
        if (adaptive_should_clean(h, now, len)) {               // cleanup(): :173-203
            int rc = do_sweep(h, now_ns, &removed);
            if (rc) return rc;
            if (removed == 0 && h->expired_count == 0) {
                __int128 d = h->cur_interval * 2;
                h->cur_interval = d < h->max_interval ? d : h->max_interval;
            } else if ((double)removed > (double)len * 0.5) {
                __int128 d = h->cur_interval / 2;
                h->cur_interval = d > h->min_interval ? d : h->min_interval;
            }
            h->last_removed = removed;
            h->last_total = len;
            h->next_cleanup = now + h->cur_interval;
            h->expired_count = 0;
            h->ops_since_cleanup = 0;
        }
    }
    return GCRA_OK;
}

// the cluster kernel: cluster dimension given at launch (cudaLaunchKernelEx)
template <bool BY_ROW, bool R16>
static int launch_giant(gcra_engine *h, Scratch &sc, const u64 *src, const OutMap &om, uint32_t n_max, cudaStream_t st) {
    cudaLaunchConfig_t cfg = {};
    // 16 clusters, or fewer when the batch cannot hold that many giant runs
    const uint32_t clusters = std::max<uint32_t>(std::min<uint32_t>(16, n_max / GIANT_RUN_MIN), 1);
    cfg.gridDim = dim3(clusters * CLUSTER_CTAS);
    cfg.blockDim = dim3(LONG_THREADS);
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CLUSTER_CTAS;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (CLUSTER_CTAS > 8) {
        static bool once = false;
        if (!once) { cudaFuncSetAttribute(decide_runs_kernel<CLUSTER_CTAS, BY_ROW, R16>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1); once = true; }
    }
    CK(cudaLaunchKernelEx(&cfg, decide_runs_kernel<CLUSTER_CTAS, BY_ROW, R16>, h->tab.view, (const u64 *)src, (const Req *)sc.drec.get(), om,
                          (const LongRun *)sc.giant_runs.get(), (const u32 *)(sc.long_count.get() + 1)));
    return GCRA_OK;
}

static BatchView single_view(const void *d_req, gcra_result *d_res, uint32_t n) {
    BatchView v{};
    v.req0 = (const unsigned char *)d_req;
    v.res0 = d_res;
    v.n = n;
    v.nseg = 1;
    v.cap_shift = 31;
    return v;
}

// stable LSD radix sort of `n` (host count) or `*n_dev` (device count) keys on the slot bits; returns the buffer
// that holds the sorted keys.  One digit-count launch, then one sweep launch per pass.
static int enqueue_sort(gcra_engine *h, Scratch &sc, uint32_t n_max, const u32 *n_dev, cudaStream_t st, u64 **sorted_out) {
    const uint32_t bits = h->tab.view.slot_bits;
    const uint32_t passes = (bits + SORT_MAX_BITS - 1) / SORT_MAX_BITS;
    const uint32_t tiles = (n_max + SORT_TILE - 1) / SORT_TILE;
    // With a device count (the residue of the index-order pipeline, usually a small part of n_max) both grids are
    // fixed at one CTA per SM: the sweep CTAs take tiles until the count's run out, and the kernels leave room for
    // the other stages' kernels that run beside the tail.  An empty count leaves the keys where they are and makes no
    // CTA wait.
    const uint32_t cap = n_dev ? h->sms : 2 * h->sms;
    const uint32_t sgrid = std::max<uint32_t>(n_dev ? std::min(tiles, h->sms) : tiles, 1);
    const uint32_t hgrid = std::max<uint32_t>(std::min<uint32_t>((n_max + 8 * TILE_THREADS - 1) / (8 * TILE_THREADS), cap), 1);
    u32 *ws = sc.sort_ws.get();
    CK(cudaMemsetAsync(ws, 0, sort_ws_words(passes, tiles) * sizeof(u32), st));
    sort_digits_kernel<<<hgrid, TILE_THREADS, 0, st>>>(sc.keys_a.get(), n_max, n_dev, bits, passes, ws);
    h->launches++;
    u64 *src = sc.keys_a.get(), *dst = sc.keys_b.get();
    uint32_t shift = 32;
    for (uint32_t p = 0; p < passes; p++) {
        const uint32_t pb = sort_pass_bits(bits, passes, p);
        sort_sweep_kernel<<<sgrid, TILE_THREADS, 0, st>>>(src, dst, n_max, n_dev, shift, pb, ws + SW_HIST + p * SORT_MAX_DIGITS,
                                                          ws + SW_TICKETS + p, ws + SW_STATUS + (size_t)p * tiles * SORT_MAX_DIGITS);
        h->launches++;
        std::swap(src, dst);
        shift += pb;
    }
    *sorted_out = src;
    return GCRA_OK;
}

// The one place where a batch's run-time row format picks kernel instantiations: calls f(F) with F =
// std::integral_constant<int, fmt>, so that `kernel<F>` and `Rows<F>` name the ones for `fmt`.
template <typename Fn>
static auto with_fmt(int fmt, Fn &&f) {
    if (fmt == FMT_16_16) return f(std::integral_constant<int, FMT_16_16>{});
    if (fmt == FMT_16_32) return f(std::integral_constant<int, FMT_16_32>{});
    return f(std::integral_constant<int, FMT_48_32>{});
}

template <bool BY_ROW, bool R16>
static int enqueue_decide_sorted_t(gcra_engine *h, Scratch &sc, uint32_t n_max, const u32 *n_dev, const u64 *src,
                                   const OutMap &om, cudaStream_t st) {
    // (sort pipeline: the work-list counters were cleared at the end of the front half, off this stream)
    if (BY_ROW) CK(cudaMemsetAsync(sc.long_count.get(), 0, 2 * sizeof(u32), st));
    const uint32_t warps = (n_max + 31) / 32;
    uint32_t grid = (warps + DECIDE_THREADS / 32 - 1) / (DECIDE_THREADS / 32);
    if (n_dev) grid = std::min<uint32_t>(grid, 4 * h->sms);
    auto decide = [&]() {   // everything but the hot runs
        decide_kernel<BY_ROW, R16><<<grid, DECIDE_THREADS, 0, st>>>(h->tab.view, src, sc.drec.get(), n_max, n_dev, om);
        h->launches++;
    };
    if (n_max < LONG_RUN_MIN) {   // no run can be hot
        decide();
        return GCRA_OK;
    }
    // The hot runs are listed first, so that their kernels run beside the decide of everything else instead of
    // after it.  Each goes to a side stream of the highest priority (fork/join with events): the cluster kernel
    // first, it holds the longest chains.  The three kernels touch disjoint slots and result rows.
    list_runs_kernel<<<grid, DECIDE_THREADS, 0, st>>>(h->tab.view, src, n_max, n_dev, sc.long_runs.get(), sc.giant_runs.get(), sc.long_count.get());
    h->launches++;
    CK(cudaEventRecord(sc.ev_fork.get(), st));
    if (n_max >= GIANT_RUN_MIN) {
        CK(cudaStreamWaitEvent(h->aux2_stream.get(), sc.ev_fork.get(), 0));
        RC((launch_giant<BY_ROW, R16>(h, sc, src, om, n_max, h->aux2_stream.get())));   // hottest keys: one cluster per run
        CK(cudaEventRecord(sc.ev_join_giant.get(), h->aux2_stream.get()));
        h->launches++;
    }
    // (at most n_max / LONG_RUN_MIN runs: no more CTAs than that)
    const uint32_t long_grid = std::min<uint32_t>(h->sms, n_max / LONG_RUN_MIN);
    CK(cudaStreamWaitEvent(h->aux_stream.get(), sc.ev_fork.get(), 0));
    decide_runs_kernel<1, BY_ROW, R16><<<long_grid, LONG_THREADS, 0, h->aux_stream.get()>>>(h->tab.view, src, sc.drec.get(), om, sc.long_runs.get(),
                                                                                          sc.long_count.get());
    CK(cudaEventRecord(sc.ev_join.get(), h->aux_stream.get()));
    h->launches++;
    decide();
    CK(cudaStreamWaitEvent(st, sc.ev_join.get(), 0));
    if (n_max >= GIANT_RUN_MIN) CK(cudaStreamWaitEvent(st, sc.ev_join_giant.get(), 0));
    return GCRA_OK;
}

// the warp-cooperative compare-and-update over sorted keys + the hot-run kernels, writing result rows of format `fmt`
static int enqueue_decide_sorted(gcra_engine *h, Scratch &sc, uint32_t n_max, const u32 *n_dev, const u64 *src,
                                 const OutMap &om, int fmt, cudaStream_t st) {
    return with_fmt(fmt, [&](auto F) {
        return om.by_row ? enqueue_decide_sorted_t<true, Rows<F>::R16>(h, sc, n_max, n_dev, src, om, st)
                         : enqueue_decide_sorted_t<false, Rows<F>::R16>(h, sc, n_max, n_dev, src, om, st);
    });
}

// every set's per-row buffers of the index-order pipeline, for batches of up to `rows` row ids (never shrinking), made
// for all sets before any set's are replaced.  The caller makes sure that no batch in flight uses the old ones.
static int alloc_index_scratch(gcra_engine *h, uint32_t rows) {
    if (rows <= h->scr[0].rows_alloc) return GCRA_OK;
    const uint32_t max_tiles = std::max<uint32_t>(h->max_tiles, (rows + TILE_THREADS - 1) / TILE_THREADS);
    struct { DevBuf<u32> slot_arr; DevBuf<unsigned char> flags; DevBuf<u64> ctrl_block; } fresh[gcra_engine::N_SCR];
    for (auto &f : fresh) {
        CK(f.slot_arr.make(rows));
        CK(f.flags.make(rows));
        CK(f.ctrl_block.make((size_t)max_tiles + 1));
    }
    for (int k = 0; k < gcra_engine::N_SCR; k++) {
        Scratch &sc = h->scr[k];
        sc.slot_arr = std::move(fresh[k].slot_arr);
        sc.flags = std::move(fresh[k].flags);
        sc.ctrl_block = std::move(fresh[k].ctrl_block);
        sc.rows_alloc = rows;
    }
    h->max_tiles = max_tiles;
    return GCRA_OK;
}

// metrics bridge: count this batch's denied rows per key.  A single-segment batch has its request and result rows
// here and a host-known row count; a segmented one (the peer-memory tick, 48-byte requests and 32-byte results only)
// has its results in the senders' outboxes and its row counts on the device: a persistent grid over the real tiles.
static int enqueue_denied(gcra_engine *h, const BatchView &v, int fmt, cudaStream_t st) {
    if (!h->denied_max) return GCRA_OK;
    if (v.nseg != 1) {
        if (fmt != FMT_48_32) { h->err = "a segmented batch counts denied rows of 48-byte requests only"; return GCRA_INTERNAL; }
        const uint32_t tiles = (uint32_t)((((uint64_t)v.nseg << v.cap_shift) + TILE_THREADS - 1) / TILE_THREADS);
        denied_count_seg_kernel<<<std::min(tiles, h->grid_denied_seg), TILE_THREADS, 0, st>>>(v, h->denied);
    } else {
        if (v.n == 0) return GCRA_OK;
        const uint32_t tiles = (v.n + TILE_THREADS - 1) / TILE_THREADS;
        with_fmt(fmt, [&](auto F) { denied_count_kernel<F><<<tiles, TILE_THREADS, 0, st>>>(v.req0, v.res0, v.n, h->denied); });
    }
    h->launches++;
    CK(cudaGetLastError());
    return GCRA_OK;
}

static bool use_index_path(const gcra_engine *h, uint32_t n) {
    // A performance choice only: both pipelines are exact at any size (the index-order pipeline's batch counters
    // hold any batch's row count, gcra_index_path.cuh).  Single batches above 2^21 rows take the sort pipeline.
    return h->index_min != 0 && n >= h->index_min && n <= (1u << 21);
}

static uint32_t view_max_rows(const BatchView &v) { return v.nseg == 1 ? v.n : (v.nseg << v.cap_shift); }

// Stage 1 of a batch.  Independent of the later stages of EARLIER batches: it only claims empty slots (a CAS on
// the keys array; it never touches the state array), which no earlier batch's decide kernels touch.
//   sort pipeline         ingest (validate, derive, probe/claim) + stable sort by slot
//   index-order pipeline  pass A (probe) + pass A' (batch bitmap)
static int enqueue_front(gcra_engine *h, Scratch &sc, const BatchView &v, bool index_path, int fmt, int64_t now_batch,
                         cudaStream_t st, bool timed, u64 **sorted_out) {
    if (timed) CK(cudaEventRecord(h->ev[0].get(), st));
    *sorted_out = nullptr;
    if (index_path) {
        const uint32_t rows = view_max_rows(v);
        const uint32_t tiles = (rows + TILE_THREADS - 1) / TILE_THREADS;
        const uint32_t grid = std::min<uint32_t>(tiles, h->grid_probe[fmt]);    // persistent, software-pipelined CTAs
        CK(cudaMemsetAsync(sc.ctrl_block.get(), 0, ((size_t)h->max_tiles + 1) * sizeof(u64), st));
        if (timed) CK(cudaEventRecord(h->evd[0].get(), st));
        with_fmt(fmt, [&](auto F) {
            probe_kernel<F><<<grid, TILE_THREADS, 0, st>>>(h->tab.view, v, h->d_pol.get(), h->npol, now_batch, sc.slot_arr.get(), sc.bitmap.get(),
                                                           h->bm_mask, h->prefetch_state);
        });
        if (timed) CK(cudaEventRecord(h->evd[1].get(), st));
        h->launches += 1;
        if (timed) { CK(cudaEventRecord(h->ev[1].get(), st)); CK(cudaEventRecord(h->evd[2].get(), st)); }
        return GCRA_OK;
    }
    const uint32_t n = v.n;
    const uint32_t tiles = (n + TILE_THREADS - 1) / TILE_THREADS;
    with_fmt(fmt, [&](auto F) {
        ingest_kernel<F><<<tiles, TILE_THREADS, 0, st>>>(h->tab.view, v.req0, h->d_pol.get(), h->npol, now_batch, n, sc.drec.get(),
                                                         sc.keys_a.get(), v.res0);
    });
    h->launches++;
    if (timed) CK(cudaEventRecord(h->ev[1].get(), st));
    RC(enqueue_sort(h, sc, n, nullptr, st, sorted_out));
    if (timed) CK(cudaEventRecord(h->ev[2].get(), st));
    CK(cudaMemsetAsync(sc.long_count.get(), 0, 2 * sizeof(u32), st));   // hot-run work lists of this batch's decide kernels
    return GCRA_OK;
}

// Stage 2 of an index-order batch: pass B (decide in batch order) + pass C (resolve).  Batches' stages 2 run
// strictly in submission order.  `next` is the scratch set the NEXT batch will use: pass C leaves the PEND bits
// of this batch's residue keys in its bitmap.  This set's own bitmap is cleared for its next use afterwards.
static int enqueue_mid_index(gcra_engine *h, Scratch &sc, Scratch &next, const BatchView &v, int fmt, int64_t now_batch,
                             bool honour_pend, cudaStream_t st, bool timed) {
    const u32 hp = honour_pend ? 1u : 0u;
    if (++h->epoch == 0) {
        // the 32-bit batch epoch wrapped: forget every mark (once per 4 G batches)
        CK(cudaMemsetAsync(h->tab.view.mark, 0xff, h->tab.slots() * sizeof(u64), st));
        h->epoch = 1;
    }
    const uint32_t rows = view_max_rows(v);
    const uint32_t grid = std::min<uint32_t>((rows + TILE_THREADS - 1) / TILE_THREADS, h->grid_decide[fmt]);   // persistent CTAs
    const uint32_t rgrid = std::min<uint32_t>((rows + RES_TILE - 1) / RES_TILE + v.nseg, 6 * h->sms);
    u32 *ctrl = reinterpret_cast<u32 *>(sc.ctrl_block.get());
    u64 *status = sc.ctrl_block.get() + 1;
    RC(with_fmt(fmt, [&](auto F) {
        decide_index_kernel<F><<<grid, TILE_THREADS, 0, st>>>(h->tab.view, v, h->d_pol.get(), h->npol, now_batch, sc.slot_arr.get(), sc.bitmap.get(),
                                                              sc.pend.get(), h->bm_mask, sc.flags.get(), h->epoch, hp, h->dbg);
        if (timed) CK(cudaEventRecord(h->evd[3].get(), st));
        resolve_kernel<F><<<rgrid, TILE_THREADS, 0, st>>>(h->tab.view, v, h->d_pol.get(), h->npol, now_batch, sc.slot_arr.get(), h->bm_mask,
                                                          sc.flags.get(), h->epoch, ctrl, status, sc.keys_a.get(), next.pend.get(),
                                                          sc.h_nres.get(), h->max_batch);
        return GCRA_OK;
    }));
    h->launches += 2;
    h->n_index_batches++;
    if (timed) CK(cudaEventRecord(h->evd[4].get(), st));
    // (pass C wrote the residue size of this batch to sc.h_nres.get(), mapped pinned host memory: read, once ev_mid has
    // completed, when later batches are submitted)
    sc.nres_rows = std::min<uint32_t>(rows, h->max_batch);
    sc.nres_counted = false;
    if (timed) CK(cudaEventRecord(h->ev[2].get(), st));
    CK(cudaGetLastError());
    return GCRA_OK;
}

// Stage 3 of an index-order batch: the residue (requests behind the first state change of their key, and
// requests deferred because the previous batch's tail still owned their key) through the sort pipeline; its
// size only exists on the device.  Tails run strictly in submission order.
static int enqueue_tail_index(gcra_engine *h, Scratch &sc, const BatchView &v, int fmt, int64_t now_batch, cudaStream_t st,
                              bool timed) {
    const u32 *n_res = reinterpret_cast<const u32 *>(sc.ctrl_block.get()) + RC_NRES;
    const uint32_t n_max = std::min<uint32_t>(view_max_rows(v), h->max_batch);
    u64 *rs = nullptr;
    // this set's bitmap has been read for the last time (pass C): cleared here, off stage 2's stream, for its next
    // use (pass A' of the batch that takes this set again, and the PEND bits the batch before that one leaves)
    CK(cudaMemsetAsync(sc.bitmap.get(), 0, h->bm_words * sizeof(u32), st));
    CK(cudaMemsetAsync(sc.pend.get(), 0, h->pend_words * sizeof(u32), st));   // (the bits the previous batch left: read by pass B)
    if (timed) CK(cudaEventRecord(h->evd[5].get(), st));
    RC(enqueue_sort(h, sc, n_max, n_res, st, &rs));
    if (timed) CK(cudaEventRecord(h->evd[6].get(), st));
    OutMap om{};
    om.out = nullptr;
    om.by_row = 1;
    om.compact = req_bytes(fmt) == sizeof(gcra_request16) ? 1 : 0;
    om.view = v;
    om.pol = h->d_pol.get();
    om.npol = h->npol;
    om.now_batch = now_batch;
    RC(enqueue_decide_sorted(h, sc, n_max, n_res, rs, om, fmt, st));
    if (timed) { CK(cudaEventRecord(h->ev[3].get(), st)); h->ev_valid = true; CK(cudaEventRecord(h->evd[7].get(), st)); h->evd_valid = true; }
    CK(cudaGetLastError());
    return GCRA_OK;
}

struct Lanes { cudaStream_t front, mid, tail; };   // a batch's stages run on the engine's three streams (pipelined) or all on the caller's (serial)
struct BatchPlan { bool index_path, overlap; };    // which pipeline; may stage 2 (index-order) overlap the previous batch's tail

// The end of every batch, on the stream of its last stage, in this order.  The denied count comes before ev_back: a
// peer-memory tick publishes its results after ev_back (gcra_p2p_submit_finish), and from then on a sender may reuse
// the inbox and outbox rows the count reads.  Everything that follows the batch waits for ev_back (`*done`, the
// set's next use, order_after_batches), so only the copy of the occupancy counters is enqueued behind it.
static int finish_batch(gcra_engine *h, Scratch &sc, const BatchView &v, uint32_t n_rows, int fmt, cudaStream_t st, cudaEvent_t *done) {
    RC(enqueue_denied(h, v, fmt, st));
    CK(cudaEventRecord(sc.ev_back.get(), st));
    sc.back_recorded = true;
    if (done) *done = sc.ev_back.get();
    return snapshot_async(h, n_rows, st);
}

// The stages of one batch (any but a small serial batch) in scratch set `k`, each on its lane, then the end of the
// batch on the last one.  Two lanes that are the same stream hand over without an event.  Knows nothing of earlier
// batches: the caller has already enqueued, on the lanes, what this one has to wait for.
static int enqueue_stages(gcra_engine *h, uint32_t k, const BatchView &v, uint32_t n_rows, int fmt, int64_t now_batch,
                          BatchPlan plan, Lanes on, bool timed, cudaEvent_t *done) {
    Scratch &sc = h->scr[k];
    const uint32_t kn = (k + 1) % gcra_engine::N_SCR;         // the set the next batch takes
    u64 *sorted = nullptr;
    RC(enqueue_front(h, sc, v, plan.index_path, fmt, now_batch, on.front, timed, &sorted));
    if (on.mid != on.front) {
        CK(cudaEventRecord(sc.ev_front.get(), on.front));
        CK(cudaStreamWaitEvent(on.mid, sc.ev_front.get(), 0));
    }
    if (plan.index_path) {
        RC(enqueue_mid_index(h, sc, h->scr[kn], v, fmt, now_batch, plan.overlap, on.mid, timed));
        CK(cudaEventRecord(sc.ev_mid.get(), on.mid));         // on one lane as well: the residue feedback reads it
        sc.mid_recorded = true;
        if (on.tail != on.mid) CK(cudaStreamWaitEvent(on.tail, sc.ev_mid.get(), 0));
        RC(enqueue_tail_index(h, sc, v, fmt, now_batch, on.tail, timed));
    } else {
        // stage 2 of a sort-pipeline batch: the compare-and-update kernels over the sorted keys
        OutMap om{};                                          // (by_row = 0: a sorted key's payload is its batch index)
        om.out = v.res0;
        RC(enqueue_decide_sorted(h, sc, v.n, nullptr, sorted, om, fmt, on.mid));
        if (timed) { CK(cudaEventRecord(h->ev[3].get(), on.mid)); h->ev_valid = true; }
        CK(cudaGetLastError());
        sc.mid_recorded = false;                              // (no residue count from this batch)
    }
    h->pend_set = plan.index_path ? (int)kn : -1;             // pass C left this batch's PEND bits in the next set
    return finish_batch(h, sc, v, n_rows, fmt, plan.index_path ? on.tail : on.mid, done);
}

static int check_batch(gcra_engine *h, uint32_t n, int fmt) {
    if (n > h->max_batch) { h->err = "batch larger than max_batch"; return GCRA_INTERNAL; }
    if (req_bytes(fmt) == sizeof(gcra_request16) && h->npol == 0) { h->err = "no policy table registered"; return GCRA_INTERNAL; }
    return ensure_room(h, n);
}

// ---- one batch, everything on the caller's stream ------------------------------------------------
static int launch_batch(gcra_engine *h, uint32_t n, const void *d_req, int fmt, int64_t now_batch,
                        void *d_res_rows, cudaStream_t st, bool timed) {
    if (n == 0) return GCRA_OK;
    RC(check_batch(h, n, fmt));
    gcra_result *d_res = (gcra_result *)d_res_rows;     // (or gcra_result16 rows: see BatchView::res16_at)
    const uint32_t k = h->scr_next;
    h->scr_next = (h->scr_next + 1) % gcra_engine::N_SCR;
    const BatchView v = single_view(d_req, d_res, n);
    // after every earlier batch (some may be in flight on the engine's streams), which also frees this scratch set
    RC(order_after_batches(h, st));
    RC(after_capture(h, st));
    static const bool no_small = getenv("GCRA_NO_SMALL") && atoi(getenv("GCRA_NO_SMALL"));   // A/B switch for tools/latency_probe.py
    if (n <= SMALL_MAX && !no_small) {
        // small batch (a single rate_limit call, a lightly loaded actor): one CTA does ingest, ordering and
        // the compare-and-update in a single launch
        Scratch &sc = h->scr[k];
        if (timed) { CK(cudaEventRecord(h->ev[0].get(), st)); CK(cudaEventRecord(h->ev[1].get(), st)); CK(cudaEventRecord(h->ev[2].get(), st)); }
        with_fmt(fmt, [&](auto F) {
            small_batch_kernel<F><<<1, TILE_THREADS, 0, st>>>(h->tab.view, d_req, h->d_pol.get(), h->npol, now_batch, n, sc.drec.get(), d_res);
        });
        h->launches++;
        if (timed) { CK(cudaEventRecord(h->ev[3].get(), st)); h->ev_valid = true; }
        CK(cudaGetLastError());
        RC(finish_batch(h, sc, v, n, fmt, st, nullptr));
    } else RC(enqueue_stages(h, k, v, n, fmt, now_batch, {use_index_path(h, n), false}, {st, st, st}, timed, nullptr));
    h->pend_set = -1;          // everything of this batch is ordered on `st`: the next batch waits for all of it
    return GCRA_OK;
}

// ---- one batch, pipelined over the engine's streams --------------------------------------------------
// How the next pipelined batch, in scratch set `k`, runs.  A host state machine over the residue counts that earlier
// batches' pass C reported: it queries events and enqueues nothing.
static BatchPlan plan_pipelined(gcra_engine *h, uint32_t k, const BatchView &v, uint32_t n_rows) {
    // residue feedback: the newest pass-C count that has reached the host
    bool residue_large = false;
    for (int back = 1; back < gcra_engine::N_SCR; back++) {
        Scratch &os = h->scr[(k + gcra_engine::N_SCR - back) % gcra_engine::N_SCR];
        if (!os.mid_recorded || cudaEventQuery(os.ev_mid.get()) != cudaSuccess) continue;
        if (!os.nres_counted) { h->residue_seen += *os.h_nres.get(); h->residue_batches_seen++; os.nres_counted = true; }
        h->last_nres = *os.h_nres.get();
        h->last_nres_rows = os.nres_rows;
        residue_large = (uint64_t)*os.h_nres.get() * 8 > os.nres_rows;
        break;
    }
    bool ip = v.nseg > 1 || use_index_path(h, n_rows);
    if (ip && v.nseg == 1 && h->adaptive) {
        // Which pipeline?  The index-order pipeline wins while most requests are decided in passes B and C; when
        // more than a quarter of a batch went through the sorted tail (keys spending a burst: every request
        // changes the state), sorting everything once is cheaper: the next 31 batches take the sort pipeline,
        // then the index-order pipeline is tried again.
        if (h->sort_hold > 0) { h->sort_hold--; ip = false; }
        else if (h->last_nres_rows && (uint64_t)h->last_nres * 4 > h->last_nres_rows) {
            h->sort_hold = 31; h->last_nres = 0; h->last_nres_rows = 0; ip = false; h->n_path_switches++;
        }
    }
    // May stage 2 of this batch overlap the tail of the batch submitted just before?  Only if that batch left its
    // PEND bits in this set's pend bitmap.  Keys the tail owns stay deferred for as long as they keep appearing
    // (their requests go from tail to tail), so the overlap is given up -- stage 2 waits for every tail and ignores
    // the PEND bits -- whenever the residue reported by an earlier batch has grown beyond 1/8 of its rows, and
    // every 64 batches.
    bool overlap = ip && h->pend_set == (int)k;
    if (ip) {
        if (residue_large && h->since_drain >= 2) overlap = false;
        if (h->since_drain >= 64) overlap = false;
        if (!overlap) { if (h->pend_set == (int)k) h->n_drains++; h->since_drain = 0; } else h->since_drain++;
    }
    return {ip, overlap};
}

// index-order pipeline: stage 1 (probe) of batch j+1 overlaps stage 2 (decide, resolve) of batch j and stage 3
// (the sorted residue) of batch j-1.  Stage 2 of batch j may run while the tail of batch j-1 is still at work
// because pass C of batch j-1 left PEND bits for exactly the keys that tail owns.  Sort pipeline: stage 1 =
// ingest + sort, stage 2 = decide, after every earlier batch has completely finished.
// `ready` (may be null) is an event after which the requests may be read; `*done` is set to an event after which
// the results are complete.
// room_reserved: the caller has made room in the table for n_rows already (ensure_room).
static int launch_pipelined_view(gcra_engine *h, const BatchView &v, uint32_t n_rows, int fmt, int64_t now_batch,
                                 cudaEvent_t ready, cudaEvent_t *done, bool room_reserved = false) {
    // 16-byte results are a single-GPU format: the multi-GPU ticks return 32-byte rows into peers' outboxes
    if (res_bytes(fmt) == sizeof(gcra_result16) && v.nseg != 1) { h->err = "16-byte results need a single-segment batch"; return GCRA_INTERNAL; }
    if (!room_reserved) RC(check_batch(h, n_rows, fmt));
    const uint32_t k = h->scr_next;
    h->scr_next = (h->scr_next + 1) % gcra_engine::N_SCR;
    const Lanes on = {h->front_stream.get(), h->back_stream.get(), h->tail_stream.get()};   // (all sets share one front stream, see gcra_create)
    if (ready) CK(cudaStreamWaitEvent(on.front, ready, 0));
    if (h->scr[k].back_recorded) CK(cudaStreamWaitEvent(on.front, h->scr[k].ev_back.get(), 0));   // scratch set free again
    RC(after_capture(h, on.front));                           // (the later stages follow this batch's front)
    const BatchPlan plan = plan_pipelined(h, k, v, n_rows);
    // stage 2 follows every earlier batch whole, but for the tail of the batch just before when it may overlap it
    const uint32_t prev = (k + gcra_engine::N_SCR - 1) % gcra_engine::N_SCR;
    for (uint32_t o = 0; o < gcra_engine::N_SCR; o++) {
        if (o == k || (o == prev && plan.overlap) || !h->scr[o].back_recorded) continue;
        CK(cudaStreamWaitEvent(on.mid, h->scr[o].ev_back.get(), 0));
    }
    return enqueue_stages(h, k, v, n_rows, fmt, now_batch, plan, on, false, done);
}

static int launch_pipelined(gcra_engine *h, uint32_t n, const void *d_req, int fmt, int64_t now_batch,
                            void *d_res, cudaEvent_t ready, cudaEvent_t *done) {
    if (n == 0) { if (done) *done = nullptr; return GCRA_OK; }
    return launch_pipelined_view(h, single_view(d_req, (gcra_result *)d_res, n), n, fmt, now_batch, ready, done);
}

// ---- the hash pass: key references -> the engine's key hashes, in place, on `st` --------------------------------
static int enqueue_hash_keys(gcra_engine *h, uint64_t n, void *d_rows, uint32_t row_bytes, const void *d_keys,
                             uint64_t keys_len, cudaStream_t st) {
    if (row_bytes != sizeof(gcra_request) && row_bytes != sizeof(gcra_request16)) {
        h->err = "row_bytes must be 48 or 16"; return GCRA_INTERNAL;
    }
    if (n > 0xffffffffULL) { h->err = "more than 2^32 - 1 rows"; return GCRA_INTERNAL; }
    if (n == 0) return GCRA_OK;
    hash_keys_kernel<<<(uint32_t)((n + TILE_THREADS - 1) / TILE_THREADS), TILE_THREADS, 0, st>>>(
        (unsigned char *)d_rows, (uint32_t)n, row_bytes, (const unsigned char *)d_keys, keys_len, h->hash_seed[0],
        h->hash_seed[1]);
    h->launches++;
    CK(cudaGetLastError());
    return GCRA_OK;
}

// CUDA loads a kernel's code lazily, at its FIRST launch, and that load may wait for running kernels.  The
// multi-GPU pipelines keep kernels running that wait for work other launches deliver (flags in peer memory), so a
// first launch behind such a kernel would stall until the wait gives up: load everything when the engine is made.
template <typename K>
static void preload(K kernel) {
    cudaFuncAttributes a;
    cudaFuncGetAttributes(&a, kernel);
}

static void preload_kernels() {
    for (int fmt = 0; fmt < FMT_COUNT; fmt++)
        with_fmt(fmt, [](auto F) {
            preload(ingest_kernel<F>); preload(small_batch_kernel<F>); preload(denied_count_kernel<F>);
            preload(probe_kernel<F>); preload(decide_index_kernel<F>); preload(resolve_kernel<F>);
        });
    preload(sort_digits_kernel); preload(sort_sweep_kernel);
    preload(decide_kernel<false, false>); preload(decide_kernel<true, false>);
    preload(decide_kernel<false, true>); preload(decide_kernel<true, true>); preload(list_runs_kernel);
    preload(decide_runs_kernel<1, false, false>); preload(decide_runs_kernel<CLUSTER_CTAS, false, false>);
    preload(decide_runs_kernel<1, true, false>); preload(decide_runs_kernel<CLUSTER_CTAS, true, false>);
    preload(decide_runs_kernel<1, false, true>); preload(decide_runs_kernel<CLUSTER_CTAS, false, true>);
    preload(decide_runs_kernel<1, true, true>); preload(decide_runs_kernel<CLUSTER_CTAS, true, true>);
    preload(sweep_kernel); preload(purge_kernel); preload(clear_slots_kernel); preload(rehash_kernel); preload(store_op_kernel);
    preload(route_count_kernel); preload(route_scan_kernel); preload(route_scatter_kernel); preload(route_unpermute_kernel);
    preload(p2p_scan_kernel); preload(p2p_scatter_kernel); preload(p2p_signal_req_kernel); preload(p2p_signal_res_kernel);
    preload(p2p_wait_kernel); preload(p2p_unpermute_kernel);
    preload(route_count_dev_kernel); preload(p2p_scatter_dev_kernel); preload(p2p_unpermute_dev_kernel);
    preload(snapshot_capture_kernel); preload(denied_count_seg_kernel); preload(hash_keys_kernel);
}

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

// everything gcra_create makes; on failure h->err says what failed and deleting `h` releases what was made
static int init_engine(gcra_engine *h, const gcra_config *cfg) {
    int ndev = 0;
    CK(cudaGetDeviceCount(&ndev));        // (this engine has no CPU path)
    if (cfg->device < 0 || cfg->device >= ndev) { h->err = "bad device ordinal"; return GCRA_INTERNAL; }
    h->device = cfg->device;
    CK(cudaSetDevice(h->device));
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device));
    if (sms <= 0) { h->err = "no streaming multiprocessors"; return GCRA_INTERNAL; }
    h->sms = (uint32_t)sms;
    if (const char *g = getenv("GCRA_L2_FETCH")) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)atoi(g));
    for (Stream *s : {&h->stream, &h->in_stream, &h->out_stream, &h->front_stream, &h->back_stream, &h->tail_stream})
        CK(s->make());
    // the hot-run kernels' streams: highest priority, so that their few CTAs are dispatched ahead of the decide
    // kernel's thousands that are launched after them
    int least_prio = 0, greatest_prio = 0;
    CK(cudaDeviceGetStreamPriorityRange(&least_prio, &greatest_prio));
    for (Stream *s : {&h->aux_stream, &h->aux2_stream}) CK(s->make(greatest_prio));
    for (Event *e : {&h->ev_ready, &h->ev_counters}) CK(e->make(cudaEventDisableTiming));
    for (Event &e : h->ev_snap) CK(e.make(cudaEventDisableTiming));
    for (Event &e : h->ev) CK(e.make(cudaEventDefault));         // (timed)
    for (Event &e : h->evd) CK(e.make(cudaEventDefault));
    for (Event &e : h->ev_sweep) CK(e.make(cudaEventDefault));
    h->max_batch = cfg->max_batch ? cfg->max_batch : (1u << 20);
    h->tight = (cfg->flags & GCRA_FLAG_TIGHT_TABLE) != 0;
    h->hash_seed[0] = cfg->hash_seed[0];
    h->hash_seed[1] = cfg->hash_seed[1];
    if (cfg->flags & GCRA_FLAG_RANDOM_SEED) {
        FILE *ur = fopen("/dev/urandom", "rb");
        const bool got = ur && fread(h->hash_seed, sizeof(h->hash_seed), 1, ur) == 1;
        if (ur) fclose(ur);
        if (!got) { h->err = "cannot read /dev/urandom for the hash seed"; return GCRA_INTERNAL; }
        h->hash_seed[0] |= 1;      // never (0, 0)
    }
    RC(make_table(h, cfg->capacity ? cfg->capacity : 1000, h->tab));   // DEFAULT_CAPACITY adaptive_cleanup.rs:10
    const size_t mb = h->max_batch;
    {
        // index-order pipeline: hashed batch counters (32 bits) and pend bits, 8 entries per row of the largest
        // batch (n distinct slots share their entry with probability ~1/8), 64 K .. 16 M entries
        uint32_t lg = ceil_log2(std::max<uint64_t>(8ULL * mb, 1ULL << 16));
        if (lg > 24) lg = 24;
        h->bm_mask = (1u << lg) - 1;
        h->bm_words = (size_t)1 << lg;            // one 32-bit counter per entry
        h->pend_words = (size_t)1 << (lg - 5);    // 1 bit per entry
        h->index_min = 32768;
        if (const char *g = getenv("GCRA_INDEX_MIN")) { h->index_min = (uint32_t)atoll(g); h->adaptive = false; }
        // tests only: the batch epoch to count on from, so that a test can cross the 32-bit wrap (which clears every
        // mark, enqueue_mid_index) in a few batches instead of 4 G
        if (const char *g = getenv("GCRA_EPOCH0")) h->epoch = (uint32_t)strtoull(g, nullptr, 0);
        if (cfg->flags & GCRA_FLAG_INDEX_PATH) { h->index_min = SMALL_MAX + 1; h->adaptive = false; }
        if (cfg->flags & GCRA_FLAG_SORT_PATH) { h->index_min = 0; h->adaptive = false; }
        if (const char *g = getenv("GCRA_ADAPTIVE")) h->adaptive = atoi(g) != 0;
        h->prefetch_state = 0;
        if (const char *g = getenv("GCRA_PREFETCH")) h->prefetch_state = atoi(g);
        for (int fmt = 0; fmt < FMT_COUNT; fmt++) {
            h->grid_probe[fmt] = 4 * h->sms;      // used when the occupancy query fails
            h->grid_decide[fmt] = 3 * h->sms;
            with_fmt(fmt, [&](auto F) {
                int nb = 0;
                if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, probe_kernel<F>, TILE_THREADS, 0) == cudaSuccess && nb > 0) h->grid_probe[fmt] = (uint32_t)(nb * sms);
                if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, decide_index_kernel<F>, TILE_THREADS, 0) == cudaSuccess && nb > 0) h->grid_decide[fmt] = (uint32_t)(nb * sms);
            });
        }
        h->grid_denied_seg = 4 * h->sms;
        {
            int nb = 0;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, denied_count_seg_kernel, TILE_THREADS, 0) == cudaSuccess && nb > 0) h->grid_denied_seg = (uint32_t)(nb * sms);
        }
        // tuning: CTAs per SM of the persistent kernels (fewer leave room for the other stages' kernels)
        if (const char *g = getenv("GCRA_CTAS_PROBE")) { uint32_t c = (uint32_t)atoi(g) * sms; if (c) for (auto &x : h->grid_probe) x = std::min(x, c); }
        if (const char *g = getenv("GCRA_CTAS_DECIDE")) { uint32_t c = (uint32_t)atoi(g) * sms; if (c) for (auto &x : h->grid_decide) x = std::min(x, c); }
    }
    CK(h->d_req.make(mb));
    CK(h->d_res.make(mb));
    CK(h->route_counts.make((size_t)ROUTE_MAX_SHARDS * ((mb + TILE_THREADS - 1) / TILE_THREADS)));
    CK(h->d_op.make(2));
    CK(h->h_op.make(2));
    CK(h->h_counters.make(C_COUNT));
    CK(h->h_snap.make((size_t)gcra_engine::N_SNAP * C_COUNT));
    if (h->max_batch > SORT_MAX_COUNT) { h->err = "max_batch must be below 2^30"; return GCRA_INTERNAL; }   // (the sort's 30-bit counts)
    for (Scratch &sc : h->scr) {
        CK(sc.drec.make(mb));
        CK(sc.keys_a.make(mb));
        CK(sc.keys_b.make(mb));
        CK(sc.sort_ws.make(sort_ws_words(SORT_MAX_PASSES, (uint32_t)((mb + SORT_TILE - 1) / SORT_TILE))));
        CK(sc.long_runs.make(mb / LONG_RUN_MIN + 1));
        CK(sc.giant_runs.make(mb / GIANT_RUN_MIN + 1));
        CK(sc.long_count.make(2));
        for (Event *e : {&sc.ev_front, &sc.ev_back, &sc.ev_mid, &sc.ev_fork, &sc.ev_join, &sc.ev_join_giant})
            CK(e->make(cudaEventDisableTiming));
        CK(sc.h_nres.make(1));
        *sc.h_nres.get() = 0;
        CK(sc.bitmap.make(h->bm_words));
        CK(sc.pend.make(h->pend_words));
        CK(cudaMemsetAsync(sc.bitmap.get(), 0, h->bm_words * sizeof(u32), h->stream.get()));   // from then on cleared after every use
        CK(cudaMemsetAsync(sc.pend.get(), 0, h->pend_words * sizeof(u32), h->stream.get()));
    }
    RC(alloc_index_scratch(h, h->max_batch));
    memset(h->h_counters.get(), 0, C_COUNT * sizeof(u64));
    // store policy, defaults as in the reference constructors
    h->kind = cfg->store_kind;
    __int128 created = cfg->created_ns;
    if (h->kind == GCRA_STORE_PERIODIC) {
        h->cleanup_interval = (__int128)(cfg->p0 ? cfg->p0 : 60) * NS_PER_S;       // periodic.rs:12
        h->next_cleanup = created + h->cleanup_interval;
    } else if (h->kind == GCRA_STORE_PROBABILISTIC) {
        h->cleanup_modulo = cfg->p0 ? cfg->p0 : 1000;                               // probabilistic.rs:12
    } else if (h->kind == GCRA_STORE_ADAPTIVE) {
        h->min_interval = (__int128)(cfg->p0 ? cfg->p0 : 1) * NS_PER_S;            // adaptive_cleanup.rs:12-15
        h->max_interval = (__int128)(cfg->p1 ? cfg->p1 : 300) * NS_PER_S;
        h->max_ops = cfg->p2 ? cfg->p2 : 100000;
        h->cur_interval = 5 * NS_PER_S;
        h->next_cleanup = created + 5 * NS_PER_S;
    }
    preload_kernels();
    CK(cudaStreamSynchronize(h->stream.get()));
    return GCRA_OK;
}

int32_t gcra_create(const gcra_config *cfg, gcra_engine **out) {
    if (!cfg || !out) return GCRA_INTERNAL;
    *out = nullptr;
    std::unique_ptr<gcra_engine> h(new gcra_engine());
    if (init_engine(h.get(), cfg) != GCRA_OK) {
        fprintf(stderr, "gcra_create: %s\n", h->err.c_str());
        return GCRA_INTERNAL;
    }
    *out = h.release();
    return GCRA_OK;
}

// the synchronize comes first: no member is released under work still running
void gcra_destroy(gcra_engine *h) {
    if (!h) return;
    if (h->job && h->job->writer.joinable()) h->job->writer.join();    // a background save finishes its file first
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    delete h;
}

const char *gcra_last_error(gcra_engine *h) { return h ? h->err.c_str() : "null handle"; }

// (both hashes are defined once, for the host and the hash pass, in gcra_device.cuh)
uint64_t gcra_hash_key(const void *key, uint64_t len) {
    return hash_key_unkeyed(KeyBytes{(const unsigned char *)key}, len);
}

uint64_t gcra_hash_key_seeded(const void *key, uint64_t len, uint64_t k0, uint64_t k1) {
    return hash_key_siphash(KeyBytes{(const unsigned char *)key}, len, k0, k1);
}

// the identity the engine's own string-keyed entry points give a key: keyed when the engine has a seed
static uint64_t engine_hash(const gcra_engine *h, const void *key, uint64_t len) {
    return hash_key_engine(KeyBytes{(const unsigned char *)key}, len, h->hash_seed[0], h->hash_seed[1]);
}

uint64_t gcra_engine_hash_key(gcra_engine *h, const void *key, uint64_t len) { return engine_hash(h, key, len); }

void gcra_get_hash_seed(gcra_engine *h, uint64_t out[2]) { out[0] = h->hash_seed[0]; out[1] = h->hash_seed[1]; }

void gcra_hash_key_ids(const void *prefix, uint64_t prefix_len, const uint64_t *ids, uint64_t n, uint64_t *out) {
    char buf[96];
    if (prefix_len > 64) prefix_len = 64;
    memcpy(buf, prefix, prefix_len);
    for (uint64_t i = 0; i < n; i++) {
        char tmp[24];
        int k = 0;
        uint64_t v = ids[i];
        do { tmp[k++] = (char)('0' + v % 10); v /= 10; } while (v);
        for (int j = 0; j < k; j++) buf[prefix_len + j] = tmp[k - 1 - j];
        out[i] = gcra_hash_key(buf, prefix_len + k);
    }
}

int32_t gcra_derive_params(int64_t max_burst, int64_t count, int64_t period, int64_t *ei, int64_t *dvt) {
    i64 a = 0, b = 0;
    int st = derive_params(max_burst, count, period, &a, &b);
    if (ei) *ei = a;
    if (dvt) *dvt = b;
    return st;
}

static int store_op(gcra_engine *h, int op, uint64_t key_hash, int64_t a, int64_t b, uint64_t ttl, int64_t now) {
    CK(cudaSetDevice(h->device));
    // the table encodes 'no state' as a negative expiry (has_state): times before the epoch are outside its domain
    if (op != 3 && now < 0) { h->err = "pre-epoch time is not supported"; return GCRA_INTERNAL; }
    if (op == 2) { int rc = ensure_room(h, 1); if (rc) return rc; }
    // a Store-trait call reads / writes a slot's state
    RC(order_after_batches(h, h->stream.get()));
    RC(after_capture(h, h->stream.get()));
    store_op_kernel<<<1, 1, 0, h->stream.get()>>>(h->tab.view, op, stored_key(key_hash), a, b, ttl, now, h->d_op.get());
    h->launches++;
    CK(cudaMemcpyAsync(h->h_op.get(), h->d_op.get(), 2 * sizeof(StoreOpResult), cudaMemcpyDeviceToHost, h->stream.get()));
    CK(cudaStreamSynchronize(h->stream.get()));
    return GCRA_OK;
}

static int policy_before_mutation(gcra_engine *h, int64_t now_ns) {
    // the reference's mutating ops start with maybe_clean_expired(now) (adaptive_cleanup.rs:229,261)
    int rc = refresh_counters(h, true);
    if (rc) return rc;
    return apply_policy(h, now_ns);
}

int32_t gcra_store_get(gcra_engine *h, const void *key, uint64_t len, int64_t now_ns, int64_t *value,
                       uint8_t *found) {
    int rc = store_op(h, 0, engine_hash(h, key, len), 0, 0, 0, now_ns);
    if (rc) return rc;
    if (found) *found = (uint8_t)h->h_op.get()[0].flag;
    if (value) *value = h->h_op.get()[0].value;
    return GCRA_OK;
}

int32_t gcra_store_cas(gcra_engine *h, const void *key, uint64_t len, int64_t old_value, int64_t new_value,
                       uint64_t ttl_ns, int64_t now_ns, uint8_t *swapped) {
    int rc = policy_before_mutation(h, now_ns);
    if (rc) return rc;
    rc = store_op(h, 1, engine_hash(h, key, len), old_value, new_value, ttl_ns, now_ns);
    if (rc) return rc;
    if (swapped) *swapped = (uint8_t)h->h_op.get()[0].flag;
    return GCRA_OK;
}

int32_t gcra_store_set_nx(gcra_engine *h, const void *key, uint64_t len, int64_t value, uint64_t ttl_ns,
                          int64_t now_ns, uint8_t *stored) {
    int rc = policy_before_mutation(h, now_ns);
    if (rc) return rc;
    rc = store_op(h, 2, engine_hash(h, key, len), value, 0, ttl_ns, now_ns);
    if (rc) return rc;
    if (h->h_op.get()[0].status) { h->err = "table full"; return GCRA_INTERNAL; }
    if (stored) *stored = (uint8_t)h->h_op.get()[0].flag;
    return GCRA_OK;
}

int32_t gcra_rate_limit_batch_device(gcra_engine *h, uint64_t n, const gcra_request *d_req, gcra_result *d_res,
                                     void *stream) {
    CK(cudaSetDevice(h->device));
    return launch_batch(h, (uint32_t)n, d_req, FMT_48_32, 0, d_res, stream ? (cudaStream_t)stream : h->stream.get(), true);
}

int32_t gcra_rate_limit_batch16_device(gcra_engine *h, uint64_t n, const gcra_request16 *d_req, int64_t now_ns,
                                       gcra_result *d_res, void *stream) {
    CK(cudaSetDevice(h->device));
    return launch_batch(h, (uint32_t)n, d_req, FMT_16_32, now_ns, d_res, stream ? (cudaStream_t)stream : h->stream.get(), true);
}

int32_t gcra_rate_limit_batch16_r16_device(gcra_engine *h, uint64_t n, const gcra_request16 *d_req, int64_t now_ns,
                                           gcra_result16 *d_res, void *stream) {
    CK(cudaSetDevice(h->device));
    return launch_batch(h, (uint32_t)n, d_req, FMT_16_16, now_ns, d_res, stream ? (cudaStream_t)stream : h->stream.get(), true);
}

int32_t gcra_rate_limit_batch_device_pipelined(gcra_engine *h, uint64_t n, const gcra_request *d_req,
                                               gcra_result *d_res, void *ready_stream) {
    CK(cudaSetDevice(h->device));
    cudaEvent_t ready = nullptr;
    if (ready_stream) {
        CK(cudaEventRecord(h->ev_ready.get(), (cudaStream_t)ready_stream));
        ready = h->ev_ready.get();
    }
    return launch_pipelined(h, (uint32_t)n, d_req, FMT_48_32, 0, d_res, ready, nullptr);
}

int32_t gcra_pipeline_join(gcra_engine *h, void *stream) {
    CK(cudaSetDevice(h->device));
    return stream ? order_after_batches(h, (cudaStream_t)stream) : wait_for_batches(h);
}

struct KeyArena { const void *keys; uint64_t len; };

// arena != null: the rows hold key references into the host arena, which goes to the device first; the hash pass
// runs on every chunk before its batch
static int host_batch(gcra_engine *h, uint64_t n, const void *req, int fmt, int64_t now_batch, void *res,
                      const KeyArena *arena = nullptr) {
    CK(cudaSetDevice(h->device));
    const size_t rsz = req_bytes(fmt), ressz = res_bytes(fmt);
    const uint64_t keys_len = arena ? arena->len : 0;
    if (keys_len > h->d_keys_cap) {
        DevBuf<unsigned char> grown;              // (a failed call keeps the old arena)
        CK(cudaStreamSynchronize(h->stream.get()));
        CK(grown.make(keys_len));
        h->d_keys = std::move(grown);
        h->d_keys_cap = keys_len;
    }
    if (keys_len) CK(cudaMemcpyAsync(h->d_keys.get(), arena->keys, keys_len, cudaMemcpyHostToDevice, h->stream.get()));
    uint64_t done = 0;
    while (done < n) {
        uint32_t m = (uint32_t)std::min<uint64_t>(n - done, h->max_batch);
        const unsigned char *src = (const unsigned char *)req + done * rsz;
        // like the reference's mutating ops, sweep (if the store's policy says so) BEFORE the work
        // (adaptive_cleanup.rs:229,261), with the clock of the first request of the chunk
        int64_t now_hint = rsz == sizeof(gcra_request) ? ((const gcra_request *)req)[done].now_ns : now_batch;
        int rc = apply_policy(h, now_hint);
        if (rc) return rc;
        CK(cudaMemcpyAsync(h->d_req.get(), src, (size_t)m * rsz, cudaMemcpyHostToDevice, h->stream.get()));
        if (arena) RC(enqueue_hash_keys(h, m, h->d_req.get(), (uint32_t)rsz, h->d_keys.get(), keys_len, h->stream.get()));
        rc = launch_batch(h, m, h->d_req.get(), fmt, now_batch, h->d_res.get(), h->stream.get(), true);
        if (rc) return rc;
        CK(cudaMemcpyAsync((unsigned char *)res + done * ressz, h->d_res.get(), (size_t)m * ressz, cudaMemcpyDeviceToHost, h->stream.get()));
        RC(refresh_counters(h, false));
        CK(cudaStreamSynchronize(h->stream.get()));
        done += m;
    }
    return GCRA_OK;
}

int32_t gcra_rate_limit_batch(gcra_engine *h, uint64_t n, const gcra_request *req, gcra_result *res) {
    return host_batch(h, n, req, FMT_48_32, 0, res);
}

int32_t gcra_rate_limit_batch_keys(gcra_engine *h, uint64_t n, const gcra_request *req, const void *keys,
                                   uint64_t keys_len, gcra_result *res) {
    if (!keys && keys_len) { h->err = "null key arena"; return GCRA_INTERNAL; }
    const KeyArena arena = {keys, keys_len};
    return host_batch(h, n, req, FMT_48_32, 0, res, &arena);
}

int32_t gcra_hash_keys_device(gcra_engine *h, uint64_t n, void *d_rows, uint32_t row_bytes, const void *d_keys,
                              uint64_t keys_len, void *stream) {
    CK(cudaSetDevice(h->device));
    return enqueue_hash_keys(h, n, d_rows, row_bytes, d_keys, keys_len, stream ? (cudaStream_t)stream : h->stream.get());
}

int32_t gcra_rate_limit_batch16(gcra_engine *h, uint64_t n, const gcra_request16 *req, int64_t now_ns,
                                gcra_result *res) {
    return host_batch(h, n, req, FMT_16_32, now_ns, res);
}

int32_t gcra_rate_limit_batch16_r16(gcra_engine *h, uint64_t n, const gcra_request16 *req, int64_t now_ns,
                                    gcra_result16 *res) {
    return host_batch(h, n, req, FMT_16_16, now_ns, res);
}

int32_t gcra_rate_limit(gcra_engine *h, const void *key, uint64_t len, int64_t max_burst, int64_t count_per_period,
                        int64_t period, int64_t quantity, int64_t now_ns, gcra_result *out) {
    gcra_request r = {engine_hash(h, key, len), max_burst, count_per_period, period, quantity, now_ns};
    gcra_result tmp;
    int rc = host_batch(h, 1, &r, FMT_48_32, 0, &tmp);
    if (rc) { if (out) { memset(out, 0, sizeof(*out)); out->status = GCRA_INTERNAL; } return rc; }
    if (out) *out = tmp;
    if (tmp.status == GCRA_INTERNAL) h->err = "rate_limit: internal (duration overflow, pre-epoch time or table full)";
    return tmp.status;
}

// validation (rate_limiter.rs:115-117) + derivation of every policy of a table, once
static std::vector<PolicyDerived> derive_policies(uint32_t n, const gcra_policy *policies) {
    std::vector<PolicyDerived> pd(n);
    for (uint32_t i = 0; i < n; i++) {
        const gcra_policy &p = policies[i];
        pd[i].ei = pd[i].dvt = 0; pd[i].pad = 0;
        if (p.max_burst <= 0 || p.count_per_period <= 0 || p.period <= 0) pd[i].status = GCRA_INVALID_RATE_LIMIT;
        else pd[i].status = derive_params(p.max_burst, p.count_per_period, p.period, &pd[i].ei, &pd[i].dvt);
    }
    return pd;
}

int32_t gcra_set_policies(gcra_engine *h, uint32_t n, const gcra_policy *policies) {
    CK(cudaSetDevice(h->device));
    std::vector<PolicyDerived> pd = derive_policies(n, policies);
    CK(cudaStreamSynchronize(h->stream.get()));
    DevBuf<PolicyDerived> d_pol;      // (a failed call keeps the registered table)
    if (n) {
        CK(d_pol.make(n));
        CK(cudaMemcpy(d_pol.get(), pd.data(), n * sizeof(PolicyDerived), cudaMemcpyHostToDevice));
    }
    h->d_pol = std::move(d_pol);
    h->npol = n;
    return GCRA_OK;
}

// Host only, no handle: the 32-byte results of a compact batch from its 16-byte results.  The same outputs_from_cur the
// kernels' outputs_of goes through (gcra_device.cuh), so the rows equal the 32-byte path's bit for bit -- given the
// policy table the batch ran with.
int32_t gcra_expand_results16(uint64_t n, const gcra_request16 *req, int64_t now_ns, const gcra_policy *policies,
                              uint32_t npol, const gcra_result16 *in, gcra_result *out) {
    const std::vector<PolicyDerived> pd = derive_policies(npol, policies);
    int32_t rc = GCRA_OK;
    for (uint64_t i = 0; i < n; i++) {
        gcra_result o;
        memset(&o, 0, sizeof(o));
        o.status = in[i].status;
        if (o.status == GCRA_OK) {
            const uint32_t p = req[i].policy;
            if (p >= npol || pd[p].status != GCRA_OK || now_ns < 0 || req[i].quantity < 0) {
                // the engine cannot have decided this row with this table: not the table the batch ran with
                o.status = GCRA_INTERNAL;
                rc = GCRA_INTERNAL;
            } else {
                const Req r = {now_ns, pd[p].ei, pd[p].dvt, req[i].quantity};
                const Outputs x = outputs_from_cur(in[i].cur_tat_ns, in[i].allowed != 0, r);
                o.remaining = x.remaining;
                o.reset_after_ns = x.reset_after;
                o.retry_after_ns = x.retry_after;
                o.allowed = in[i].allowed;
            }
        }
        out[i] = o;
    }
    return rc;
}

// ---- ring --------------------------------------------------------------------------------------
// key_capacity > 0: every slot also gets a pinned and a device key arena of that many bytes (gcra_ring_create_keyed)
static int ring_create(gcra_engine *h, uint32_t slots, uint32_t slot_capacity, int32_t mode, uint64_t key_capacity) {
    CK(cudaSetDevice(h->device));
    if (!h->ring.empty()) { h->err = "ring already created"; return GCRA_INTERNAL; }
    if (slot_capacity == 0 || slot_capacity > h->max_batch) { h->err = "slot_capacity must be in 1..max_batch"; return GCRA_INTERNAL; }
    if (key_capacity > (1ULL << 32)) { h->err = "key_capacity must be at most 2^32 (32-bit key offsets)"; return GCRA_INTERNAL; }
    // 0: 48-byte requests, 32-byte results; any other value but 2: 16-byte requests, 32-byte results; 2: 16 / 16
    const int fmt = mode == 0 ? FMT_48_32 : mode == 2 ? FMT_16_16 : FMT_16_32;
    const size_t rsz = req_bytes(fmt), ressz = res_bytes(fmt);
    std::vector<RingSlot> ring(slots);    // (a failed call leaves no ring)
    for (auto &s : ring) {
        // request slots are only WRITTEN by the host: optionally write-combined pinned memory (GCRA_RING_WC=1)
        CK(s.h_req.make(slot_capacity * rsz,
                        getenv("GCRA_RING_WC") && atoi(getenv("GCRA_RING_WC")) ? cudaHostAllocWriteCombined : cudaHostAllocDefault));
        CK(s.h_res.make(slot_capacity * ressz));
        CK(s.d_req.make(slot_capacity * rsz));
        CK(s.d_res.make(slot_capacity * ressz));
        if (key_capacity) { CK(s.h_keys.make(key_capacity)); CK(s.d_keys.make(key_capacity)); }
        for (Event *e : {&s.ev_in, &s.ev_done}) CK(e->make(cudaEventDisableTiming));
    }
    h->ring = std::move(ring);
    h->ring_cap = slot_capacity;
    h->ring_fmt = fmt;
    h->ring_key_cap = key_capacity;
    return GCRA_OK;
}

int32_t gcra_ring_create(gcra_engine *h, uint32_t slots, uint32_t slot_capacity, int32_t mode) {
    return ring_create(h, slots, slot_capacity, mode, 0);
}

int32_t gcra_ring_create_keyed(gcra_engine *h, uint32_t slots, uint32_t slot_capacity, int32_t mode,
                               uint64_t key_capacity) {
    if (key_capacity == 0) { h->err = "key_capacity must be at least 1"; return GCRA_INTERNAL; }
    return ring_create(h, slots, slot_capacity, mode, key_capacity);
}

void *gcra_ring_keys(gcra_engine *h, uint32_t slot) { return slot < h->ring.size() ? h->ring[slot].h_keys.get() : nullptr; }

void *gcra_ring_requests(gcra_engine *h, uint32_t slot) { return slot < h->ring.size() ? h->ring[slot].h_req.get() : nullptr; }
gcra_result *gcra_ring_results(gcra_engine *h, uint32_t slot) {
    return slot < h->ring.size() && res_bytes(h->ring_fmt) == sizeof(gcra_result) ? (gcra_result *)h->ring[slot].h_res.get() : nullptr;
}
gcra_result16 *gcra_ring_results16(gcra_engine *h, uint32_t slot) {
    return slot < h->ring.size() && res_bytes(h->ring_fmt) == sizeof(gcra_result16) ? (gcra_result16 *)h->ring[slot].h_res.get() : nullptr;
}

// keys_len != null: the rows hold key references into the slot's arena, whose first *keys_len bytes go to the device
// with the rows; the hash pass runs on in_stream before ev_in, so everything after it is the unkeyed path
static int ring_submit(gcra_engine *h, uint32_t slot, uint32_t n, int64_t now_ns, const uint64_t *keys_len) {
    CK(cudaSetDevice(h->device));
    if (slot >= h->ring.size() || n > h->ring_cap) { h->err = "bad ring slot / size"; return GCRA_INTERNAL; }
    if (h->ring_proto) { h->err = "a RESP, HTTP, gRPC or mixed ring takes gcra_resp_ring_submit"; return GCRA_INTERNAL; }
    if (keys_len && *keys_len > h->ring_key_cap) { h->err = "keys_len larger than the ring's key_capacity"; return GCRA_INTERNAL; }
    RingSlot &s = h->ring[slot];
    if (s.in_flight) { h->err = "ring slot still in flight"; return GCRA_INTERNAL; }
    // sweep policy with the counters of the batches finished so far (no stall)
    if (cudaEventQuery(h->ev_counters.get()) == cudaSuccess) { int rc = apply_policy(h, now_ns); if (rc) return rc; }
    const size_t rsz = req_bytes(h->ring_fmt), ressz = res_bytes(h->ring_fmt);
    CK(cudaMemcpyAsync(s.d_req.get(), s.h_req.get(), (size_t)n * rsz, cudaMemcpyHostToDevice, h->in_stream.get()));
    if (keys_len) {
        if (*keys_len) CK(cudaMemcpyAsync(s.d_keys.get(), s.h_keys.get(), *keys_len, cudaMemcpyHostToDevice, h->in_stream.get()));
        RC(enqueue_hash_keys(h, n, s.d_req.get(), (uint32_t)rsz, s.d_keys.get(), *keys_len, h->in_stream.get()));
    }
    CK(cudaEventRecord(s.ev_in.get(), h->in_stream.get()));
    // front half (ingest + order) of this slot overlaps the back half (decide) of the previous one
    cudaEvent_t done = nullptr;
    int rc = launch_pipelined(h, n, s.d_req.get(), h->ring_fmt, now_ns, s.d_res.get(), s.ev_in.get(), &done);
    if (rc) return rc;
    if (done) CK(cudaStreamWaitEvent(h->out_stream.get(), done, 0));
    CK(cudaMemcpyAsync(h->h_counters.get(), h->tab.view.counters, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost, h->out_stream.get()));
    CK(cudaEventRecord(h->ev_counters.get(), h->out_stream.get()));
    CK(cudaMemcpyAsync(s.h_res.get(), s.d_res.get(), (size_t)n * ressz, cudaMemcpyDeviceToHost, h->out_stream.get()));
    CK(cudaEventRecord(s.ev_done.get(), h->out_stream.get()));
    s.in_flight = true;
    return GCRA_OK;
}

int32_t gcra_ring_submit(gcra_engine *h, uint32_t slot, uint32_t n, int64_t now_ns) {
    return ring_submit(h, slot, n, now_ns, nullptr);
}

int32_t gcra_ring_submit_keyed(gcra_engine *h, uint32_t slot, uint32_t n, uint64_t keys_len, int64_t now_ns) {
    if (h->ring_key_cap == 0) { h->err = "the ring has no key arenas (gcra_ring_create_keyed)"; return GCRA_INTERNAL; }
    return ring_submit(h, slot, n, now_ns, &keys_len);
}

int32_t gcra_ring_wait(gcra_engine *h, uint32_t slot) {
    if (slot >= h->ring.size()) { h->err = "bad ring slot"; return GCRA_INTERNAL; }
    RingSlot &s = h->ring[slot];
    if (!s.in_flight) return GCRA_OK;
    CK(cudaEventSynchronize(s.ev_done.get()));
    s.in_flight = false;
    return GCRA_OK;
}

int32_t gcra_ring_poll(gcra_engine *h, uint32_t slot, int32_t *done) {
    if (slot >= h->ring.size()) { h->err = "bad ring slot"; return GCRA_INTERNAL; }
    RingSlot &s = h->ring[slot];
    if (!s.in_flight) { *done = 1; return GCRA_OK; }
    cudaError_t e = cudaEventQuery(s.ev_done.get());
    if (e == cudaSuccess) { s.in_flight = false; *done = 1; return GCRA_OK; }
    if (e == cudaErrorNotReady) { *done = 0; return GCRA_OK; }
    h->err = cudaGetErrorString(e);
    return GCRA_INTERNAL;
}

// ---- sweep / introspection ---------------------------------------------------------------------
int32_t gcra_sweep(gcra_engine *h, int64_t now_ns, uint64_t *removed) { return do_sweep(h, now_ns, removed); }

// The store kind's own sweep policy (maybe_clean_expired: adaptive_cleanup.rs:205-211, periodic.rs:128-142,
// probabilistic.rs:110-125) evaluated against the counters of everything finished so far.  The host-buffer calls
// and the ring do this themselves before every batch; the device-resident, pipelined and sharded submissions
// cannot (the requests' clocks live on the device): their caller ticks the policy with its own clock.
int32_t gcra_policy_tick(gcra_engine *h, int64_t now_ns, uint64_t *swept) {
    CK(cudaSetDevice(h->device));
    if (swept) *swept = 0;
    if (h->kind == GCRA_STORE_MANUAL) return GCRA_OK;
    RC(wait_for_batches(h));
    RC(refresh_counters(h, true));
    const uint64_t before = h->h_counters.get()[C_SWEPT];
    RC(apply_policy(h, now_ns));
    if (swept) { RC(refresh_counters(h, true)); *swept = h->h_counters.get()[C_SWEPT] - before; }
    return GCRA_OK;
}

uint64_t gcra_len(gcra_engine *h) {
    cudaSetDevice(h->device);
    if (refresh_counters(h, true)) return 0;
    return h->h_counters.get()[C_REAL];
}

int32_t gcra_get_stats(gcra_engine *h, gcra_stats *out) {
    CK(cudaSetDevice(h->device));
    int rc = refresh_counters(h, true);
    if (rc) return rc;
    const u64 *c = h->h_counters.get();
    out->len = c[C_REAL];
    out->occupied_slots = c[C_OCCUPIED];
    out->table_slots = h->tab.slots();
    out->stash_entries = c[C_STASH];
    out->allowed = c[C_ALLOWED];
    out->denied = c[C_DENIED];
    out->errors = c[C_ERRORS];
    out->expired_hits = c[C_EXPIRED_HITS];
    out->sweeps = h->n_sweeps;
    out->swept = c[C_SWEPT];
    out->grows = h->n_grows;
    out->purges = h->n_purges;
    out->index_batches = h->n_index_batches;
    out->residue_rows = h->residue_seen;
    out->residue_batches = h->residue_batches_seen;
    out->drains = h->n_drains;
    out->path_switches = h->n_path_switches;
    return GCRA_OK;
}

int32_t gcra_peek(gcra_engine *h, uint64_t key_hash, int64_t *tat, int64_t *expiry_ns, uint8_t *found) {
    int rc = store_op(h, 3, key_hash, 0, 0, 0, 0);
    if (rc) return rc;
    *found = (uint8_t)h->h_op.get()[0].flag;
    if (*found) { *tat = h->h_op.get()[0].value; *expiry_ns = h->h_op.get()[1].value; }
    return GCRA_OK;
}

// ---- metrics bridge: top denied keys (throttlecrab-server/src/metrics.rs:24-64,162-173) --------------------------
// the names of a table of `cap` entries (ring metrics), none known
static int make_names(gcra_engine *h, DevBuf<unsigned char> &names, DevBuf<u32> &name_len, uint64_t cap) {
    CK(names.make((size_t)cap * GCRA_DENIED_NAME_MAX));
    CK(name_len.make(cap));
    CK(cudaMemset(name_len.get(), 0xff, cap * sizeof(u32)));           // GCRA_NAME_UNKNOWN
    return GCRA_OK;
}
static int make_denied_names(gcra_engine *h, DeniedArrays &a, uint64_t cap) {
    return make_names(h, a.names, a.name_len, cap);
}

// entries of a denied table, or of a name table, for max_keys > 0 keys: 16 per key, at least 1024, a power of two
static uint64_t denied_entries(uint32_t max_keys) {
    return 1ULL << ceil_log2(std::max<uint64_t>(16ULL * max_keys, 1024));
}

int32_t gcra_track_denied(gcra_engine *h, uint32_t max_keys) {
    CK(cudaSetDevice(h->device));
    // the table holds 16 entries per tracked key: at most 2^31
    if (max_keys > (1u << 27)) { h->err = "track_denied: max_keys must be at most 2^27"; return GCRA_INTERNAL; }
    if (h->ring_metrics && max_keys > GCRA_RING_METRICS_MAX_KEYS) {
        h->err = "track_denied: max_keys must be at most 10,000 while ring metrics are on";
        return GCRA_INTERNAL;
    }
    RC(wait_for_metrics_writers(h));
    CK(cudaDeviceSynchronize());
    DeniedArrays a;
    const uint64_t cap = max_keys ? denied_entries(max_keys) : 0;
    if (max_keys) {
        CK(a.keys.make(cap));
        CK(a.counts.make(cap));
        CK(a.dropped.make(1));
        CK(cudaMemset(a.keys.get(), 0, cap * sizeof(u64)));
        CK(cudaMemset(a.counts.get(), 0, cap * sizeof(u64)));
        CK(cudaMemset(a.dropped.get(), 0, sizeof(u64)));
        if (h->ring_metrics) RC(make_denied_names(h, a, cap));
    }
    h->denied = max_keys ? DeniedTable{a.keys.get(), a.counts.get(), (u32)(cap - 1), a.dropped.get()} : DeniedTable{};
    h->denied_arrays = std::move(a);
    h->denied_max = max_keys;
    h->denied_cap = cap;
    return GCRA_OK;
}

// the k most denied keys (hash, count), most denied first; *dropped = denials of keys that found the table full.
// The pruning moves each surviving key's name (ring metrics) with it and forgets the others'.
// Like the reference's cleanup (metrics.rs:52-64) the table is pruned to its `max_keys` top entries when more than
// three times as many have accumulated.  Waits for every scratch set's ev_back, which a peer-memory tick records
// after its count and before it publishes its results: multi-GPU callers query between ticks, after joining them.
int32_t gcra_top_denied(gcra_engine *h, uint32_t k, uint64_t *key_hashes, uint64_t *counts, uint32_t *n_out, uint64_t *dropped) {
    CK(cudaSetDevice(h->device));
    if (n_out) *n_out = 0;
    if (!h->denied_max) { h->err = "gcra_track_denied first"; return GCRA_INTERNAL; }
    RC(wait_for_metrics_writers(h));
    std::vector<u64> keys(h->denied_cap), cnts(h->denied_cap);
    CK(cudaMemcpy(keys.data(), h->denied.keys, keys.size() * sizeof(u64), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(cnts.data(), h->denied.counts, cnts.size() * sizeof(u64), cudaMemcpyDeviceToHost));
    if (dropped) CK(cudaMemcpy(dropped, h->denied.dropped, sizeof(u64), cudaMemcpyDeviceToHost));
    struct Entry { u64 count, key; uint32_t at; };
    std::vector<Entry> top;
    for (uint32_t i = 0; i < h->denied_cap; i++) if (keys[i]) top.push_back({cnts[i], keys[i], i});
    std::sort(top.begin(), top.end(), [](const Entry &a, const Entry &b) {
        return a.count != b.count ? a.count > b.count : a.key < b.key;
    });
    const uint32_t n = (uint32_t)std::min<size_t>(k, top.size());
    for (uint32_t i = 0; i < n; i++) { key_hashes[i] = top[i].key; counts[i] = top[i].count; }
    if (n_out) *n_out = n;
    if (top.size() > (size_t)3 * h->denied_max) {
        DeniedArrays &a = h->denied_arrays;
        const bool named = a.name_len.get() != nullptr;
        const size_t nb = named ? (size_t)h->denied_cap * GCRA_DENIED_NAME_MAX : 0;
        std::vector<u32> len(named ? h->denied_cap : 0), new_len(len.size(), GCRA_NAME_UNKNOWN);
        std::vector<unsigned char> names(nb), new_names(nb);
        if (named) {
            CK(cudaMemcpy(len.data(), a.name_len.get(), len.size() * sizeof(u32), cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(names.data(), a.names.get(), nb, cudaMemcpyDeviceToHost));
        }
        std::fill(keys.begin(), keys.end(), 0);
        std::fill(cnts.begin(), cnts.end(), 0);
        for (uint32_t i = 0; i < h->denied_max; i++) {
            uint32_t s = (uint32_t)(mix64(top[i].key ^ 0x9E3779B97F4A7C15ULL)) & h->denied.mask;
            while (keys[s]) s = (s + 1) & h->denied.mask;
            keys[s] = top[i].key;
            cnts[s] = top[i].count;
            if (named) {
                const uint32_t from = top[i].at;
                new_len[s] = len[from];
                if (len[from] <= GCRA_DENIED_NAME_MAX)
                    memcpy(&new_names[(size_t)s * GCRA_DENIED_NAME_MAX], &names[(size_t)from * GCRA_DENIED_NAME_MAX], len[from]);
            }
        }
        CK(cudaMemcpy(h->denied.keys, keys.data(), keys.size() * sizeof(u64), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(h->denied.counts, cnts.data(), cnts.size() * sizeof(u64), cudaMemcpyHostToDevice));
        if (named) {
            CK(cudaMemcpy(a.name_len.get(), new_len.data(), new_len.size() * sizeof(u32), cudaMemcpyHostToDevice));
            CK(cudaMemcpy(a.names.get(), new_names.data(), nb, cudaMemcpyHostToDevice));
        }
    }
    return GCRA_OK;
}

// ---- ring metrics (metrics.rs:233-310: requests by transport, top denied keys by name) ------------------------------
int32_t gcra_ring_metrics(gcra_engine *h, uint32_t on) {
    CK(cudaSetDevice(h->device));
    if (on && h->ring_p2p) { h->err = "ring metrics: the ring's ticks are peer-memory ticks (gcra_ring_p2p)"; return GCRA_INTERNAL; }
    if (on && h->ring_metrics_sharded) { h->err = "ring metrics: sharded ring metrics are on"; return GCRA_INTERNAL; }
    if (on && h->denied_max > GCRA_RING_METRICS_MAX_KEYS) {
        h->err = "ring metrics: denied tracking runs with max_keys above 10,000";
        return GCRA_INTERNAL;
    }
    RC(wait_for_metrics_writers(h));
    if (!on) {
        h->ring_metrics = false;
        h->denied_arrays.names.reset();
        h->denied_arrays.name_len.reset();
        return GCRA_OK;
    }
    DevBuf<u64> counts;                                 // (built whole before anything is swapped in)
    CK(counts.make(9));
    CK(cudaMemset(counts.get(), 0, 9 * sizeof(u64)));
    DeniedArrays named;
    if (h->denied_max) RC(make_denied_names(h, named, h->denied_cap));
    h->ring_counts = std::move(counts);
    h->denied_arrays.names = std::move(named.names);
    h->denied_arrays.name_len = std::move(named.name_len);
    h->ring_metrics = true;
    return GCRA_OK;
}

int32_t gcra_ring_transport_counts(gcra_engine *h, gcra_transport_counts out[3]) {
    CK(cudaSetDevice(h->device));
    if (!h->ring_counts.get()) { memset(out, 0, 3 * sizeof(gcra_transport_counts)); return GCRA_OK; }
    RC(wait_for_metrics_writers(h));
    static_assert(sizeof(gcra_transport_counts) == 3 * sizeof(u64), "three counters per transport");
    CK(cudaMemcpy(out, h->ring_counts.get(), 9 * sizeof(u64), cudaMemcpyDeviceToHost));
    return GCRA_OK;
}

// ---- sharded ring metrics: names in a table of this rank's own (the denied counts are on the keys' owners) ---------
// an empty name table of `cap` entries, built on the engine's stream
static int make_name_table(gcra_engine *h, NameTable &t, uint64_t cap) {
    const cudaStream_t st = h->stream.get();
    CK(t.keys.make(cap));
    CK(t.full.make(1));
    RC(make_names(h, t.names, t.name_len, cap));
    CK(cudaMemsetAsync(t.keys.get(), 0, cap * sizeof(u64), st));
    CK(cudaMemsetAsync(t.full.get(), 0, sizeof(u64), st));
    CK(cudaStreamSynchronize(st));
    t.cap = cap;
    return GCRA_OK;
}

int32_t gcra_ring_metrics_sharded(gcra_engine *h, uint32_t on, uint32_t max_keys) {
    CK(cudaSetDevice(h->device));
    // (a routed slot's parse chose whether to write key positions; its finish must launch what the parse chose for)
    if (h->p2p && h->p2p->ring_slot_pending >= 0) { h->err = "a routed ring tick is not finished yet"; return GCRA_INTERNAL; }
    if (on && h->ring_metrics) { h->err = "sharded ring metrics: ring metrics are on (gcra_ring_metrics)"; return GCRA_INTERNAL; }
    if (on && max_keys > GCRA_RING_METRICS_MAX_KEYS) {
        h->err = "sharded ring metrics: max_keys must be at most 10,000";
        return GCRA_INTERNAL;
    }
    RC(wait_for_metrics_writers(h));
    if (!on) {
        h->ring_metrics_sharded = false;
        h->ring_names = NameTable();
        return GCRA_OK;
    }
    DevBuf<u64> counts;                                 // (built whole before anything is swapped in)
    CK(counts.make(9));
    CK(cudaMemset(counts.get(), 0, 9 * sizeof(u64)));
    NameTable t;
    if (max_keys) RC(make_name_table(h, t, denied_entries(max_keys)));
    h->ring_counts = std::move(counts);
    h->ring_names = std::move(t);
    h->ring_metrics_sharded = true;
    return GCRA_OK;
}

int32_t gcra_ring_names_keep(gcra_engine *h, uint32_t n, const uint64_t *key_hashes, uint64_t *full) {
    CK(cudaSetDevice(h->device));
    if (full) *full = 0;
    if (!h->ring_metrics_sharded) { h->err = "gcra_ring_metrics_sharded first"; return GCRA_INTERNAL; }
    RC(wait_for_metrics_writers(h));
    const NameTable &old = h->ring_names;
    if (!old.cap) return GCRA_OK;
    uint64_t was_full = 0;
    CK(cudaMemcpy(&was_full, old.full.get(), sizeof(u64), cudaMemcpyDeviceToHost));
    NameTable t;                                        // (built whole before it replaces the old one)
    RC(make_name_table(h, t, old.cap));
    if (n) {
        const cudaStream_t st = h->stream.get();
        DevBuf<u64> d_hashes;
        CK(d_hashes.make(n));
        CK(cudaMemcpyAsync(d_hashes.get(), key_hashes, n * sizeof(u64), cudaMemcpyHostToDevice, st));
        CK(launch_ring_names_keep(old.view(), t.view(), d_hashes.get(), n, t.full.get(), st));
        h->launches++;
        CK(cudaStreamSynchronize(st));
    }
    h->ring_names = std::move(t);
    if (full) *full = was_full;
    return GCRA_OK;
}

// gcra_denied_names on sharded ring metrics: the lookup kernel over the name table, only the n names copied back
static int ring_names_lookup(gcra_engine *h, uint32_t n, const uint64_t *key_hashes, char *names, uint32_t *lens) {
    RC(wait_for_metrics_writers(h));
    for (uint32_t i = 0; i < n; i++) lens[i] = GCRA_NAME_UNKNOWN;
    const NameTable &t = h->ring_names;
    if (!t.cap || !n) return GCRA_OK;
    const cudaStream_t st = h->stream.get();
    DevBuf<u64> d_hashes;
    DevBuf<u32> d_len;
    DevBuf<unsigned char> d_names;
    CK(d_hashes.make(n));
    CK(d_len.make(n));
    CK(d_names.make((size_t)n * GCRA_DENIED_NAME_MAX));
    CK(cudaMemcpyAsync(d_hashes.get(), key_hashes, n * sizeof(u64), cudaMemcpyHostToDevice, st));
    CK(launch_ring_names_lookup(t.view(), d_hashes.get(), n, d_len.get(), d_names.get(), st));
    h->launches++;
    std::vector<unsigned char> all((size_t)n * GCRA_DENIED_NAME_MAX);
    CK(cudaMemcpyAsync(lens, d_len.get(), n * sizeof(u32), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(all.data(), d_names.get(), all.size(), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (uint32_t i = 0; i < n; i++)        // (each name's bytes, and no more, as from the denied table)
        if (lens[i] <= GCRA_DENIED_NAME_MAX)
            memcpy(names + (size_t)i * GCRA_DENIED_NAME_MAX, &all[(size_t)i * GCRA_DENIED_NAME_MAX], lens[i]);
    return GCRA_OK;
}

int32_t gcra_denied_names(gcra_engine *h, uint32_t n, const uint64_t *key_hashes, char *names, uint32_t *lens) {
    CK(cudaSetDevice(h->device));
    if (h->ring_metrics_sharded) return ring_names_lookup(h, n, key_hashes, names, lens);
    if (!h->denied_max) { h->err = "gcra_track_denied first"; return GCRA_INTERNAL; }
    RC(wait_for_metrics_writers(h));
    for (uint32_t i = 0; i < n; i++) lens[i] = GCRA_NAME_UNKNOWN;
    const DeniedArrays &a = h->denied_arrays;
    if (!a.name_len.get() || !n) return GCRA_OK;
    // (the whole table in three copies: a scrape asks for every entry gcra_top_denied returns)
    std::vector<u64> keys(h->denied_cap);
    std::vector<u32> len(h->denied_cap);
    std::vector<unsigned char> all((size_t)h->denied_cap * GCRA_DENIED_NAME_MAX);
    CK(cudaMemcpy(keys.data(), h->denied.keys, keys.size() * sizeof(u64), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(len.data(), a.name_len.get(), len.size() * sizeof(u32), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(all.data(), a.names.get(), all.size(), cudaMemcpyDeviceToHost));
    for (uint32_t i = 0; i < n; i++) {
        const u64 k = key_hashes[i] ? key_hashes[i] : 1;                     // (as the table stores it)
        uint32_t s = (uint32_t)(mix64(k ^ 0x9E3779B97F4A7C15ULL)) & h->denied.mask;
        for (uint32_t probe = 0; probe < 64 && keys[s]; probe++, s = (s + 1) & h->denied.mask) {
            if (keys[s] != k) continue;
            lens[i] = len[s];
            if (len[s] <= GCRA_DENIED_NAME_MAX)
                memcpy(names + (size_t)i * GCRA_DENIED_NAME_MAX, &all[(size_t)s * GCRA_DENIED_NAME_MAX], len[s]);
            break;
        }
    }
    return GCRA_OK;
}

int32_t gcra_sync(gcra_engine *h) {
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->in_stream.get()));
    CK(cudaStreamSynchronize(h->front_stream.get()));
    CK(cudaStreamSynchronize(h->back_stream.get()));
    CK(cudaStreamSynchronize(h->tail_stream.get()));
    CK(cudaStreamSynchronize(h->aux_stream.get()));
    CK(cudaStreamSynchronize(h->aux2_stream.get()));
    CK(cudaStreamSynchronize(h->stream.get()));
    CK(cudaStreamSynchronize(h->out_stream.get()));
    return GCRA_OK;
}

int32_t gcra_last_kernel_ms(gcra_engine *h, float out[4]) {
    if (!h->ev_valid) { h->err = "no timed batch yet"; return GCRA_INTERNAL; }
    CK(cudaEventSynchronize(h->ev[3].get()));
    CK(cudaEventElapsedTime(&out[0], h->ev[0].get(), h->ev[3].get()));
    CK(cudaEventElapsedTime(&out[1], h->ev[0].get(), h->ev[1].get()));
    CK(cudaEventElapsedTime(&out[2], h->ev[1].get(), h->ev[2].get()));
    CK(cudaEventElapsedTime(&out[3], h->ev[2].get(), h->ev[3].get()));
    return GCRA_OK;
}

int32_t gcra_last_kernel_ms_detail(gcra_engine *h, float out[7]) {
    if (!h->evd_valid) { h->err = "no timed index-order batch yet"; return GCRA_INTERNAL; }
    CK(cudaEventSynchronize(h->evd[7].get()));
    for (int i = 0; i < 7; i++) CK(cudaEventElapsedTime(&out[i], h->evd[i].get(), h->evd[i + 1].get()));
    return GCRA_OK;
}

void gcra_debug_set(gcra_engine *h, uint32_t mask) { h->dbg = mask; }

int32_t gcra_last_sweep_ms(gcra_engine *h, float *ms) {
    if (!h->sweep_timed) { h->err = "no sweep yet"; return GCRA_INTERNAL; }
    CK(cudaEventSynchronize(h->ev_sweep[1].get()));
    CK(cudaEventElapsedTime(ms, h->ev_sweep[0].get(), h->ev_sweep[1].get()));
    return GCRA_OK;
}

uint64_t gcra_launch_count(gcra_engine *h) { return h->launches; }

// ---- snapshot / restore (absent in the reference: its state is lost on restart; SURVEY 8f #4) -----------
// the header of a file of the engine's table; the caller fills in the counters
static SnapshotHeader header_of(const gcra_engine *h, uint32_t version) {
    SnapshotHeader hd{};
    memcpy(hd.magic, SNAP_MAGIC, 8);
    hd.version = version;
    hd.total_lines = h->tab.lines(); hd.nb_main = h->tab.view.nb_main; hd.stash_slots = h->tab.view.stash_slots;
    hd.capacity = h->tab.capacity;
    hd.hash_seed[0] = h->hash_seed[0]; hd.hash_seed[1] = h->hash_seed[1];
    return hd;
}

static int copy_to_file(gcra_engine *h, FILE *f, const void *dptr, size_t bytes, std::vector<char> &buf) {
    for (size_t off = 0; off < bytes; off += SNAP_CHUNK) {
        size_t m = std::min(SNAP_CHUNK, bytes - off);
        CK(cudaMemcpy(buf.data(), (const char *)dptr + off, m, cudaMemcpyDeviceToHost));
        if (fwrite(buf.data(), 1, m, f) != m) { h->err = "snapshot: short write"; return GCRA_INTERNAL; }
    }
    return GCRA_OK;
}

int32_t gcra_snapshot_save(gcra_engine *h, const char *path) {
    CK(cudaSetDevice(h->device));
    CK(cudaDeviceSynchronize());
    FILE *f = fopen(path, "wb");
    if (!f) { h->err = std::string("snapshot: cannot open ") + path; return GCRA_INTERNAL; }
    SnapshotHeader hd = header_of(h, 2);
    int rc = GCRA_OK;
    if (cudaMemcpy(hd.counters, h->tab.view.counters, sizeof(hd.counters), cudaMemcpyDeviceToHost) != cudaSuccess ||
        fwrite(&hd, sizeof(hd), 1, f) != 1) { h->err = "snapshot: header"; rc = GCRA_INTERNAL; }
    std::vector<char> buf(SNAP_CHUNK);
    const size_t slots = h->tab.slots();
    if (!rc) rc = copy_to_file(h, f, h->tab.view.keys, slots * sizeof(u64), buf);
    if (!rc) rc = copy_to_file(h, f, h->tab.view.state, slots * sizeof(TatOff), buf);
    if (!rc) rc = copy_to_file(h, f, h->tab.view.ei, slots * sizeof(i64), buf);
    if (fclose(f) != 0 && !rc) { h->err = "snapshot: close"; rc = GCRA_INTERNAL; }
    return rc;
}

// Streams a file through the GPU in chunks of RESTORE_CHUNK slots (one staging set = SNAP_CHUNK bytes over the three
// sections; two sets, so that reading chunk i + 1 overlaps the copy and kernel of chunk i).
namespace {
const size_t RESTORE_CHUNK = SNAP_CHUNK / (sizeof(u64) + sizeof(TatOff) + sizeof(i64));

struct RestoreBuffers {
    PinnedBuf<char> host[2];           // keys | state | ei of one chunk
    DevBuf<char> dev[2];
    DevBuf<u64> counts;                // [RESTORE_COUNTS]
    Event done[2];                     // the set's copy + kernel finished: its host buffer may be refilled
    int fd = -1;
};

// What restore_pass does with each chunk: restore_kernel counts the entries this shard takes (COUNT) or inserts them
// (INSERT); COPY writes the sections to the same slots of the table (a version 2 load: they are its arrays).
enum RestorePass { PASS_COUNT, PASS_INSERT, PASS_COPY };
}  // namespace

static bool pread_all(int fd, void *buf, size_t bytes, uint64_t off) {
    for (size_t got = 0; got < bytes;) {
        const ssize_t r = pread(fd, (char *)buf + got, bytes - got, (off_t)(off + got));
        if (r <= 0) return false;
        got += (size_t)r;
    }
    return true;
}

// The sections of a snapshot file, checked against the file's length.  Version 2: every slot of the table (header,
// keys, (tat, off) pairs, ei).  Version 3 (gcra_snapshot_begin): the header, the entry count n, then the same three
// sections restricted to the n carried entries.
struct SnapSections { uint64_t rows, keys_off, state_off, ei_off; };

// the header of the file open at `fd` and where its sections lie; null, or why the file is refused
static const char *read_header(int fd, SnapshotHeader &hd, SnapSections &sec) {
    if (!pread_all(fd, &hd, sizeof(hd), 0) || memcmp(hd.magic, SNAP_MAGIC, 8) != 0 || (hd.version != 2 && hd.version != 3))
        return "bad header";
    struct stat sb;
    if (fstat(fd, &sb) != 0) return "cannot stat the file";
    const uint64_t size = (uint64_t)sb.st_size, row = sizeof(u64) + sizeof(TatOff) + sizeof(i64);
    const uint64_t slots = (uint64_t)hd.total_lines * 4;
    if ((uint64_t)hd.nb_main * 4 + hd.stash_slots > slots) return "bad geometry";
    if (hd.version == 2) {
        sec.rows = slots;
        sec.keys_off = sizeof(hd);
    } else {
        uint64_t n = 0;
        if (size < sizeof(hd) + sizeof(n) || !pread_all(fd, &n, sizeof(n), sizeof(hd))) return "file length does not match its header";
        if (n > (size - sizeof(hd) - sizeof(n)) / row) return "file length does not match its header";
        sec.rows = n;
        sec.keys_off = sizeof(hd) + sizeof(n);
    }
    if (size != sec.keys_off + sec.rows * row) return "file length does not match its header";
    sec.state_off = sec.keys_off + sec.rows * sizeof(u64);
    sec.ei_off = sec.state_off + sec.rows * sizeof(TatOff);
    return nullptr;
}

static int make_restore_buffers(gcra_engine *h, RestoreBuffers &b) {
    for (int s = 0; s < 2; s++) {
        CK(b.host[s].make(SNAP_CHUNK));
        CK(b.dev[s].make(SNAP_CHUNK));
        CK(b.done[s].make(cudaEventDisableTiming));
    }
    CK(b.counts.make(RESTORE_COUNTS));
    CK(cudaMemsetAsync(b.counts.get(), 0, RESTORE_COUNTS * sizeof(u64), h->stream.get()));
    return GCRA_OK;
}

// one pass over the `sec.rows` rows of a file's sections into table `t`
static int restore_pass(gcra_engine *h, RestoreBuffers &b, const Table &t, const SnapSections &sec, uint32_t rank,
                        uint32_t world, RestorePass pass) {
    for (uint64_t first = 0, c = 0; first < sec.rows; first += RESTORE_CHUNK, c++) {
        const int s = (int)(c & 1);
        const uint64_t n = std::min<uint64_t>(RESTORE_CHUNK, sec.rows - first);
        char *hk = b.host[s].get(), *hs = hk + RESTORE_CHUNK * sizeof(u64), *he = hs + RESTORE_CHUNK * sizeof(TatOff);
        char *dk = b.dev[s].get(), *ds = dk + RESTORE_CHUNK * sizeof(u64), *de = ds + RESTORE_CHUNK * sizeof(TatOff);
        if (pass == PASS_COPY) { dk = (char *)(t.keys + first); ds = (char *)(t.state + first); de = (char *)(t.ei + first); }
        CK(cudaEventSynchronize(b.done[s].get()));
        if (!pread_all(b.fd, hk, n * sizeof(u64), sec.keys_off + first * sizeof(u64)) ||
            !pread_all(b.fd, hs, n * sizeof(TatOff), sec.state_off + first * sizeof(TatOff)) ||
            (pass != PASS_COUNT && !pread_all(b.fd, he, n * sizeof(i64), sec.ei_off + first * sizeof(i64)))) {
            h->err = "snapshot: short read";
            return GCRA_INTERNAL;
        }
        CK(cudaMemcpyAsync(dk, hk, n * sizeof(u64), cudaMemcpyHostToDevice, h->stream.get()));
        CK(cudaMemcpyAsync(ds, hs, n * sizeof(TatOff), cudaMemcpyHostToDevice, h->stream.get()));
        if (pass != PASS_COUNT) CK(cudaMemcpyAsync(de, he, n * sizeof(i64), cudaMemcpyHostToDevice, h->stream.get()));
        if (pass != PASS_COPY) {
            const uint32_t grid = (uint32_t)std::min<uint64_t>((n + TILE_THREADS - 1) / TILE_THREADS, 8 * h->sms);
            (pass == PASS_INSERT ? restore_kernel<true> : restore_kernel<false>)<<<grid, TILE_THREADS, 0, h->stream.get()>>>(
                t, (const u64 *)dk, (const TatOff *)ds, (const i64 *)de, n, rank, world, b.counts.get());
            h->launches++;
            CK(cudaGetLastError());
        }
        CK(cudaEventRecord(b.done[s].get(), h->stream.get()));
    }
    CK(cudaStreamSynchronize(h->stream.get()));
    return GCRA_OK;
}

static int restore_file(gcra_engine *h, RestoreBuffers &b, uint32_t rank, uint32_t world, uint64_t *restored,
                        uint64_t *conflicts) {
    SnapshotHeader hd{};
    SnapSections sec;
    if (const char *why = read_header(b.fd, hd, sec)) { h->err = std::string("snapshot restore: ") + why; return GCRA_INTERNAL; }
    CK(cudaDeviceSynchronize());
    RC(refresh_counters(h, true));
    const bool adopt_seed = h->h_counters.get()[C_REAL] == 0;
    if (!adopt_seed && (hd.hash_seed[0] != h->hash_seed[0] || hd.hash_seed[1] != h->hash_seed[1])) {
        h->err = "snapshot restore: the file's key-hash seed differs from that of the entries held";
        return GCRA_INTERNAL;
    }
    RC(make_restore_buffers(h, b));
    RC(restore_pass(h, b, h->tab.view, sec, rank, world, PASS_COUNT));
    u64 counts[RESTORE_COUNTS];
    CK(cudaMemcpy(counts, b.counts.get(), sizeof(counts), cudaMemcpyDeviceToHost));
    RC(ensure_room(h, counts[RESTORE_OWNED]));     // may purge or grow: h->tab is read after it
    RC(restore_pass(h, b, h->tab.view, sec, rank, world, PASS_INSERT));
    CK(cudaMemcpy(counts, b.counts.get(), sizeof(counts), cudaMemcpyDeviceToHost));
    RC(refresh_counters(h, true));
    reset_occupancy(h, h->h_counters.get()[C_OCCUPIED]);
    if (counts[RESTORE_FAILED]) {
        h->err = "snapshot restore: table full (" + std::to_string(counts[RESTORE_FAILED]) + " entries not inserted)";
        return GCRA_INTERNAL;
    }
    if (adopt_seed) { h->hash_seed[0] = hd.hash_seed[0]; h->hash_seed[1] = hd.hash_seed[1]; }
    if (restored) *restored = counts[RESTORE_INSERTED];
    if (conflicts) *conflicts = counts[RESTORE_CONFLICTS];
    return GCRA_OK;
}

// the staging buffers of `b` may still be read by queued copies: wait for them before `b` releases them
static void close_restore(RestoreBuffers &b) {
    for (Event &e : b.done) if (e.get()) cudaEventSynchronize(e.get());
    close(b.fd);
}

int32_t gcra_snapshot_restore(gcra_engine *h, const char *path, uint32_t rank, uint32_t world, uint64_t *restored,
                              uint64_t *conflicts) {
    if (restored) *restored = 0;
    if (conflicts) *conflicts = 0;
    CK(cudaSetDevice(h->device));
    if (world == 0 || rank >= world) { h->err = "snapshot restore: needs rank < world"; return GCRA_INTERNAL; }
    RestoreBuffers b;
    b.fd = open(path, O_RDONLY);
    if (b.fd < 0) { h->err = std::string("snapshot restore: cannot open ") + path; return GCRA_INTERNAL; }
    const int rc = restore_file(h, b, rank, world, restored, conflicts);
    close_restore(b);
    return rc;
}

// gcra_snapshot_load: a new table of the file's geometry is filled -- a version 2 file's sections copied slot for slot,
// a version 3 file's entries inserted -- and replaces the engine's table only once every entry is in.  The counters
// are the file's; after a version 3 file len, occupied slots and stash follow the insertion (occupied = len: keys
// without an entry are not in the file).
static int load_file(gcra_engine *h, RestoreBuffers &b) {
    SnapshotHeader hd{};
    SnapSections sec;
    if (const char *why = read_header(b.fd, hd, sec)) { h->err = std::string("snapshot: ") + why; return GCRA_INTERNAL; }
    const Geometry g = table_geometry(hd.capacity, h->tight);
    if (g.total_lines != hd.total_lines || g.nb_main != hd.nb_main || g.stash_slots != hd.stash_slots) {
        h->err = "snapshot: geometry not reproducible with this build/flags";
        return GCRA_INTERNAL;
    }
    RC(make_restore_buffers(h, b));
    HostTable t;
    RC(make_table(h, hd.capacity, t));
    u64 c[C_COUNT];
    memcpy(c, hd.counters, sizeof(c));
    if (hd.version == 2) {
        RC(restore_pass(h, b, t.view, sec, 0, 1, PASS_COPY));
    } else {
        RC(restore_pass(h, b, t.view, sec, 0, 1, PASS_INSERT));
        u64 counts[RESTORE_COUNTS], fresh[C_COUNT];
        CK(cudaMemcpy(counts, b.counts.get(), sizeof(counts), cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(fresh, t.counters.get(), sizeof(fresh), cudaMemcpyDeviceToHost));
        if (counts[RESTORE_FAILED] || counts[RESTORE_CONFLICTS]) {
            h->err = "snapshot: the file's entries do not fit its own geometry (a key twice, or a full table)";
            return GCRA_INTERNAL;
        }
        take_occupancy(c, fresh);
    }
    RC(install_table(h, std::move(t), c));
    h->hash_seed[0] = hd.hash_seed[0];
    h->hash_seed[1] = hd.hash_seed[1];
    h->seen_allowed = c[C_ALLOWED];
    h->seen_expired_hits = c[C_EXPIRED_HITS];
    return GCRA_OK;
}

int32_t gcra_snapshot_load(gcra_engine *h, const char *path) {
    CK(cudaSetDevice(h->device));
    CK(cudaDeviceSynchronize());
    RestoreBuffers b;
    b.fd = open(path, O_RDONLY);
    if (b.fd < 0) { h->err = std::string("snapshot: cannot open ") + path; return GCRA_INTERNAL; }
    const int rc = load_file(h, b);
    close_restore(b);
    return rc;
}

// ---- background snapshot: capture on the GPU at the call's place in submission order, write on a thread ----------
static bool pwrite_all(int fd, const void *buf, size_t bytes, uint64_t off) {
    for (size_t put = 0; put < bytes;) {
        const ssize_t r = pwrite(fd, (const char *)buf + put, bytes - put, (off_t)(off + put));
        if (r <= 0) return false;
        put += (size_t)r;
    }
    return true;
}

// The writer thread's whole job.  It waits only for the staging's own events and stream, so it never holds up the
// engine's traffic or another engine's; the file appears at `path` (rename) only when it is complete and on disk.
static int write_snapshot_file(SnapshotJob *j, SnapshotStaging *sg, int device) {
    cudaError_t e = cudaSuccess;
    auto fail = [&](const std::string &what) {
        j->err = "snapshot: " + what + (e != cudaSuccess ? std::string(": ") + cudaGetErrorString(e) : std::string());
        return GCRA_INTERNAL;
    };
    if ((e = cudaSetDevice(device)) || (e = cudaEventSynchronize(sg->ev_capture.get()))) return fail("capture");
    const u64 n = sg->meta.get()[C_COUNT];
    if (n > j->cap) return fail("more entries than the staging holds");
    SnapshotHeader &hd = j->hd;
    memcpy(hd.counters, sg->meta.get(), sizeof(hd.counters));
    if (!pwrite_all(j->fd, &hd, sizeof(hd), 0) || !pwrite_all(j->fd, &n, sizeof(n), sizeof(hd))) return fail("short write");
    struct Piece { const unsigned char *src; size_t bytes; uint64_t off; };
    std::vector<Piece> pieces;
    const unsigned char *dev = sg->dev.get();
    const Piece sections[3] = {{dev + j->keys_off, n * sizeof(u64), sizeof(hd) + sizeof(n)},
                               {dev + j->state_off, n * sizeof(TatOff), sizeof(hd) + sizeof(n) + n * sizeof(u64)},
                               {dev + j->ei_off, n * sizeof(i64), sizeof(hd) + sizeof(n) + n * (sizeof(u64) + sizeof(TatOff))}};
    for (const Piece &p : sections)
        for (size_t o = 0; o < p.bytes; o += SNAP_CHUNK) pieces.push_back({p.src + o, std::min(SNAP_CHUNK, p.bytes - o), p.off + o});
    // piece i + 1 is copied while piece i is written; its pinned chunk last held piece i - 1, written already
    auto issue = [&](size_t i) {
        const int c = (int)(i & 1);
        if ((e = cudaMemcpyAsync(sg->chunk[c].get(), pieces[i].src, pieces[i].bytes, cudaMemcpyDeviceToHost, sg->stream.get()))) return false;
        return (e = cudaEventRecord(sg->ev_chunk[c].get(), sg->stream.get())) == cudaSuccess;
    };
    if (!pieces.empty() && !issue(0)) return fail("copy");
    for (size_t i = 0; i < pieces.size(); i++) {
        if (i + 1 < pieces.size() && !issue(i + 1)) return fail("copy");
        if ((e = cudaEventSynchronize(sg->ev_chunk[i & 1].get()))) return fail("copy");
        if (!pwrite_all(j->fd, sg->chunk[i & 1].get(), pieces[i].bytes, pieces[i].off)) return fail("short write");
    }
    if (fsync(j->fd) != 0) return fail("fsync");
    const int fd = j->fd;
    j->fd = -1;
    if (close(fd) != 0) return fail("close");
    if (rename(j->tmp.c_str(), j->path.c_str()) != 0) return fail("rename");
    j->entries = n;
    return GCRA_OK;
}

static void snapshot_writer(SnapshotJob *j, SnapshotStaging *sg, int device) {
    j->rc = write_snapshot_file(j, sg, device);
    if (j->rc != GCRA_OK) {
        // the copies may still be reading into the pinned chunks: done before the next save reuses them
        cudaStreamSynchronize(sg->stream.get());
        if (j->fd >= 0) close(j->fd);
        unlink(j->tmp.c_str());
    }
    j->finished.store(true);
}

static int make_snapshot_staging(gcra_engine *h) {
    if (h->snap) return GCRA_OK;
    std::unique_ptr<SnapshotStaging> sg(new SnapshotStaging());
    CK(sg->stream.make());
    for (Event *e : {&sg->ev_store, &sg->ev_capture, &sg->ev_chunk[0], &sg->ev_chunk[1]}) CK(e->make(cudaEventDisableTiming));
    for (auto &c : sg->chunk) CK(c.make(SNAP_CHUNK));
    CK(sg->meta.make(C_COUNT + 1));
    int nb = 0;
    sg->grid = 2 * h->sms;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, snapshot_capture_kernel, TILE_THREADS, 0) == cudaSuccess && nb > 0)
        sg->grid = (uint32_t)nb * h->sms;
    h->snap = std::move(sg);
    return GCRA_OK;
}

// Everything that can fail is done before the capture is enqueued: the temporary file, the staging.
static int snapshot_begin(gcra_engine *h, SnapshotJob &j) {
    CK(cudaSetDevice(h->device));
    RC(make_snapshot_staging(h));
    SnapshotStaging &sg = *h->snap;
    // an upper bound of the entries at the cut, known without waiting for the device
    tighten_occupied_ub(h);
    const uint64_t slots = h->tab.slots(), tiles = (slots + SNAP_TILE - 1) / SNAP_TILE;
    j.cap = std::min<uint64_t>(h->occupied_ub, slots);
    auto up = [](size_t x) { return (x + 255) / 256 * 256; };
    const size_t ctrl_bytes = (SC_STATUS + tiles) * sizeof(u64);
    j.keys_off = up(ctrl_bytes);
    j.state_off = j.keys_off + up(j.cap * sizeof(u64));
    j.ei_off = j.state_off + up(j.cap * sizeof(TatOff));
    const size_t need = j.ei_off + up(j.cap * sizeof(i64));
    if (need > sg.dev_bytes) {
        // Twice the need, so that the bound's drift between saves does not make each save allocate (a large allocation
        // takes tens of ms), but never more than the whole table needs.  The smaller buffer is released in stream
        // order, after the last save's copies.
        const size_t full = j.keys_off + up(slots * sizeof(u64)) + up(slots * sizeof(TatOff)) + up(slots * sizeof(i64));
        const size_t bytes = std::min(up(2 * need), full);
        StreamBuf<unsigned char> fresh;
        CK(fresh.make(bytes, sg.stream.get()));
        sg.dev = std::move(fresh);
        sg.dev_bytes = bytes;
    }
    j.hd = header_of(h, 3);
    // the cut: after every batch submitted so far (their last stage records ev_back) and every Store-trait op
    cudaStream_t st = sg.stream.get();
    RC(order_after_batches(h, st));
    CK(cudaEventRecord(sg.ev_store.get(), h->stream.get()));
    CK(cudaStreamWaitEvent(st, sg.ev_store.get(), 0));
    u64 *ctrl = (u64 *)sg.dev.get();
    CK(cudaMemsetAsync(ctrl, 0, ctrl_bytes, st));
    const uint32_t grid = (uint32_t)std::min<uint64_t>(tiles, sg.grid);
    snapshot_capture_kernel<<<grid, TILE_THREADS, 0, st>>>(h->tab.view, slots, ctrl, (u64 *)(sg.dev.get() + j.keys_off),
                                                         (TatOff *)(sg.dev.get() + j.state_off), (i64 *)(sg.dev.get() + j.ei_off), j.cap);
    h->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(sg.meta.get(), h->tab.view.counters, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(sg.meta.get() + C_COUNT, ctrl + SC_ENTRIES, sizeof(u64), cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(sg.ev_capture.get(), st));
    h->capture_pending = true;
    h->pend_set = -1;          // the next batch's stage 2 waits for every tail: no overlap reaches across the capture
    return GCRA_OK;
}

int32_t gcra_snapshot_begin(gcra_engine *h, const char *path) {
    if (h->job && !h->job->finished.load()) { h->err = "snapshot: a background save is already in flight"; return GCRA_INTERNAL; }
    if (h->job) {                  // a finished save (wait may have joined its writer already)
        if (h->job->writer.joinable()) h->job->writer.join();
        h->job.reset();
    }
    std::unique_ptr<SnapshotJob> j(new SnapshotJob());
    j->path = path;
    std::vector<char> tmpl(j->path.begin(), j->path.end());
    const char suffix[] = ".tmp.XXXXXX";
    tmpl.insert(tmpl.end(), suffix, suffix + sizeof(suffix));
    j->fd = mkstemp(tmpl.data());
    if (j->fd < 0) { h->err = std::string("snapshot: cannot create a file next to ") + path; return GCRA_INTERNAL; }
    j->tmp = tmpl.data();
    fchmod(j->fd, 0644);
    int rc = snapshot_begin(h, *j);
    if (rc == GCRA_OK) {
        try {
            j->writer = std::thread(snapshot_writer, j.get(), h->snap.get(), h->device);
        } catch (const std::exception &) {
            h->err = "snapshot: cannot start the writer thread";
            rc = GCRA_INTERNAL;
        }
    }
    if (rc != GCRA_OK) {
        close(j->fd);
        unlink(j->tmp.c_str());
        return rc;
    }
    h->job = std::move(j);
    return GCRA_OK;
}

int32_t gcra_snapshot_poll(gcra_engine *h, int32_t *done) {
    *done = 1;
    if (!h->job) return GCRA_OK;
    if (!h->job->finished.load()) { *done = 0; return GCRA_OK; }
    if (h->job->rc != GCRA_OK) { h->err = h->job->err; return GCRA_INTERNAL; }
    return GCRA_OK;
}

int32_t gcra_snapshot_wait(gcra_engine *h, uint64_t *entries) {
    if (entries) *entries = 0;
    if (!h->job) return GCRA_OK;
    if (h->job->writer.joinable()) h->job->writer.join();
    if (h->job->rc != GCRA_OK) { h->err = h->job->err; return GCRA_INTERNAL; }
    if (entries) *entries = h->job->entries;
    return GCRA_OK;
}


// ---- multi-GPU: the whole sharded tick in native code (one call per tick) ------------------------------
#define NK(call)                                                                              \
    do {                                                                                      \
        int r_ = (call);                                                                      \
        if (r_ != 0) {                                                                        \
            h->err = std::string(#call) + ": " + (nccl_rt::g_api.GetErrorString ? nccl_rt::g_api.GetErrorString(r_) : "nccl error"); \
            return GCRA_INTERNAL;                                                             \
        }                                                                                     \
    } while (0)

int32_t gcra_shard_unique_ids(void *out_3x128) {
    if (!nccl_rt::load()) return GCRA_INTERNAL;
    for (int i = 0; i < 3; i++)
        if (nccl_rt::g_api.GetUniqueId((nccl_rt::UniqueId *)((char *)out_3x128 + 128 * i)) != 0) return GCRA_INTERNAL;
    return GCRA_OK;
}

int32_t gcra_shard_init(gcra_engine *h, int32_t rank, int32_t world, const void *ids_3x128, uint32_t max_rows) {
    CK(cudaSetDevice(h->device));
    if (h->shard) { h->err = "shard already initialised"; return GCRA_INTERNAL; }
    if (world < 1 || world > ROUTE_MAX_SHARDS || rank < 0 || rank >= world) { h->err = "bad rank / world"; return GCRA_INTERNAL; }
    if (max_rows == 0 || max_rows > h->max_batch) { h->err = "max_rows must be in 1..max_batch"; return GCRA_INTERNAL; }
    if (!nccl_rt::load()) { h->err = "libnccl.so.2 not found"; return GCRA_INTERNAL; }
    std::unique_ptr<Shard> sh(new Shard());    // (assigned to the engine only once complete)
    sh->rank = rank; sh->world = world; sh->max_rows = max_rows;
    const nccl_rt::UniqueId *ids = (const nccl_rt::UniqueId *)ids_3x128;
    // one communicator per stage: NCCL runs the operations of ONE communicator in issue order
    NK(sh->comm_counts.make(world, ids[0], rank));
    NK(sh->comm_req.make(world, ids[1], rank));
    NK(sh->comm_res.make(world, ids[2], rank));
    for (Stream *s : {&sh->s_part, &sh->s_route, &sh->s_return}) CK(s->make());
    CK(sh->ev_tmp.make(cudaEventDisableTiming));
    for (auto &sl : sh->slots) {
        CK(sl.routed.make(max_rows));
        // a shard can receive up to world x max_rows rows in one tick (every rank's whole tick): sized for that, so
        // no rank ever has to bail out of a tick its peers have already posted their sends for
        CK(sl.recv_req.make((size_t)world * max_rows));
        CK(sl.recv_res.make((size_t)world * max_rows));
        CK(sl.back_res.make(max_rows));
        CK(sl.src_index.make(max_rows));
        CK(sl.counts_dev.make(2 * ROUTE_MAX_SHARDS));
        CK(sl.counts_host.make(2 * ROUTE_MAX_SHARDS));
        for (Event *e : {&sl.ev_ready, &sl.ev_counts, &sl.ev_routed, &sl.ev_done}) CK(e->make(cudaEventDisableTiming));
        sl.send.resize(world); sl.recv.resize(world); sl.send_off.resize(world); sl.recv_off.resize(world);
    }
    h->shard = std::move(sh);
    return GCRA_OK;
}

// stages 3+4 of a tick: the engine's kernels (pipelined inside the engine) and the way back
static int shard_issue_decide_return(gcra_engine *h) {
    Shard *sh = h->shard.get();
    if (sh->pending < 0) return GCRA_OK;
    ShardSlot &sl = sh->slots[sh->pending];
    sh->pending = -1;
    const int W = sh->world;
    cudaEvent_t done = nullptr;
    // (more rows than one engine batch carries: several batches, cut anywhere -- the order is kept)
    for (uint32_t a = 0; a < sl.n_recv || a == 0; a += h->max_batch) {
        const uint32_t m = std::min<uint32_t>(sl.n_recv - a, h->max_batch);
        cudaEvent_t dn = nullptr;
        RC(launch_pipelined(h, m, sl.recv_req.get() + a, FMT_48_32, 0, sl.recv_res.get() + a, sl.ev_routed.get(), &dn));
        if (dn) { done = dn; CK(cudaStreamWaitEvent(sh->s_return.get(), dn, 0)); }
        if (sl.n_recv == 0) break;
    }
    if (!done) CK(cudaStreamWaitEvent(sh->s_return.get(), sl.ev_routed.get(), 0));
    NK(nccl_rt::g_api.GroupStart());
    for (int p = 0; p < W; p++) {
        // results of the rows peer p sent me go back to p; my own rows' results arrive in partition order
        NK(nccl_rt::g_api.Send(sl.recv_res.get() + sl.recv_off[p], sl.recv[p] * sizeof(gcra_result), nccl_rt::kUint8, p, sh->comm_res.get(), sh->s_return.get()));
        NK(nccl_rt::g_api.Recv(sl.back_res.get() + sl.send_off[p], sl.send[p] * sizeof(gcra_result), nccl_rt::kUint8, p, sh->comm_res.get(), sh->s_return.get()));
    }
    NK(nccl_rt::g_api.GroupEnd());
    if (sl.n) {
        route_unpermute_kernel<<<(sl.n + TILE_THREADS - 1) / TILE_THREADS, TILE_THREADS, 0, sh->s_return.get()>>>(
            sl.back_res.get(), sl.src_index.get(), sl.n, sl.d_res_user);
        h->launches++;
    }
    CK(cudaEventRecord(sl.ev_done.get(), sh->s_return.get()));
    CK(cudaGetLastError());
    return GCRA_OK;
}

int32_t gcra_shard_submit(gcra_engine *h, uint64_t n64, const gcra_request *d_req, gcra_result *d_res, void *ready_stream) {
    CK(cudaSetDevice(h->device));
    Shard *sh = h->shard.get();
    if (!sh) { h->err = "gcra_shard_init first"; return GCRA_INTERNAL; }
    if (n64 > sh->max_rows) { h->err = "tick larger than max_rows"; return GCRA_INTERNAL; }
    const uint32_t n = (uint32_t)n64;
    const int W = sh->world;
    const int k = (int)(sh->next++ % Shard::DEPTH);
    ShardSlot &sl = sh->slots[k];
    if ((int)sh->pending == k) RC(shard_issue_decide_return(h));
    if (sl.used) CK(cudaStreamWaitEvent(sh->s_part.get(), sl.ev_done.get(), 0));     // the slot's buffers are free again
    sl.used = true; sl.n = n; sl.d_res_user = d_res;
    if (ready_stream) {
        CK(cudaEventRecord(sl.ev_ready.get(), (cudaStream_t)ready_stream));
        CK(cudaStreamWaitEvent(sh->s_part.get(), sl.ev_ready.get(), 0));
    }
    // stage 1: stable partition by owner + count exchange
    if (n) {
        uint32_t tiles = (n + TILE_THREADS - 1) / TILE_THREADS;
        route_count_kernel<<<tiles, TILE_THREADS, 0, sh->s_part.get()>>>(d_req, n, (u32)W, tiles, h->route_counts.get());
        route_scan_kernel<<<1, TILE_THREADS, 0, sh->s_part.get()>>>(h->route_counts.get(), (u32)W, tiles, sl.counts_dev.get());
        route_scatter_kernel<<<tiles, TILE_THREADS, 0, sh->s_part.get()>>>(d_req, n, (u32)W, tiles, h->route_counts.get(), sl.routed.get(), sl.src_index.get());
        h->launches += 3;
    } else {
        CK(cudaMemsetAsync(sl.counts_dev.get(), 0, W * sizeof(u32), sh->s_part.get()));
    }
    NK(nccl_rt::g_api.GroupStart());
    for (int p = 0; p < W; p++) {
        NK(nccl_rt::g_api.Send(sl.counts_dev.get() + p, 1, nccl_rt::kUint32, p, sh->comm_counts.get(), sh->s_part.get()));
        NK(nccl_rt::g_api.Recv(sl.counts_dev.get() + W + p, 1, nccl_rt::kUint32, p, sh->comm_counts.get(), sh->s_part.get()));
    }
    NK(nccl_rt::g_api.GroupEnd());
    CK(cudaMemcpyAsync(sl.counts_host.get(), sl.counts_dev.get(), 2 * W * sizeof(u32), cudaMemcpyDeviceToHost, sh->s_part.get()));
    CK(cudaEventRecord(sl.ev_counts.get(), sh->s_part.get()));
    // while this runs, enqueue the previous tick's engine kernels and its way back
    RC(shard_issue_decide_return(h));
    // stage 2: request all-to-all on its own stream (the partition + count exchange of the NEXT tick overlap
    // it); the counts are the only thing the host waits for
    CK(cudaEventSynchronize(sl.ev_counts.get()));
    CK(cudaStreamWaitEvent(sh->s_route.get(), sl.ev_counts.get(), 0));
    size_t so = 0, ro = 0;
    for (int p = 0; p < W; p++) {
        sl.send[p] = sl.counts_host.get()[p]; sl.recv[p] = sl.counts_host.get()[W + p];
        sl.send_off[p] = so; sl.recv_off[p] = ro;
        so += sl.send[p]; ro += sl.recv[p];
    }
    sl.n_recv = (uint32_t)ro;             // <= world x max_rows, which the buffers hold
    NK(nccl_rt::g_api.GroupStart());
    for (int p = 0; p < W; p++) {
        NK(nccl_rt::g_api.Send(sl.routed.get() + sl.send_off[p], sl.send[p] * sizeof(gcra_request), nccl_rt::kUint8, p, sh->comm_req.get(), sh->s_route.get()));
        NK(nccl_rt::g_api.Recv(sl.recv_req.get() + sl.recv_off[p], sl.recv[p] * sizeof(gcra_request), nccl_rt::kUint8, p, sh->comm_req.get(), sh->s_route.get()));
    }
    NK(nccl_rt::g_api.GroupEnd());
    CK(cudaEventRecord(sl.ev_routed.get(), sh->s_route.get()));
    CK(cudaGetLastError());
    sh->pending = k;
    return GCRA_OK;
}

// make `stream` wait for the results of the tick submitted `ticks_back` submissions ago (0 = the latest);
// only the last DEPTH-1 ticks can be addressed
int32_t gcra_shard_wait_tick(gcra_engine *h, uint32_t ticks_back, void *stream) {
    CK(cudaSetDevice(h->device));
    Shard *sh = h->shard.get();
    if (!sh || ticks_back >= (uint32_t)Shard::DEPTH - 1 || ticks_back >= sh->next) { h->err = "bad tick"; return GCRA_INTERNAL; }
    const int k = (int)((sh->next - 1 - ticks_back) % Shard::DEPTH);
    if (sh->pending == k) RC(shard_issue_decide_return(h));
    if (stream) CK(cudaStreamWaitEvent((cudaStream_t)stream, sh->slots[k].ev_done.get(), 0));
    else CK(cudaEventSynchronize(sh->slots[k].ev_done.get()));
    return GCRA_OK;
}

int32_t gcra_shard_join(gcra_engine *h, void *stream) {
    CK(cudaSetDevice(h->device));
    Shard *sh = h->shard.get();
    if (!sh) { h->err = "gcra_shard_init first"; return GCRA_INTERNAL; }
    RC(shard_issue_decide_return(h));
    CK(cudaEventRecord(sh->ev_tmp.get(), sh->s_return.get()));
    if (stream) CK(cudaStreamWaitEvent((cudaStream_t)stream, sh->ev_tmp.get(), 0));
    else CK(cudaEventSynchronize(sh->ev_tmp.get()));
    return GCRA_OK;
}


// ---- multi-GPU over NVLink peer memory: the whole sharded tick without NCCL and without a host sync ------------
static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// segments of the owner's view of an inbox slot: one per sender, and at least 2 -- a view of one segment is a batch
// whose row count the host knows (BatchView), so world 1 adds an empty second segment (its count stays 0).  Without
// it a world-1 tick, bulk (gcra_p2p_submit) or ring, ran the single-segment path over a view with no rows and failed.
static uint32_t p2p_segs(int world) { return (uint32_t)std::max(world, 2); }

int32_t gcra_p2p_prepare(gcra_engine *h, int32_t rank, int32_t world, uint32_t cap_rows, void *ipc_handle_out_64,
                         void **window_out) {
    CK(cudaSetDevice(h->device));
    if (h->p2p) { h->err = "p2p already prepared"; return GCRA_INTERNAL; }
    if (world < 1 || world > P2P_MAX_WORLD || rank < 0 || rank >= world) { h->err = "bad rank / world"; return GCRA_INTERNAL; }
    if (cap_rows == 0 || cap_rows > (1u << 24)) { h->err = "cap_rows must be in 1..2^24"; return GCRA_INTERNAL; }
    std::unique_ptr<P2P> p(new P2P());    // (assigned to the engine only once complete)
    p->rank = rank; p->world = world;
    p->cap_shift = std::max<uint32_t>(ceil_log2(cap_rows), 10);      // whole resolve tiles per segment
    p->cap = 1u << p->cap_shift;
    if (((uint64_t)world << p->cap_shift) >= INDEX_MAX_ROWS) { h->err = "world * cap_rows too large"; return GCRA_INTERNAL; }
    const size_t seg_rows = (size_t)P2P_DEPTH * world * p->cap;
    p->inbox_off = align_up(sizeof(P2PHeader), 256);
    p->outbox_off = align_up(p->inbox_off + seg_rows * sizeof(gcra_request), 256);
    p->window_bytes = align_up(p->outbox_off + seg_rows * sizeof(gcra_result), 256);
    CK(p->window.make(p->window_bytes));
    CK(cudaMemset(p->window.get(), 0, p->inbox_off));
    CK(cudaMemcpy((char *)p->window.get() + offsetof(P2PHeader, seed), h->hash_seed, sizeof(h->hash_seed),
                  cudaMemcpyHostToDevice));
    if (ipc_handle_out_64) {
        cudaIpcMemHandle_t hd;
        CK(cudaIpcGetMemHandle(&hd, p->window.get()));
        static_assert(sizeof(hd) == 64, "cudaIpcMemHandle_t is 64 bytes");
        memcpy(ipc_handle_out_64, &hd, 64);
    }
    if (window_out) *window_out = p->window.get();
    for (Stream *s : {&p->s_part, &p->s_wait, &p->s_sig, &p->s_return}) CK(s->make());
    for (Event &e : p->ev_t) CK(e.make(cudaEventDefault));
    CK(p->peers_dev.make(1));
    CK(p->tile_counts.make((size_t)ROUTE_MAX_SHARDS * ((p->cap + TILE_THREADS - 1) / TILE_THREADS)));
    for (auto &sl : p->slots) {
        CK(sl.res_loc.make(p->cap));
        CK(sl.counts_dev.make(P2P_MAX_WORLD));
        CK(sl.segs_dev.make(P2P_MAX_WORLD));
        for (Event *e : {&sl.ev_ready, &sl.ev_wait, &sl.ev_done}) CK(e->make(cudaEventDisableTiming));
    }
    // the engine's per-row buffers now span the row-id space of a whole inbox slot
    CK(cudaDeviceSynchronize());
    RC(alloc_index_scratch(h, (uint32_t)p2p_segs(world) << p->cap_shift));
    h->p2p = std::move(p);
    return GCRA_OK;
}

// every rank's window: `ipc_handles` (world x 64 bytes, other processes) or `windows` (world pointers valid in THIS
// process: engines that share a process, on one GPU or several -- a window on another device gets peer access)
int32_t gcra_p2p_connect(gcra_engine *h, const void *ipc_handles, void *const *windows) {
    CK(cudaSetDevice(h->device));
    P2P *p = h->p2p.get();
    if (!p) { h->err = "gcra_p2p_prepare first"; return GCRA_INTERNAL; }
    if (!ipc_handles && !windows) { h->err = "need ipc handles or window pointers"; return GCRA_INTERNAL; }
    P2PPeers peers{};
    for (int r = 0; r < p->world; r++) {
        void *base = nullptr;
        if (r == p->rank) base = p->window.get();
        else if (windows) {
            base = windows[r];
            cudaPointerAttributes at;
            CK(cudaPointerGetAttributes(&at, base));
            if (at.type == cudaMemoryTypeDevice && at.device != h->device) {
                const cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);
                if (e == cudaErrorPeerAccessAlreadyEnabled) (void)cudaGetLastError();
                else CK(e);
            }
        } else {
            cudaIpcMemHandle_t hd;
            memcpy(&hd, (const char *)ipc_handles + 64 * r, 64);
            CK(p->peer_map[r].make(hd));
            base = p->peer_map[r].get();
        }
        peers.hdr[r] = (P2PHeader *)base;
        peers.inbox[r] = (unsigned char *)base + p->inbox_off;
        peers.outbox[r] = (unsigned char *)base + p->outbox_off;
    }
    CK(cudaMemcpy(p->peers_dev.get(), &peers, sizeof(peers), cudaMemcpyHostToDevice));
    p->peers_host = peers;
    for (int d = 0; d < P2P_DEPTH; d++) {
        SegDesc segs[P2P_MAX_WORLD] = {};
        for (int r = 0; r < p->world; r++) {
            // segment r of MY inbox slot d holds sender r's rows; their results go to slot d, segment `rank` of
            // sender r's outbox
            segs[r].req = peers.inbox[p->rank] + (((size_t)d * p->world + r) << p->cap_shift) * sizeof(gcra_request);
            segs[r].res = (gcra_result *)(peers.outbox[r] + (((size_t)d * p->world + p->rank) << p->cap_shift) * sizeof(gcra_result));
        }
        for (int r = p->world; r < (int)p2p_segs(p->world); r++) segs[r] = segs[0];   // (world 1: 0 rows)
        CK(cudaMemcpy(p->slots[d].segs_dev.get(), segs, sizeof(segs), cudaMemcpyHostToDevice));
    }
    p->connected = true;
    return GCRA_OK;
}

// Room in the table for the keys a tick of n rows from this rank may insert.  How many rows arrive is only known on the
// device; with a hash-sharded key space it is about what this rank submitted itself, so 1.25 x that (+ slack) is
// reserved -- a reservation of the full inbox would make the host wait for the device every tick.  Should a tick bring
// more NEW keys than the table has room for, the surplus rows are answered with GCRA_INTERNAL ("table full"), as
// find_or_claim always does; the next tick's check then sees the real occupancy and grows the table.  (A ring tick's n
// is the host's bound of its rows.)
static uint32_t p2p_room(gcra_engine *h, uint32_t n) {
    const P2P *p = h->p2p.get();
    return (uint32_t)std::min<uint64_t>((uint64_t)n + n / 4 + 4096, std::min<uint64_t>((uint64_t)p->world << p->cap_shift, h->max_batch));
}

// first half of a tick: the sender's side (partition + transfer + flags).  n rows at d_req, or, with dev_n, the
// *dev_n <= n rows there (a ring slot's parsed rows: the grids are sized from the bound n).  s_part starts after
// `ready`.
static int p2p_route(gcra_engine *h, uint32_t n, const u32 *dev_n, const gcra_request *d_req, cudaEvent_t ready,
                     bool room_reserved = false) {
    P2P *p = h->p2p.get();
    const uint32_t W = (uint32_t)p->world, me = (uint32_t)p->rank;
    const uint64_t tick = ++p->next_tick;
    const uint32_t d = (uint32_t)((tick - 1) % P2P_DEPTH);
    P2PSlot &sl = p->slots[d];
    // slot d again: its previous tick has been un-permuted here, i.e. every owner is through with my rows of that
    // tick and with my outbox slot
    if (sl.used) CK(cudaStreamWaitEvent(p->s_part.get(), sl.ev_done.get(), 0));
    sl.used = true; sl.n = n; sl.dev_n = dev_n; sl.room_reserved = room_reserved;
    if (ready) CK(cudaStreamWaitEvent(p->s_part.get(), ready, 0));
    // stable partition by owner, rows stored straight into the owners' inboxes, then the flags
    const uint32_t tiles = (n + TILE_THREADS - 1) / TILE_THREADS;
    if (p->timed) CK(cudaEventRecord(p->ev_t[0].get(), p->s_part.get()));
    if (n) {
        if (dev_n)
            route_count_dev_kernel<<<tiles, TILE_THREADS, 0, p->s_part.get()>>>(d_req, n, dev_n, W, tiles, p->tile_counts.get());
        else
            route_count_kernel<<<tiles, TILE_THREADS, 0, p->s_part.get()>>>(d_req, n, W, tiles, p->tile_counts.get());
        p2p_scan_kernel<<<W, TILE_THREADS, 0, p->s_part.get()>>>(p->tile_counts.get(), tiles, sl.counts_dev.get());
        if (dev_n)
            p2p_scatter_dev_kernel<<<tiles, TILE_THREADS, 0, p->s_part.get()>>>(d_req, n, dev_n, W, me, d, p->cap_shift, tiles,
                                                                         p->tile_counts.get(), p->peers_dev.get(), sl.res_loc.get());
        else
            p2p_scatter_kernel<<<tiles, TILE_THREADS, 0, p->s_part.get()>>>(d_req, n, W, me, d, p->cap_shift, tiles, p->tile_counts.get(),
                                                                     p->peers_dev.get(), sl.res_loc.get());
        h->launches += 3;
    } else {
        CK(cudaMemsetAsync(sl.counts_dev.get(), 0, W * sizeof(u32), p->s_part.get()));
    }
    p2p_signal_req_kernel<<<1, 32, 0, p->s_part.get()>>>(p->peers_dev.get(), sl.counts_dev.get(), W, me, d, tick);
    if (p->timed) CK(cudaEventRecord(p->ev_t[1].get(), p->s_part.get()));
    h->launches++;
    CK(cudaGetLastError());
    p->routed_pending = true;
    return GCRA_OK;
}

int32_t gcra_p2p_submit_route(gcra_engine *h, uint64_t n64, const gcra_request *d_req, void *ready_stream) {
    CK(cudaSetDevice(h->device));
    P2P *p = h->p2p.get();
    if (!p || !p->connected) { h->err = "gcra_p2p_prepare / gcra_p2p_connect first"; return GCRA_INTERNAL; }
    if (p->routed_pending) { h->err = "gcra_p2p_submit_finish the previous tick first"; return GCRA_INTERNAL; }
    if (n64 > p->cap) { h->err = "tick larger than cap_rows"; return GCRA_INTERNAL; }
    cudaEvent_t ready = nullptr;
    if (ready_stream) {
        P2PSlot &sl = p->slots[p->next_tick % P2P_DEPTH];     // (the slot this tick takes)
        CK(cudaEventRecord(sl.ev_ready.get(), (cudaStream_t)ready_stream));
        ready = sl.ev_ready.get();
    }
    return p2p_route(h, (uint32_t)n64, nullptr, d_req, ready);
}

// second half: the owner's side (wait for every sender, decide, results into the senders' outboxes, flags) and the
// way back (wait for every owner, results into input order, into d_res); the tick's ev_done follows the last
static int p2p_finish(gcra_engine *h, gcra_result *d_res) {
    P2P *p = h->p2p.get();
    p->routed_pending = false;
    const uint32_t W = (uint32_t)p->world, me = (uint32_t)p->rank;
    const uint64_t tick = p->next_tick;
    const uint32_t d = (uint32_t)((tick - 1) % P2P_DEPTH);
    P2PSlot &sl = p->slots[d];
    P2PHeader *hdr = (P2PHeader *)p->window.get();
    // owner: wait for every sender's rows of this tick, then the engine over the inbox slot as one batch of W
    // segments (row counts in the header); its kernels store the results into the senders' outboxes
    p2p_wait_kernel<<<1, 32, 0, p->s_wait.get()>>>(hdr, 0, W, tick);
    CK(cudaEventRecord(sl.ev_wait.get(), p->s_wait.get()));
    BatchView v{};
    v.req0 = nullptr; v.res0 = nullptr;
    v.segs = sl.segs_dev.get();
    v.dev_counts = &hdr->counts[d][0];
    v.n = 0;
    v.nseg = p2p_segs(p->world);
    v.cap_shift = p->cap_shift;
    cudaEvent_t done = nullptr;
    const uint32_t n_rows = p2p_room(h, sl.n);
    if (p->timed) CK(cudaEventRecord(p->ev_t[2].get(), p->s_wait.get()));
    RC(launch_pipelined_view(h, v, n_rows, FMT_48_32, 0, sl.ev_wait.get(), &done, sl.room_reserved));
    CK(cudaStreamWaitEvent(p->s_sig.get(), done, 0));
    if (p->timed) CK(cudaEventRecord(p->ev_t[3].get(), p->s_sig.get()));
    p2p_signal_res_kernel<<<1, 32, 0, p->s_sig.get()>>>(p->peers_dev.get(), W, me, tick);
    // sender again: every owner's results of this tick are in my outbox -> input order, into the caller's buffer
    p2p_wait_kernel<<<1, 32, 0, p->s_return.get()>>>(hdr, 1, W, tick);
    if (p->timed) CK(cudaEventRecord(p->ev_t[4].get(), p->s_return.get()));
    if (sl.n) {
        const uint32_t tiles = (sl.n + TILE_THREADS - 1) / TILE_THREADS;
        const unsigned char *outbox = (const unsigned char *)p->window.get() + p->outbox_off;
        if (sl.dev_n)
            p2p_unpermute_dev_kernel<<<tiles, TILE_THREADS, 0, p->s_return.get()>>>(outbox, sl.res_loc.get(), sl.n, sl.dev_n, W, d,
                                                                                 p->cap_shift, d_res);
        else
            p2p_unpermute_kernel<<<tiles, TILE_THREADS, 0, p->s_return.get()>>>(outbox, sl.res_loc.get(), sl.n, W, d, p->cap_shift,
                                                                             d_res);
        h->launches++;
    }
    CK(cudaEventRecord(sl.ev_done.get(), p->s_return.get()));
    if (p->timed) { CK(cudaEventRecord(p->ev_t[5].get(), p->s_return.get())); p->timed_valid = true; }
    h->launches += 3;
    CK(cudaGetLastError());
    return GCRA_OK;
}

int32_t gcra_p2p_submit_finish(gcra_engine *h, gcra_result *d_res) {
    CK(cudaSetDevice(h->device));
    P2P *p = h->p2p.get();
    if (!p || !p->routed_pending || p->ring_slot_pending >= 0) { h->err = "gcra_p2p_submit_route first"; return GCRA_INTERNAL; }
    return p2p_finish(h, d_res);
}

// stage times (ms) of the most recent tick submitted with timing on (gcra_p2p_set_timing(h, 1)) -- meaningful when
// ticks are run one at a time (submit, join): [0] partition + transfer + flags, [1] until every sender's rows are
// here (includes the other ranks' skew), [2] the engine over the inbox, [3] until every owner's results are here,
// [4] un-permutation
int32_t gcra_p2p_set_timing(gcra_engine *h, int32_t on) {
    P2P *p = h->p2p.get();
    if (!p) { h->err = "gcra_p2p_prepare first"; return GCRA_INTERNAL; }
    p->timed = on != 0;
    return GCRA_OK;
}

int32_t gcra_p2p_last_tick_ms(gcra_engine *h, float out[5]) {
    CK(cudaSetDevice(h->device));
    P2P *p = h->p2p.get();
    if (!p || !p->timed_valid) { h->err = "no timed tick yet"; return GCRA_INTERNAL; }
    CK(cudaEventSynchronize(p->ev_t[5].get()));
    for (int i = 0; i < 5; i++) CK(cudaEventElapsedTime(&out[i], p->ev_t[i].get(), p->ev_t[i + 1].get()));
    return GCRA_OK;
}

int32_t gcra_p2p_submit(gcra_engine *h, uint64_t n, const gcra_request *d_req, gcra_result *d_res, void *ready_stream) {
    RC(gcra_p2p_submit_route(h, n, d_req, ready_stream));
    return gcra_p2p_submit_finish(h, d_res);
}

// make `stream` wait for the results of the tick submitted `ticks_back` submissions ago (0 = the latest, < DEPTH)
int32_t gcra_p2p_wait_tick(gcra_engine *h, uint32_t ticks_back, void *stream) {
    CK(cudaSetDevice(h->device));
    P2P *p = h->p2p.get();
    if (!p || ticks_back >= (uint32_t)P2P_DEPTH || ticks_back >= p->next_tick) { h->err = "bad tick"; return GCRA_INTERNAL; }
    P2PSlot &sl = p->slots[(p->next_tick - 1 - ticks_back) % P2P_DEPTH];
    if (stream) CK(cudaStreamWaitEvent((cudaStream_t)stream, sl.ev_done.get(), 0));
    else CK(cudaEventSynchronize(sl.ev_done.get()));
    return GCRA_OK;
}

int32_t gcra_p2p_join(gcra_engine *h, void *stream) {
    CK(cudaSetDevice(h->device));
    P2P *p = h->p2p.get();
    if (!p) { h->err = "gcra_p2p_prepare first"; return GCRA_INTERNAL; }
    for (auto &sl : p->slots) {
        if (!sl.used) continue;
        if (stream) CK(cudaStreamWaitEvent((cudaStream_t)stream, sl.ev_done.get(), 0));
        else CK(cudaEventSynchronize(sl.ev_done.get()));
    }
    return GCRA_OK;
}

// 1 when a wait on this rank gave up (a peer never delivered a tick): results since then are not to be trusted
int32_t gcra_p2p_error(gcra_engine *h, uint32_t *error) {
    CK(cudaSetDevice(h->device));
    P2P *p = h->p2p.get();
    if (!p) { h->err = "gcra_p2p_prepare first"; return GCRA_INTERNAL; }
    CK(cudaMemcpy(error, (const char *)p->window.get() + offsetof(P2PHeader, error), sizeof(u32), cudaMemcpyDeviceToHost));
    return GCRA_OK;
}

// ---- routing -------------------------------------------------------------------------------------
uint32_t gcra_owner_of(uint64_t key_hash, uint32_t n_shards) { return owner_of(key_hash, n_shards); }

int32_t gcra_route_partition(gcra_engine *h, uint64_t n, const gcra_request *d_req, uint32_t n_shards,
                             gcra_request *d_out, uint32_t *d_src_index, uint32_t *d_counts, void *stream) {
    CK(cudaSetDevice(h->device));
    if (n_shards == 0 || n_shards > ROUTE_MAX_SHARDS || n > h->max_batch) { h->err = "bad shard count / batch size"; return GCRA_INTERNAL; }
    cudaStream_t st = stream ? (cudaStream_t)stream : h->stream.get();
    if (n == 0) { CK(cudaMemsetAsync(d_counts, 0, n_shards * sizeof(u32), st)); return GCRA_OK; }
    uint32_t tiles = (uint32_t)((n + TILE_THREADS - 1) / TILE_THREADS);
    route_count_kernel<<<tiles, TILE_THREADS, 0, st>>>(d_req, (u32)n, n_shards, tiles, h->route_counts.get());
    route_scan_kernel<<<1, TILE_THREADS, 0, st>>>(h->route_counts.get(), n_shards, tiles, d_counts);
    route_scatter_kernel<<<tiles, TILE_THREADS, 0, st>>>(d_req, (u32)n, n_shards, tiles, h->route_counts.get(), d_out, d_src_index);
    h->launches += 3;
    CK(cudaGetLastError());
    return GCRA_OK;
}

int32_t gcra_route_unpermute(gcra_engine *h, uint64_t n, const gcra_result *d_res_routed, const uint32_t *d_src_index,
                             gcra_result *d_res, void *stream) {
    CK(cudaSetDevice(h->device));
    if (n == 0) return GCRA_OK;
    cudaStream_t st = stream ? (cudaStream_t)stream : h->stream.get();
    route_unpermute_kernel<<<(uint32_t)((n + TILE_THREADS - 1) / TILE_THREADS), TILE_THREADS, 0, st>>>(
        d_res_routed, d_src_index, (u32)n, d_res);
    h->launches++;
    CK(cudaGetLastError());
    return GCRA_OK;
}

}  // extern "C"

#include "gcra_actor.inc"
#include "gcra_resp.inc"
#include "gcra_server.inc"
