/*
 * gcra_b200.h -- C ABI of the H100-native (sm_90a) batched GCRA rate-limit engine.
 *
 * This is the drop-in boundary for ONE path of lazureykis/throttlecrab: the GCRA
 * decide-and-update behind `RateLimiter::rate_limit` over a `Store`, plus the
 * expired-key sweep.  Every entry point names the reference interface it replaces
 * (paths relative to the reference checkout).  Plain pointers and sizes only; no
 * torch / CUDA types in any signature (a `void *stream` is a cudaStream_t, NULL =
 * the engine's own stream).  A handle is single-owner, like the reference's
 * `&mut self` stores (core/store/mod.rs:40-43): no internal locking.
 *
 * The engine never falls back to the CPU: gcra_create fails (GCRA_INTERNAL) when
 * no CUDA device is usable.
 */
#ifndef GCRA_B200_H
#define GCRA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Status codes mirror CellError (core/mod.rs:48-56). */
enum {
    GCRA_OK = 0,
    GCRA_NEGATIVE_QUANTITY = 1,  /* CellError::NegativeQuantity  rate_limiter.rs:111-113 */
    GCRA_INVALID_RATE_LIMIT = 2, /* CellError::InvalidRateLimit  rate_limiter.rs:115-117 */
    GCRA_INTERNAL = 3            /* CellError::Internal(String); see gcra_last_error()   */
};

/* Sweep policy = which reference store the table stands in for. */
enum {
    GCRA_STORE_PERIODIC = 0,      /* PeriodicStore       periodic.rs:128-142        p0 = interval s (0 -> 60)        */
    GCRA_STORE_PROBABILISTIC = 1, /* ProbabilisticStore  probabilistic.rs:110-125   p0 = modulo (0 -> 1000)          */
    GCRA_STORE_ADAPTIVE = 2,      /* AdaptiveStore       adaptive_cleanup.rs:138-211 p0/p1 = min/max s, p2 = max ops */
    GCRA_STORE_MANUAL = 3         /* never sweeps on its own; call gcra_sweep()                                     */
};

/* tests only: size the table at 1x capacity and fill it to 15/16 before growing, so that the
 * second-choice buckets, the stash and table growth are exercised by small traces */
#define GCRA_FLAG_TIGHT_TABLE 1u
/* tests / A-B measurements: which K1 pipeline a batch takes.  Default: batches of >= 32768 requests take the
 * index-order pipeline (probe -> decide in batch order -> resolve -> sorted residue), smaller ones the sort
 * pipeline (ingest -> radix sort by slot -> warp-cooperative decide), <= 255 requests a single-CTA kernel.
 * INDEX_PATH forces the first for every batch above 255 requests, SORT_PATH disables it. */
#define GCRA_FLAG_INDEX_PATH 2u
#define GCRA_FLAG_SORT_PATH 4u
/* draw the key-hash seed from /dev/urandom (see "key identity" below); overrides gcra_config.hash_seed */
#define GCRA_FLAG_RANDOM_SEED 8u

typedef struct gcra_engine gcra_engine;

typedef struct {
    uint64_t capacity;    /* expected live keys, like Store::with_capacity (adaptive_cleanup.rs:91-104) */
    int32_t device;       /* CUDA ordinal */
    int32_t store_kind;   /* GCRA_STORE_* */
    uint64_t p0, p1, p2;  /* policy parameters, 0 = the reference's library default */
    int64_t created_ns;   /* stands in for SystemTime::now() in the constructors (adaptive_cleanup.rs:94) */
    uint32_t max_batch;   /* largest number of requests one kernel pass carries (0 -> 1<<20) */
    uint32_t flags;       /* GCRA_FLAG_* */
    uint64_t hash_seed[2]; /* SipHash key of the string-keyed entry points; (0,0) = the unkeyed gcra_hash_key */
} gcra_config;

/* One call of RateLimiter::rate_limit(key, max_burst, count_per_period, period, quantity, now)
 * (rate_limiter.rs:102-110), the key replaced by its 64-bit hash. 48 bytes. */
typedef struct {
    uint64_t key_hash;
    int64_t max_burst;
    int64_t count_per_period;
    int64_t period;           /* seconds */
    int64_t quantity;
    int64_t now_ns;           /* now.duration_since(UNIX_EPOCH).as_nanos() as i64 (rate_limiter.rs:126-127) */
} gcra_request;

/* (bool, RateLimitResult) (rate_limiter.rs:12-22); `limit` is the request's max_burst. 32 bytes. */
typedef struct {
    int64_t remaining;
    int64_t reset_after_ns;
    int64_t retry_after_ns;
    int32_t status;           /* GCRA_OK or the CellError the reference returns for this request */
    uint8_t allowed;
    uint8_t pad[3];
} gcra_result;

/* Compact request for the policy-table path: 16 bytes over PCIe instead of 48.
 * policy = index into the table registered with gcra_set_policies(); `now` is per call. */
typedef struct {
    uint64_t key_hash;
    int32_t quantity;
    uint32_t policy;
} gcra_request16;

typedef struct {
    int64_t max_burst, count_per_period, period;
} gcra_policy;

typedef struct {
    uint64_t len;             /* entries holding state, like HashMap::len() (periodic.rs:113-116) */
    uint64_t occupied_slots;  /* slots whose key word is taken: len + keys without an entry (swept, or only ever denied) */
    uint64_t table_slots;
    uint64_t stash_entries;
    uint64_t allowed, denied, errors;   /* totals since creation */
    uint64_t expired_hits;    /* writes that replaced an expired entry (adaptive_cleanup.rs:233,267) */
    uint64_t sweeps, swept;   /* sweep launches / entries removed */
    uint64_t grows;
    uint64_t purges;          /* passes that reclaimed the slots of keys without an entry */
    /* index-order K1 pipeline: batches it carried; residue rows (requests that went through the sorted tail) summed
     * over the `residue_batches` batches whose count has reached the host; times stage 2 waited for every tail */
    uint64_t index_batches, residue_rows, residue_batches, drains;
    uint64_t path_switches;   /* times the residue feedback sent the following batches to the sort pipeline */
} gcra_stats;

/* ---- lifetime ------------------------------------------------------------------------- */
/* AdaptiveStore::with_capacity / builders (adaptive_cleanup.rs:91-136, periodic.rs:84-111) */
int32_t gcra_create(const gcra_config *cfg, gcra_engine **out);
void gcra_destroy(gcra_engine *h);
/* text of the last GCRA_INTERNAL on this handle (the String of CellError::Internal) */
const char *gcra_last_error(gcra_engine *h);

/* ---- host helpers (no device work) ---------------------------------------------------- */
/* KEY IDENTITY.  The reference keeps the key String in its map and compares it (adaptive_cleanup.rs:40, a randomly
 * seeded AHashMap).  This table identifies a key by a 64-bit hash ONLY: two keys with the same hash share one entry
 * (one quota).  Among n honest keys that happens with probability ~n^2 / 2^65 (10^8 keys: ~3 * 10^-4).  But
 * gcra_hash_key is UNKEYED and every step of it is invertible: whoever chooses key bytes can construct a key that
 * collides with a victim's, or keys that fill one bucket pair and the stash ("table full" errors for others).  Where
 * keys come from untrusted clients give the engine a secret seed (gcra_config.hash_seed, or GCRA_FLAG_RANDOM_SEED):
 * the string-keyed entry points (gcra_rate_limit, gcra_store_*, gcra_actor_throttle) then hash with SipHash-2-4
 * under that seed, and callers of the batch entry points fill gcra_request.key_hash with gcra_engine_hash_key (or
 * gcra_hash_key_seeded and the seed, which gcra_get_hash_seed returns; a snapshot carries it; engines that shard one
 * key space must share it).  gcra_hash_key stays for trusted / synthetic key universes (tests, benches). */
uint64_t gcra_hash_key(const void *key, uint64_t len);
uint64_t gcra_hash_key_seeded(const void *key, uint64_t len, uint64_t seed0, uint64_t seed1);
uint64_t gcra_engine_hash_key(gcra_engine *h, const void *key, uint64_t len);
void gcra_get_hash_seed(gcra_engine *h, uint64_t out[2]);
/* hash n keys of the form "<prefix><decimal id>" (trace generation: "k:<i>") */
void gcra_hash_key_ids(const void *prefix, uint64_t prefix_len, const uint64_t *ids, uint64_t n,
                       uint64_t *out);
/* Rate::from_count_and_period(..).period() and the dvt product, in i64 ns
 * (rate/mod.rs:164-176, rate_limiter.rs:120-122,154-155).  GCRA_INTERNAL where the reference panics. */
int32_t gcra_derive_params(int64_t max_burst, int64_t count_per_period, int64_t period,
                           int64_t *emission_interval_ns, int64_t *tolerance_ns);

/* ---- Store trait, one key at a time (core/store/mod.rs:85-133) ------------------------- */
/* Store::get (adaptive_cleanup.rs:246-252) */
int32_t gcra_store_get(gcra_engine *h, const void *key, uint64_t len, int64_t now_ns,
                       int64_t *value, uint8_t *found);
/* Store::compare_and_swap_with_ttl (adaptive_cleanup.rs:221-244) */
int32_t gcra_store_cas(gcra_engine *h, const void *key, uint64_t len, int64_t old_value,
                       int64_t new_value, uint64_t ttl_ns, int64_t now_ns, uint8_t *swapped);
/* Store::set_if_not_exists_with_ttl (adaptive_cleanup.rs:254-278) */
int32_t gcra_store_set_nx(gcra_engine *h, const void *key, uint64_t len, int64_t value,
                          uint64_t ttl_ns, int64_t now_ns, uint8_t *stored);

/* ---- RateLimiter::rate_limit ---------------------------------------------------------- */
/* one decision (rate_limiter.rs:102-250); returns the status also written to out->status */
int32_t gcra_rate_limit(gcra_engine *h, const void *key, uint64_t len, int64_t max_burst,
                        int64_t count_per_period, int64_t period, int64_t quantity,
                        int64_t now_ns, gcra_result *out);

/* n decisions with results defined as if the requests were applied in index order -- what the
 * server's actor loop does one message at a time (throttlecrab-server/src/actor.rs:217-236).
 * Host buffers; copies in, runs the kernels, copies out, returns when `res` is filled. */
int32_t gcra_rate_limit_batch(gcra_engine *h, uint64_t n, const gcra_request *req, gcra_result *res);
/* same with device-resident buffers, asynchronous on `stream` (n <= max_batch) */
int32_t gcra_rate_limit_batch_device(gcra_engine *h, uint64_t n, const gcra_request *d_req,
                                     gcra_result *d_res, void *stream);

/* pipelined submission: the batch's ingest + ordering run on an engine stream as soon as `ready_stream`
 * (a cudaStream_t, may be NULL = inputs are ready now) reaches this point, overlapping the decide kernels
 * of the previously submitted batch; decisions are still applied strictly in submission order.  Results
 * of all submitted batches are complete once gcra_pipeline_join() has made `stream` wait for them
 * (stream NULL = block the host). */
int32_t gcra_rate_limit_batch_device_pipelined(gcra_engine *h, uint64_t n, const gcra_request *d_req,
                                               gcra_result *d_res, void *ready_stream);
int32_t gcra_pipeline_join(gcra_engine *h, void *stream);

/* compact requests: register the (max_burst, count, period) table once, then 16-byte requests */
int32_t gcra_set_policies(gcra_engine *h, uint32_t n, const gcra_policy *policies);
int32_t gcra_rate_limit_batch16(gcra_engine *h, uint64_t n, const gcra_request16 *req,
                                int64_t now_ns, gcra_result *res);
int32_t gcra_rate_limit_batch16_device(gcra_engine *h, uint64_t n, const gcra_request16 *d_req,
                                       int64_t now_ns, gcra_result *d_res, void *stream);

/* ---- pinned host ring: fill a slot in place, submit, collect ---------------------------- */
/* replaces the actor's mpsc channel hand-off (actor.rs:68-82,217-236) for batched callers.
 * Slots are processed strictly in submission order. compact != 0 -> slots hold gcra_request16. */
int32_t gcra_ring_create(gcra_engine *h, uint32_t slots, uint32_t slot_capacity, int32_t compact);
void *gcra_ring_requests(gcra_engine *h, uint32_t slot);        /* pinned, caller fills */
gcra_result *gcra_ring_results(gcra_engine *h, uint32_t slot);  /* pinned, valid after wait */
int32_t gcra_ring_submit(gcra_engine *h, uint32_t slot, uint32_t n, int64_t now_ns);
int32_t gcra_ring_wait(gcra_engine *h, uint32_t slot);
int32_t gcra_ring_poll(gcra_engine *h, uint32_t slot, int32_t *done);

/* ---- sweep and introspection ------------------------------------------------------------ */
/* HashMap::retain(expiry > now) (adaptive_cleanup.rs:176-182), unconditionally */
int32_t gcra_sweep(gcra_engine *h, int64_t now_ns, uint64_t *removed);
/* the store kind's own policy (maybe_clean_expired) against the caller's clock: for callers of the device-resident,
 * pipelined and sharded submissions, which -- unlike the host-buffer calls and the ring -- never sweep by themselves
 * (the requests' clocks live on the device).  Waits for the submitted batches; *swept = entries removed. */
int32_t gcra_policy_tick(gcra_engine *h, int64_t now_ns, uint64_t *swept);
/* len() (periodic.rs:113-116) */
uint64_t gcra_len(gcra_engine *h);
int32_t gcra_get_stats(gcra_engine *h, gcra_stats *out);
/* metrics bridge (throttlecrab-server/src/metrics.rs:24-64,162-173: top denied keys).  After gcra_track_denied(h,
 * max_keys > 0) a pass over every finished single-GPU batch counts its denied requests per key hash in a device
 * table; gcra_top_denied returns the k most denied (hash, count) pairs, most denied first, and prunes the table to
 * its max_keys top entries once more than 3 x max_keys keys have accumulated (the reference's cleanup rule).  Keys
 * are hashes here -- the caller of the batch entry points owns the strings.  max_keys = 0 switches tracking off. */
int32_t gcra_track_denied(gcra_engine *h, uint32_t max_keys);
int32_t gcra_top_denied(gcra_engine *h, uint32_t k, uint64_t *key_hashes, uint64_t *counts, uint32_t *n_out,
                        uint64_t *dropped);
/* table entry of a key after the fact: returns found, tat and expiry (saturated to INT64_MAX) */
int32_t gcra_peek(gcra_engine *h, uint64_t key_hash, int64_t *tat, int64_t *expiry_ns, uint8_t *found);
/* dump the table to a file / load it back (the reference keeps its state in memory only and loses it on
 * restart); decisions after a load are identical to those of the engine that saved */
int32_t gcra_snapshot_save(gcra_engine *h, const char *path);
int32_t gcra_snapshot_load(gcra_engine *h, const char *path);
/* block until all device work of this handle has finished */
int32_t gcra_sync(gcra_engine *h);
/* device time (ms) of the kernels of the most recent batch call, measured with CUDA events on
 * the launching stream: [0] total, [1] ingest (hash probe), [2] sort, [3] decide */
int32_t gcra_last_kernel_ms(gcra_engine *h, float out[4]);
/* the most recent batch that took the index-order pipeline on ONE stream (gcra_rate_limit_batch_device): device
 * time (ms) of [0] probe, [1] unused (0), [2] decide in batch order, [3] resolve, [4] bitmap clear + residue-count copy,
 * [5] residue radix sort, [6] residue decide + hot-run kernels */
int32_t gcra_last_kernel_ms_detail(gcra_engine *h, float out[7]);
/* timing experiments only (tools/): a non-zero mask makes pass B of the index-order pipeline skip parts of its work
 * -- results are then WRONG; never set outside a profiling session */
void gcra_debug_set(gcra_engine *h, uint32_t mask);
/* device time (ms) of the most recent sweep kernel (CUDA events on the launching stream) */
int32_t gcra_last_sweep_ms(gcra_engine *h, float *ms);
/* number of kernels this handle has launched since creation */
uint64_t gcra_launch_count(gcra_engine *h);

/* ---- multi-GPU routing (key space hash-sharded across engines, one per GPU) --------------- */
/* owner shard of a key hash among n_shards */
uint32_t gcra_owner_of(uint64_t key_hash, uint32_t n_shards);
/* stable partition of a device-resident batch by owner shard: writes the requests grouped by
 * owner (order inside a group = input order), per-owner counts, and for every output row its
 * input index.  All pointers are device pointers except none; asynchronous on `stream`. */
int32_t gcra_route_partition(gcra_engine *h, uint64_t n, const gcra_request *d_req,
                             uint32_t n_shards, gcra_request *d_out, uint32_t *d_src_index,
                             uint32_t *d_counts, void *stream);
/* inverse: d_res_routed[i] belongs to input row d_src_index[i] */
int32_t gcra_route_unpermute(gcra_engine *h, uint64_t n, const gcra_result *d_res_routed,
                             const uint32_t *d_src_index, gcra_result *d_res, void *stream);

/* ---- the whole sharded tick in native code: one call per tick ------------------------------------------
 * Partition by owner -> count exchange -> request all-to-all -> engine kernels (pipelined) -> result
 * all-to-all -> un-permutation, on three streams with one NCCL communicator per stage (NCCL is resolved
 * with dlopen("libnccl.so.2") at the first call).  Rank 0 creates three ncclUniqueIds
 * (gcra_shard_unique_ids, 3 x 128 bytes), the caller broadcasts them to all ranks by whatever means it
 * has, and every rank calls gcra_shard_init.  Within a tick, rank r's rows precede rank r+1's; ticks are
 * decided in submission order.  d_res is complete once gcra_shard_join() has made `stream` wait (NULL =
 * block the host). */
int32_t gcra_shard_unique_ids(void *out_3x128);
int32_t gcra_shard_init(gcra_engine *h, int32_t rank, int32_t world, const void *ids_3x128, uint32_t max_rows);
int32_t gcra_shard_submit(gcra_engine *h, uint64_t n, const gcra_request *d_req, gcra_result *d_res,
                          void *ready_stream);
int32_t gcra_shard_join(gcra_engine *h, void *stream);
/* make `stream` wait for the results of the tick submitted `ticks_back` submissions ago (0 = latest, < 3) */
int32_t gcra_shard_wait_tick(gcra_engine *h, uint32_t ticks_back, void *stream);

/* ---- the sharded tick over NVLink peer memory: no NCCL in the data path, no host synchronisation -------------
 * Every rank owns a window of device memory (inboxes, outboxes, flags) that all peers map.  The partition kernel
 * stores each request row straight into its owner's inbox, the owner's engine runs over the inbox as one batch of
 * `world` segments and stores every result straight into the sender's outbox, one-warp kernels wait on tick
 * numbers that peers publish with system-scope release stores (csrc/gcra_p2p.cuh).  Same ordering contract as
 * gcra_shard_*: within a tick rank r's rows precede rank r+1's; ticks are decided in submission order; every rank
 * submits every tick.  gcra_p2p_prepare allocates the window (cap_rows = most rows a rank submits per tick) and
 * returns its CUDA IPC handle (64 bytes) and its address; the caller hands all ranks' handles (other processes) or
 * addresses (engines of one process) to gcra_p2p_connect. */
int32_t gcra_p2p_prepare(gcra_engine *h, int32_t rank, int32_t world, uint32_t cap_rows, void *ipc_handle_out_64,
                         void **window_out);
int32_t gcra_p2p_connect(gcra_engine *h, const void *ipc_handles_world_x_64, void *const *windows);
int32_t gcra_p2p_submit(gcra_engine *h, uint64_t n, const gcra_request *d_req, gcra_result *d_res,
                        void *ready_stream);
/* the two halves of gcra_p2p_submit, for callers that drive several engines from ONE process: enqueue the route
 * of every engine before the first finish (a finish enqueues kernels that wait for the other engines' routes) */
int32_t gcra_p2p_submit_route(gcra_engine *h, uint64_t n, const gcra_request *d_req, void *ready_stream);
int32_t gcra_p2p_submit_finish(gcra_engine *h, gcra_result *d_res);
int32_t gcra_p2p_wait_tick(gcra_engine *h, uint32_t ticks_back, void *stream);
int32_t gcra_p2p_join(gcra_engine *h, void *stream);
/* stage times (ms) of the most recent tick submitted while timing was on; meaningful when ticks run one at a time:
 * [0] partition + transfer + flags, [1] until every sender's rows are here, [2] the engine over the inbox,
 * [3] until every owner's results are here, [4] un-permutation */
int32_t gcra_p2p_set_timing(gcra_engine *h, int32_t on);
int32_t gcra_p2p_last_tick_ms(gcra_engine *h, float out[5]);
/* *error = 1 when a wait on this rank gave up after ~20 s (a peer never delivered a tick) */
int32_t gcra_p2p_error(gcra_engine *h, uint32_t *error);

/* ---- the batch-draining actor: per-request callers in front of the batched engine ---------------------------
 * replaces RateLimiterActor / RateLimiterHandle (throttlecrab-server/src/actor.rs:68-82,217-236): one actor thread
 * owns the engine and applies requests strictly in arrival order; gcra_actor_throttle is thread-safe and blocks
 * until its own result is there; everything that queues up while a batch is on the GPU becomes the next batch.
 * buffer_size = the bounded channel (0 -> 100000, the server's --buffer-size), max_batch = most requests per
 * drain (0 -> the engine's max_batch).  While an actor exists it is the ONLY caller of the engine. */
typedef struct gcra_actor gcra_actor;
int32_t gcra_actor_create(gcra_engine *h, uint32_t buffer_size, uint32_t max_batch, gcra_actor **out);
int32_t gcra_actor_throttle(gcra_actor *a, const void *key, uint64_t len, int64_t max_burst,
                            int64_t count_per_period, int64_t period, int64_t quantity, int64_t now_ns,
                            gcra_result *out);
/* out[0] batches run, out[1] requests served, out[2] largest batch */
int32_t gcra_actor_stats(gcra_actor *a, uint64_t out[3]);
void gcra_actor_destroy(gcra_actor *a);

/* ---- batch RESP ingest: a pipelined read buffer -> request rows, results -> reply bytes -------------------------
 * replaces the per-value parse + per-command await of the Redis transport (transport/redis/resp.rs:28-177,
 * redis/mod.rs:128-149,221-295) for its hot command.  gcra_resp_parse_throttle walks `buf` once and writes one
 * request row per plain `THROTTLE key max_burst count_per_period period [quantity]` frame into req_out (e.g. a
 * pinned ring slot); it never consumes part of a frame.  *stop: 0 buffer ended on a frame boundary, 1 an incomplete
 * frame follows, 2 a frame follows that is not a plain THROTTLE (hand THAT frame to a general RESP parser, then call
 * again), 3 max_frames reached.  h (may be NULL) supplies the engine's key-hash seed. */
int32_t gcra_resp_parse_throttle(gcra_engine *h, const void *buf, uint64_t len, int64_t now_ns, uint32_t max_frames,
                                 gcra_request *req_out, uint64_t *consumed, uint32_t *n_frames, int32_t *stop);
/* replies of n decided THROTTLE commands, in order (mod.rs:274-285, seconds as types.rs:87-97); needs cap >= 160 n */
uint64_t gcra_resp_format_replies(const gcra_request *req, const gcra_result *res, uint32_t n, void *out,
                                  uint64_t cap);

#ifdef __cplusplus
}
#endif
#endif
