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
    uint32_t max_batch;   /* largest number of requests one kernel pass carries (0 -> 1<<20; below 1<<30) */
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

/* Key reference: the key is the bytes [off, off + len) of a byte arena.  It travels in a request row's key_hash field
 * (offset 0 of gcra_request and gcra_request16) until the hash pass (gcra_hash_keys_device) replaces it with the
 * engine's hash of those bytes; rows keep their size.  GCRA_KEY_REF(off, len) is the same 64-bit value. */
typedef struct {
    uint32_t off;
    uint32_t len;
} gcra_key_ref;
#define GCRA_KEY_REF(off, len) (((uint64_t)(uint32_t)(len) << 32) | (uint64_t)(uint32_t)(off))

/* 16-byte result of a compact request: what rate_limiter.rs:208 calls `cur`, plus status and allowed.
 * gcra_expand_results16 turns it into the gcra_result the 32-byte path returns, bit for bit. */
typedef struct {
    int64_t cur_tat_ns;   /* allowed ? new_tat : the tat the request started from; 0 when status != GCRA_OK */
    int32_t status;
    uint8_t allowed;
    uint8_t pad[3];
} gcra_result16;

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
 * key space must share it).  gcra_hash_key stays for trusted / synthetic key universes (tests, benches).
 * Callers that hold key STRINGS need not hash on the host: they put the key bytes in an arena and a key reference
 * (gcra_key_ref) in each row, and the hash pass on the GPU (gcra_hash_keys_device, gcra_rate_limit_batch_keys, the
 * keyed ring, gcra_resp_parse_throttle_keyed) writes exactly gcra_engine_hash_key of those bytes into the row. */
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
/* The hash pass: in n device-resident rows of row_bytes = 48 (gcra_request) or 16 (gcra_request16) bytes, replace
 * every key reference with gcra_engine_hash_key(h, d_keys + off, len), in place, asynchronously on `stream` (NULL =
 * the engine's stream).  Enqueue it in front of any batch call that takes device rows (gcra_rate_limit_batch*_device,
 * the pipelined and the multi-GPU submissions).  Reads nothing outside [d_keys, d_keys + keys_len).  A row whose
 * reference leaves the arena (off + len > keys_len) gets key_hash 0 and now_ns = -1 (48 bytes) or policy =
 * UINT32_MAX (16 bytes): the batch answers it GCRA_INTERNAL, counts it in `errors` and touches no entry. */
int32_t gcra_hash_keys_device(gcra_engine *h, uint64_t n, void *d_rows, uint32_t row_bytes, const void *d_keys,
                              uint64_t keys_len, void *stream);
/* gcra_rate_limit_batch with key references in req[i].key_hash into the host arena `keys` (keys_len bytes): the
 * arena goes to the device once, and the hash pass runs before every chunk.  Same chunking by max_batch and the same
 * sweep policy before every chunk; `req` is not modified. */
int32_t gcra_rate_limit_batch_keys(gcra_engine *h, uint64_t n, const gcra_request *req, const void *keys,
                                   uint64_t keys_len, gcra_result *res);

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
/* compact requests, 16-byte results: the same decisions, table updates, counters and sweeps as the two calls above
 * (same chunking by max_batch, same sweep policy before every chunk), but every result row is a gcra_result16 --
 * half the device-to-host bytes, and no kernel computes remaining / reset_after / retry_after.
 * gcra_expand_results16 derives them on the host. */
int32_t gcra_rate_limit_batch16_r16(gcra_engine *h, uint64_t n, const gcra_request16 *req, int64_t now_ns,
                                    gcra_result16 *res);
int32_t gcra_rate_limit_batch16_r16_device(gcra_engine *h, uint64_t n, const gcra_request16 *d_req, int64_t now_ns,
                                           gcra_result16 *d_res, void *stream);
/* Host only: no handle, no device work, thread-safe, works without a GPU.  out[i] = the gcra_result the 32-byte path
 * returns for row i of a compact batch decided at now_ns, derived from in[i] (rate_limiter.rs:208-238 from cur, the
 * request's quantity and its policy, each policy derived once).  A row with status != GCRA_OK becomes
 * {0, 0, 0, status, 0} without reading the table.  Bit-exact ONLY with the policy table that was registered
 * (gcra_set_policies) when the batch ran: a caller that changes its table keeps the old one until the results of the
 * batches decided under it have been expanded.  Returns GCRA_INTERNAL (and writes status GCRA_INTERNAL into such rows)
 * when an OK row names a policy the table lacks or one that is invalid -- i.e. not the batch's table. */
int32_t gcra_expand_results16(uint64_t n, const gcra_request16 *req, int64_t now_ns, const gcra_policy *policies,
                              uint32_t npol, const gcra_result16 *in, gcra_result *out);

/* ---- pinned host ring: fill a slot in place, submit, collect ---------------------------- */
/* replaces the actor's mpsc channel hand-off (actor.rs:68-82,217-236) for batched callers.
 * Slots are processed strictly in submission order.  mode: 0 -> slots hold gcra_request / gcra_result; 2 -> slots
 * hold gcra_request16 / gcra_result16 (gcra_ring_results16; the D2H copy moves n x 16 bytes); any other value ->
 * gcra_request16 / gcra_result.  Pipelining, the sweep policy on submit and the counters read-back are the same in
 * every mode. */
int32_t gcra_ring_create(gcra_engine *h, uint32_t slots, uint32_t slot_capacity, int32_t mode);
void *gcra_ring_requests(gcra_engine *h, uint32_t slot);        /* pinned, caller fills */
gcra_result *gcra_ring_results(gcra_engine *h, uint32_t slot);  /* pinned, valid after wait; NULL in mode 2 */
gcra_result16 *gcra_ring_results16(gcra_engine *h, uint32_t slot);  /* pinned, valid after wait; NULL unless mode 2 */
int32_t gcra_ring_submit(gcra_engine *h, uint32_t slot, uint32_t n, int64_t now_ns);
int32_t gcra_ring_wait(gcra_engine *h, uint32_t slot);
int32_t gcra_ring_poll(gcra_engine *h, uint32_t slot, int32_t *done);
/* keyed ring: the same ring (any mode) plus a pinned and a device key arena of key_capacity bytes (1 .. 2^32) per
 * slot.  The caller writes key bytes into gcra_ring_keys(h, slot) and key references into the rows; submit_keyed
 * copies the rows and the first keys_len arena bytes to the device and runs the hash pass before the batch.  Submit
 * (rows that already hold hashes), wait and poll work on a keyed ring as on any other.  keys_len > key_capacity, or a
 * ring without arenas, returns GCRA_INTERNAL and enqueues nothing. */
int32_t gcra_ring_create_keyed(gcra_engine *h, uint32_t slots, uint32_t slot_capacity, int32_t mode,
                               uint64_t key_capacity);
void *gcra_ring_keys(gcra_engine *h, uint32_t slot);             /* pinned, caller fills; NULL unless keyed */
int32_t gcra_ring_submit_keyed(gcra_engine *h, uint32_t slot, uint32_t n, uint64_t keys_len, int64_t now_ns);

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
 * max_keys > 0) a pass over every batch the engine finishes counts its denied requests (status GCRA_OK, allowed 0)
 * per key hash in a device table; gcra_top_denied returns the k most denied (hash, count) pairs, most denied first
 * (ties: smaller hash first), and prunes the table to its max_keys top entries once more than 3 x max_keys keys have
 * accumulated (the reference's cleanup rule).  Keys are hashes here -- the caller of the batch entry points owns the
 * strings; the rings name theirs on the GPU (gcra_ring_metrics, gcra_denied_names).  max_keys = 0 switches tracking off.  max_keys is at most 2^27 (the table holds 16 entries per key, at
 * most 2^31); a larger value, or a failed allocation, returns GCRA_INTERNAL and leaves the previous setting and its
 * counts as they were.
 *   - Multi-GPU: every pipeline counts a denied request on the engine that owns its key (gcra_owner_of): the owner's
 *     batches of gcra_shard_*, of gcra_p2p_* and of gcra_route_* with the caller's own all-to-all, as well as
 *     single-GPU batches.  The ranks' lists therefore hold disjoint keys, and the global top k is the top k of the
 *     ranks' concatenated top-k lists (no count is summed across ranks).  max_keys, the pruning rule and *dropped
 *     are per rank.
 *   - While tracking is on, a peer-memory tick counts its rows before it publishes its results, so the count is on
 *     the tick's path; with tracking off no kernel is launched.
 *   - gcra_top_denied waits for the engine's submitted batches.  On engines of a multi-GPU pipeline call it between
 *     ticks, after gcra_p2p_join (or gcra_shard_join) on every rank, like gcra_snapshot_restore: the engine's
 *     kernels of a tick wait for its peers' rows. */
int32_t gcra_track_denied(gcra_engine *h, uint32_t max_keys);
int32_t gcra_top_denied(gcra_engine *h, uint32_t k, uint64_t *key_hashes, uint64_t *counts, uint32_t *n_out,
                        uint64_t *dropped);
/* table entry of a key after the fact: returns found, tat and expiry (saturated to INT64_MAX) */
int32_t gcra_peek(gcra_engine *h, uint64_t key_hash, int64_t *tat, int64_t *expiry_ns, uint8_t *found);
/* dump the table to a file / load it back (the reference keeps its state in memory only and loses it on
 * restart); decisions after a load are identical to those of the engine that saved.  gcra_snapshot_save writes a
 * version 2 file (every slot); gcra_snapshot_load also reads version 3 files (gcra_snapshot_begin).  A load fills a
 * new table of the file's geometry -- a version 2 file slot for slot, a version 3 file's entries inserted -- that
 * replaces the engine's table only once every entry is in: a failed load leaves the engine as it was. */
int32_t gcra_snapshot_save(gcra_engine *h, const char *path);
int32_t gcra_snapshot_load(gcra_engine *h, const char *path);
/* Insert the entries of a snapshot file (gcra_snapshot_save, any geometry, any source engine) that shard `rank`
 * of `world` owns (gcra_owner_of(key_hash, world) == rank) into this engine's table, next to what it holds.  This is
 * how a deployment changes its GPU count: every new rank restores every old rank's file (world = 1, rank = 0 takes
 * every entry).
 *   - Checked before any change (else GCRA_INTERNAL, engine untouched): the path opens; world > 0 and rank < world;
 *     the header (magic, version 2 or 3, nb_main x 4 + stash_slots <= total_lines x 4); the file length is the header
 *     + total_lines x 4 x (8 + 16 + 8) bytes (version 2), or the header + 8 + n x 32 bytes (version 3, n entries:
 *     gcra_snapshot_begin).  The file's geometry need not be one this build would choose: entries are
 *     re-inserted, not copied.
 *   - Carried: every slot whose key word is >= 2 and whose state is an entry (expiry = tat + off >= 0), expired but
 *     not swept ones included; tat, off and ei verbatim.  Keys that hold no entry (swept, only ever denied) are not.
 *   - The table stores mix64(key_hash), so ownership is decided on the unmixed key word.  The two key hashes whose
 *     mix64 is 0 or 1 share the key words 2 and 3 with the two whose mix64 is 2 or 3 (one entry for both, in any
 *     table); such an entry goes to the owner of the latter.
 *   - A key that already holds an entry here keeps it and counts in *conflicts; every other key is inserted
 *     (*restored).  The table first grows by the usual rule for the entries this shard takes from the file (not for
 *     the file's whole len), then the keys are placed as traffic places them; a key that finds the table full is an
 *     error.
 *   - An engine that holds no entries (len 0) adopts the file's key-hash seed, as gcra_snapshot_load does; otherwise
 *     the seeds must be equal.
 *   - len, occupied slots and stash follow the inserted keys; the traffic totals and the sweep policy's state do not
 *     change.  Memory use is bounded: the file is streamed in chunks.
 * Waits for the engine's submitted work.  Multi-GPU callers restore between ticks, after gcra_p2p_join (or
 * gcra_shard_join) on every rank. */
int32_t gcra_snapshot_restore(gcra_engine *h, const char *path, uint32_t rank, uint32_t world, uint64_t *restored,
                              uint64_t *conflicts);
/* Background snapshot.  The cut is the call's position in submission order: the file holds the table as every batch
 * (ring slot, device / pipelined / sharded / peer-memory submission, Store-trait call) submitted to this engine before
 * the call left it, and no later one.  Returns without waiting for the device.  The capture runs on the GPU after
 * those batches; later batches wait for the capture only (one streaming pass over the table); an engine thread then
 * copies the captured entries to the host and writes them to `path` (written to a temporary file in the same
 * directory, flushed, renamed into place: `path` is either the old file or the complete new one).
 * One background save per engine at a time (a second begin returns GCRA_INTERNAL and leaves the first running).
 *   - The file is version 3: the version 2 header (geometry, capacity, the counters at the cut, the hash seed), a
 *     uint64 entry count n, then keys[n], (tat, off)[n] and ei[n] -- the slots gcra_snapshot_restore carries, in slot
 *     order.  gcra_snapshot_load and gcra_snapshot_restore read it as well as version 2.
 *   - begin fails (GCRA_INTERNAL, engine untouched, nothing written) when it cannot create the temporary file or the
 *     staging buffers, which it makes or reuses before it enqueues anything.
 *   - An error of the writer is reported by poll and wait (gcra_last_error gives its text), on the caller's thread.
 *     A finished save's status and count stay until the next begin.
 *   - gcra_destroy during a save waits for the file first. */
int32_t gcra_snapshot_begin(gcra_engine *h, const char *path);
int32_t gcra_snapshot_poll(gcra_engine *h, int32_t *done);        /* done = 1: no save in flight (finished or none) */
int32_t gcra_snapshot_wait(gcra_engine *h, uint64_t *entries);     /* blocks; the save's status, entries written */
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
 * input index.  All pointers are device pointers except none; asynchronous on `stream`.
 * The partition's per-tile counts live in one scratch buffer per engine, which gcra_shard_submit uses too, whatever
 * stream either is given: an engine's partitions must be ordered, for example issued on one stream. */
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
 * addresses (engines of one process) to gcra_p2p_connect.  Given addresses, connect enables peer access to each
 * window's device that is not the engine's own, so that one process can drive engines on several GPUs.  World 1 is a
 * valid world: the owner decides its one sender's rows (its inbox is viewed as that segment and an empty one). */
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
/* the same walk (same frames, same UTF-8 rule, same stop codes), but no hashing on the host: each key is copied to
 * keys_out at offset *keys_used (in: bytes already used, out: after this call's keys) and the row gets its key
 * reference; the hash pass hashes them on the GPU (e.g. keys_out = the ring slot's arena, then
 * gcra_ring_submit_keyed).  A frame whose key does not fit in keys_cap stops the walk unconsumed with *stop = 3,
 * like max_frames ("slot full").  A key longer than the whole arena never fits: when the walk stops there with
 * *keys_used = 0 and no frame taken, hash that one frame on the host (gcra_resp_parse_throttle, max_frames = 1) and
 * submit it as an unkeyed batch, as resp.process_pipeline_native does. */
int32_t gcra_resp_parse_throttle_keyed(gcra_engine *h, const void *buf, uint64_t len, int64_t now_ns,
                                       uint32_t max_frames, gcra_request *req_out, void *keys_out, uint64_t keys_cap,
                                       uint64_t *keys_used, uint64_t *consumed, uint32_t *n_frames, int32_t *stop);
/* replies of n decided THROTTLE commands, in order (mod.rs:274-285, seconds as types.rs:87-97); needs cap >= 160 n */
uint64_t gcra_resp_format_replies(const gcra_request *req, const gcra_result *res, uint32_t n, void *out,
                                  uint64_t cap);

/* ---- RESP ring: connections' read buffers in, reply bytes out -------------------------------------------------
 * The engine's ring (one per engine: it takes the place of gcra_ring_create; the mixed ring below serves RESP, HTTP
 * and gRPC connections from one ring), whose slots carry bytes instead of
 * rows.  The caller reads its sockets into gcra_resp_ring_input(h, slot) and describes each connection's bytes in
 * gcra_resp_ring_conns(h, slot)[c] = {off, len}, len <= GCRA_RESP_MAX_CONN_BYTES (the reference's MAX_BUFFER_SIZE,
 * redis/mod.rs:83).  Submit parses every connection on the GPU, decides the rows as one batch and writes the replies;
 * gcra_ring_wait / gcra_ring_poll complete the slot as for any ring.
 *
 * Contract: for connection c, in table order, the GPU takes exactly what
 *     gcra_resp_parse_throttle(h, input + off_c, len_c, now_ns, row_capacity - base_c, rows + base_c, ...)
 * takes -- the same rows (key hashes under the engine's seed), consumed, n_frames and stop -- where base_c is the
 * number of rows of the connections before c.  The rows of all connections form one batch in that order.  After
 * wait, gcra_resp_ring_outcome(h, slot)[c] gives consumed, n_frames, stop, and where the connection's replies lie in
 * gcra_resp_ring_replies(h, slot): reply_len bytes at reply_off, one reply per frame, in frame order, each the bytes
 * gcra_resp_format_replies writes for it.  What the caller does at each stop:
 *   0  every byte was a plain THROTTLE frame: send the replies;
 *   1  an incomplete frame follows at `consumed`: keep its bytes and read more;
 *   2  a frame that is not a plain THROTTLE follows at `consumed`: hand that ONE frame to a general RESP parser
 *      (PING, QUIT, RESP-integer arguments, malformed input), then submit the rest again;
 *   3  the slot's row_capacity is used up: submit the rest again (every connection after c also stops with 3 unless it
 *      is empty).
 * Submit validates everything before it enqueues anything: n_conns > max_conns, a connection past in_capacity or
 * longer than GCRA_RESP_MAX_CONN_BYTES, or a slot in flight returns GCRA_INTERNAL and leaves the engine usable.  Like
 * gcra_ring_submit it applies the store's sweep policy first.  The replies travel to the host as they are written
 * (pinned memory written by the kernel): exactly the reply bytes and 32 bytes of outcome per connection cross the
 * link, not a bound. */
#define GCRA_RESP_MAX_CONN_BYTES 65536u
#define GCRA_RESP_REPLY_MAX 160u       /* bytes of reply per row that gcra_resp_ring_replies has room for */
typedef struct {
    uint32_t off, len;                 /* bytes [off, off + len) of the slot's input */
} gcra_resp_conn;
typedef struct {
    uint32_t consumed, n_frames;
    int32_t stop;                      /* 0 .. 3, as gcra_resp_parse_throttle */
    uint32_t reserved;
    uint64_t reply_off, reply_len;     /* the connection's replies in gcra_resp_ring_replies */
} gcra_resp_outcome;
/* slots x (in_capacity bytes of input (1 .. 2^32), max_conns connections (1 .. 65536), row_capacity rows
 * (1 .. max_batch) and row_capacity x GCRA_RESP_REPLY_MAX bytes of replies) */
int32_t gcra_resp_ring_create(gcra_engine *h, uint32_t slots, uint32_t max_conns, uint64_t in_capacity,
                              uint32_t row_capacity);
void *gcra_resp_ring_input(gcra_engine *h, uint32_t slot);                 /* pinned, caller fills */
gcra_resp_conn *gcra_resp_ring_conns(gcra_engine *h, uint32_t slot);       /* pinned [max_conns], caller fills */
int32_t gcra_resp_ring_submit(gcra_engine *h, uint32_t slot, uint32_t n_conns, int64_t now_ns);
void *gcra_resp_ring_replies(gcra_engine *h, uint32_t slot);               /* pinned, valid after wait */
gcra_resp_outcome *gcra_resp_ring_outcome(gcra_engine *h, uint32_t slot);  /* pinned [max_conns], valid after wait */
/* cold path, after wait: the slot's parsed rows and their results (*n rows; GCRA_INTERNAL if cap < *n) */
int32_t gcra_resp_ring_rows(gcra_engine *h, uint32_t slot, gcra_request *req_out, gcra_result *res_out, uint32_t cap,
                            uint32_t *n);

/* ---- batch HTTP ingest: POST /throttle requests -> request rows, results -> responses ----------------------------
 * The HTTP transport's hot request (transport/http.rs:60-73,103-159), the way gcra_resp_parse_throttle takes RESP's.
 * gcra_http_parse_throttle walks `buf` once and writes one request row per plain request: exactly
 * "POST /throttle HTTP/1.1" CRLF, at most 64 header lines "name: value" CRLF with Content-Length (1-5 digits,
 * <= 65536) and Content-Type: application/json once each (names in any case, other headers skipped) and none of
 * Transfer-Encoding, Connection, Expect, Upgrade, the empty line, then a Content-Length body that is one JSON object
 * with the members key (a string without escapes or control bytes, UTF-8), max_burst, count_per_period, period and
 * optionally quantity (null or absent: 1), in any order, each once, integers without fraction or exponent within
 * (-2^63, 2^63), -0 excluded.  Key hashes under the engine's seed (h may be NULL).  It never consumes part of a
 * request.  *stop: 0 the buffer ended on a request boundary, 1 an incomplete request follows (read more), 2 a request
 * follows that is not plain (hand THAT request to a general HTTP parser, e.g. throttlecrab_b200.http, then call
 * again), 3 max_frames reached. */
int32_t gcra_http_parse_throttle(gcra_engine *h, const void *buf, uint64_t len, int64_t now_ns, uint32_t max_frames,
                                 gcra_request *req_out, uint64_t *consumed, uint32_t *n_frames, int32_t *stop);
/* responses of n decided requests, in order: "HTTP/1.1 200 OK" with the compact JSON body
 * {"allowed":..,"limit":..,"remaining":..,"reset_after":..,"retry_after":..} (seconds, types.rs:73-97), or
 * "HTTP/1.1 500 Internal Server Error" with {"error":"Internal server error: Rate limit check failed: ..."}; headers
 * content-type: application/json, content-length, date (the IMF-fixdate of the row's now_ns, whole seconds).
 * Returns the bytes written, 0 if cap < GCRA_HTTP_REPLY_MAX n. */
#define GCRA_HTTP_REPLY_MAX 256u
uint64_t gcra_http_format_replies(const gcra_request *req, const gcra_result *res, uint32_t n, void *out,
                                  uint64_t cap);
/* The engine's ring as an HTTP ring: a RESP ring in everything but its grammar and replies.  Same limits, same
 * validation and the same calls: gcra_resp_ring_input, _conns, _submit, _replies, _outcome, _rows, gcra_ring_wait and
 * gcra_ring_poll, with gcra_resp_conn, gcra_resp_outcome and GCRA_RESP_MAX_CONN_BYTES.  Its replies area holds
 * row_capacity x GCRA_HTTP_REPLY_MAX bytes.  Contract: for connection c, in table order, the GPU takes exactly what
 *     gcra_http_parse_throttle(h, input + off_c, len_c, now_ns, row_capacity - base_c, rows + base_c, ...)
 * takes, base_c being the rows of the connections before c; the connection's replies are the bytes
 * gcra_http_format_replies writes for its rows.  What the caller does at each stop:
 *   0  every byte was a plain request: send the responses;
 *   1  an incomplete request follows at `consumed`: keep its bytes and read more;
 *   2  a request that is not plain follows at `consumed`: hand that ONE request to a general HTTP parser (other
 *      routes, other headers, escaped keys, malformed input), then submit the rest again;
 *   3  the slot's row_capacity is used up: submit the rest again. */
int32_t gcra_http_ring_create(gcra_engine *h, uint32_t slots, uint32_t max_conns, uint64_t in_capacity,
                              uint32_t row_capacity);

/* ---- batch gRPC ingest: Throttle calls on HTTP/2 connections -> request rows, results -> response frames ---------
 * The gRPC transport's only call (transport/grpc.rs:148-193, proto/throttlecrab.proto) the way
 * gcra_resp_parse_throttle takes RESP's hot command.  HTTP/2 keeps state per connection, so a connection is described
 * by a gcra_grpc_conn: its bytes (for the ring: in the slot's input) and the state the walk needs.  The host's HPACK
 * decoder owns the dynamic table: dyn_class[k] is the class byte of dynamic index 62 + k (gcra_grpc_header_class of
 * the entry's name and value | gcra_grpc_header_class of its name alone << 4), and it rewrites them only when the
 * general path changed the table.  send_window is the connection's send window, init_window the peer's
 * SETTINGS_INITIAL_WINDOW_SIZE (every new stream's send window).
 *
 * gcra_grpc_parse_throttle walks `buf` once and writes one request row per plain call (the grammar: gcra_grpc.cuh):
 * HEADERS on a new odd stream with an HPACK block of indexed fields and literals that leave the table as it is,
 * :method POST, :path /throttlecrab.RateLimiter/Throttle and content-type application/grpc[+proto]; then one DATA
 * frame with an uncompressed ThrottleRequest (END_STREAM, or an empty DATA(END_STREAM) after it); in between only
 * WINDOW_UPDATE and at most one PING per walk.  The row is the message as prost decodes it: absent fields are 0 (so
 * quantity defaults to 0, grpc.rs:158-165), int32 fields sign-extended, the key UTF-8.  stream_ids_out[k] is row k's
 * stream.  WINDOW_UPDATE and PING frames between calls are taken on their own, so `consumed` can cover frames that
 * make no row.  A call is taken only if the windows can take its response: the peer's stream window (init_window plus
 * the stream's WINDOW_UPDATEs) and the connection's send window (after the WINDOW_UPDATEs so far) must hold the
 * largest response DATA (GCRA_GRPC_RESPONSE_DATA_MAX) of this call and of every call before it.  *out receives
 * consumed, n_frames (calls), stop (0 .. 3 as gcra_resp_parse_throttle), data_octets (the DATA octets taken: the
 * connection owes the peer one WINDOW_UPDATE of that much), ping / ping_opaque (a PING that wants its ACK), and the
 * state after the walk: last_stream and send_window before the responses are sent.  The caller subtracts the
 * responses' data_sent from send_window and writes the WINDOW_UPDATE and PING ACK (at most 30 bytes) after the
 * responses.  h (may be NULL) supplies the engine's key-hash seed.  GCRA_INTERNAL if n_dyn > 128 or len >= 2^32. */
#define GCRA_GRPC_MAX_DYN 128u
#define GCRA_GRPC_RESPONSE_DATA_MAX 51u
typedef struct {
    uint32_t off, len;                 /* bytes [off, off + len) of the ring slot's input (the ring only) */
    uint32_t last_stream;              /* the highest client stream id seen so far */
    int32_t send_window;               /* the connection's send window */
    int32_t init_window;               /* the peer's SETTINGS_INITIAL_WINDOW_SIZE */
    uint32_t n_dyn;                    /* dynamic-table entries, <= GCRA_GRPC_MAX_DYN */
    uint8_t dyn_class[GCRA_GRPC_MAX_DYN];
} gcra_grpc_conn;
typedef struct {
    uint32_t consumed, n_frames;
    int32_t stop;
    uint32_t data_octets;              /* DATA octets taken: owed to the peer as a connection WINDOW_UPDATE */
    uint64_t reply_off, reply_len;     /* the ring: the connection's responses in gcra_resp_ring_replies */
    uint32_t last_stream;              /* state out */
    int32_t send_window;               /* state out, before this walk's responses */
    uint32_t data_sent;                /* the ring: the DATA octets of the connection's responses */
    uint32_t ping;                     /* 1: a PING was taken; ACK it with ping_opaque */
    uint8_t ping_opaque[8];
} gcra_grpc_outcome;
int32_t gcra_grpc_parse_throttle(gcra_engine *h, const void *buf, uint64_t len, int64_t now_ns, uint32_t max_frames,
                                 const gcra_grpc_conn *conn, gcra_request *req_out, uint32_t *stream_ids_out,
                                 gcra_grpc_outcome *out);
/* the responses of n decided calls, in order, row k on stream stream_ids[k]: HEADERS(:status 200, content-type:
 * application/grpc), DATA(ThrottleResponse exactly as prost encodes it: fields in number order, zero values omitted,
 * each field `as i32`, seconds as types.rs:87-97) and trailers HEADERS(END_STREAM, grpc-status: 0); for a decide
 * error one trailers-only HEADERS(END_STREAM) with grpc-status: 13 and grpc-message "Rate limiter error: <the
 * actor's error>", percent-encoded (grpc.rs:177-180).  No HPACK state: literals without indexing.  *data_sent (may be
 * NULL) receives the DATA octets written.  Returns the bytes written, 0 if cap < GCRA_GRPC_REPLY_MAX n. */
#define GCRA_GRPC_REPLY_MAX 168u
uint64_t gcra_grpc_format_replies(const gcra_request *req, const gcra_result *res, const uint32_t *stream_ids,
                                  uint32_t n, void *out, uint64_t cap, uint32_t *data_sent);
/* the class of one decoded header field, or of a name alone (value NULL): 0 ignorable, 1 :method POST, 2 the
 * Throttle :path, 3 :scheme, 4 :authority, 5 a gRPC content-type, 6 grpc-encoding: identity, 7 not plain; for a
 * name alone, 8 .. 12 name a header whose value decides (:method, :path, content-type, grpc-encoding, te). */
uint32_t gcra_grpc_header_class(const void *name, uint64_t name_len, const void *value, uint64_t value_len);
/* The engine's ring as a gRPC ring: the RESP ring's slots, calls and validation (gcra_resp_ring_input, _submit,
 * _replies, _rows, gcra_ring_wait, gcra_ring_poll), with gcra_grpc_ring_conns and gcra_grpc_ring_outcome in place of
 * the RESP tables and row_capacity x GCRA_GRPC_REPLY_MAX bytes of replies.  Contract: for connection c, in table
 * order, the GPU takes exactly what
 *     gcra_grpc_parse_throttle(h, input + off_c, len_c, now_ns, row_capacity - base_c, &conns[c], rows + base_c, ...)
 * takes -- the same rows, stream ids, consumed, n_frames, stop, data_octets, ping and state out -- base_c being the
 * rows of the connections before c; its responses are the bytes gcra_grpc_format_replies writes for those rows, and
 * data_sent their DATA octets.  What the caller does at each stop (after sending the responses, the WINDOW_UPDATE for
 * data_octets and the PING ACK, and taking last_stream and send_window - data_sent as the connection's state):
 *   0  every byte was taken: read more;
 *   1  an incomplete frame or call follows at `consumed`: keep its bytes and read more;
 *   2  a frame that is not plain follows at `consumed`: the general HTTP/2 path takes the connection from there and
 *      keeps it until no stream is open; then it hands back the updated state (and class bytes);
 *   3  the slot's row_capacity is used up: submit the rest again.
 * Submit also refuses (GCRA_INTERNAL, nothing enqueued) a connection with n_dyn > GCRA_GRPC_MAX_DYN. */
int32_t gcra_grpc_ring_create(gcra_engine *h, uint32_t slots, uint32_t max_conns, uint64_t in_capacity,
                              uint32_t row_capacity);
gcra_grpc_conn *gcra_grpc_ring_conns(gcra_engine *h, uint32_t slot);       /* pinned [max_conns], caller fills */
gcra_grpc_outcome *gcra_grpc_ring_outcome(gcra_engine *h, uint32_t slot);  /* pinned [max_conns], valid after wait */

/* ---- mixed ring: RESP, HTTP and gRPC connections in one slot, decided as one batch --------------------------------
 * The engine's ring as all three at once, so that one server serves every transport against one table, one submit
 * per tick: every connection parsed in one launch, whatever its protocol, all rows decided as ONE batch, all replies
 * written in one launch.  The caller describes connection c in gcra_mixed_ring_conns(h, slot)[c]: its bytes in
 * gcra_resp_ring_input, its protocol and, for a gRPC connection, grpc_state = k, the row of gcra_grpc_ring_conns
 * (h, slot) that holds its HTTP/2 state (whose off and len are not read) and of gcra_grpc_ring_outcome(h, slot) that
 * receives its outcome.  Every other call is the rings' own: gcra_resp_ring_input, _submit, _replies, _outcome, _rows,
 * gcra_ring_wait and gcra_ring_poll.  A submit writes the gRPC outcome rows of its gRPC connections only; the rows
 * past them hold what an earlier submit wrote, or zeros (every ring's replies and outcomes start zeroed).
 *
 * Contract: for connection c, in table order, with base_c the rows of the connections before it, the GPU takes
 * exactly what its protocol's host walk takes at max_frames = row_capacity - base_c:
 *     GCRA_PROTO_RESP  gcra_resp_parse_throttle,
 *     GCRA_PROTO_HTTP  gcra_http_parse_throttle,
 *     GCRA_PROTO_GRPC  gcra_grpc_parse_throttle with gcra_grpc_ring_conns(h, slot)[grpc_state]
 * -- the same rows (key hashes under the engine's seed, so one key string is one entry from every transport),
 * consumed, n_frames and stop.  All rows of a submit form one batch, in table order.  After wait,
 * gcra_resp_ring_outcome(h, slot)[c] gives every connection's consumed, n_frames, stop, reply_off and reply_len; its
 * replies are the bytes its protocol's formatter writes for its rows (gcra_resp_format_replies,
 * gcra_http_format_replies, or gcra_grpc_format_replies with the stream ids).  gcra_grpc_ring_outcome(h, slot)[k] gets
 * everything a gRPC ring writes for the gRPC connection whose grpc_state is k (data_octets, data_sent, ping, the state
 * out).  Stop codes are each protocol's ring's.  A stop 3 in any connection leaves no rows to every later connection,
 * whatever its protocol: a RESP or HTTP connection with bytes stops with 3, and a gRPC connection where its walk at
 * max_frames 0 stops (3 at its first call, or 2 at a frame that is not plain before it).  The replies area holds
 * row_capacity x GCRA_HTTP_REPLY_MAX bytes (the longest reply).
 *
 * Submit validates everything before it enqueues anything, and returns GCRA_INTERNAL leaving the engine usable, for:
 * a protocol outside 1 .. 3; grpc_state values that are not 0, 1, 2, ... in table order among the gRPC connections;
 * a gRPC state with n_dyn > GCRA_GRPC_MAX_DYN; n_conns > max_conns; a connection past in_capacity or longer than
 * GCRA_RESP_MAX_CONN_BYTES; a slot in flight.  gcra_ring_submit refuses a mixed ring, gcra_resp_ring_conns returns
 * NULL on it, and a second ring create on the engine is refused as always. */
#define GCRA_PROTO_RESP 1u
#define GCRA_PROTO_HTTP 2u
#define GCRA_PROTO_GRPC 3u
typedef struct {
    uint32_t off, len;                 /* bytes [off, off + len) of the slot's input, len <= GCRA_RESP_MAX_CONN_BYTES */
    uint32_t protocol;                 /* GCRA_PROTO_* */
    uint32_t grpc_state;               /* gRPC only: its row in gcra_grpc_ring_conns / gcra_grpc_ring_outcome */
} gcra_mixed_conn;
/* slots x (in_capacity bytes of input (1 .. 2^32), max_conns connections (1 .. 65536) of any protocol, as many gRPC
 * state and outcome rows, row_capacity rows (1 .. max_batch) and row_capacity x GCRA_HTTP_REPLY_MAX bytes of replies) */
int32_t gcra_mixed_ring_create(gcra_engine *h, uint32_t slots, uint32_t max_conns, uint64_t in_capacity,
                               uint32_t row_capacity);
gcra_mixed_conn *gcra_mixed_ring_conns(gcra_engine *h, uint32_t slot);     /* pinned [max_conns], caller fills */

/* ---- rings over peer memory: N engines' connections served against one hash-sharded table ------------------------
 * gcra_ring_p2p(h, 1) makes every later submit of the engine's RESP, HTTP, gRPC or mixed ring a peer-memory tick
 * (gcra_p2p_*): the slot is parsed on this engine's GPU as always, its rows (their count known only on the device)
 * go to their keys' owners, each owner decides its inbox as one batch, and the results come back into the slot's row
 * order, where the reply and outcome kernels write replies and outcomes as for any ring.  It refuses (GCRA_INTERNAL,
 * the engine as it was) when the engine is not gcra_p2p_connect-ed or has no such ring, when row_capacity exceeds the
 * peer-memory cap (the power of two >= cap_rows), when ring metrics are on, or when any rank's key-hash seed differs
 * from this engine's (gcra_p2p_prepare publishes each rank's seed in its window).  gcra_ring_metrics(h, 1) refuses
 * while it is on; sharded ring metrics (gcra_ring_metrics_sharded) run with it.  gcra_ring_p2p(h, 0) returns the ring
 * to the engine's own table.
 *
 * Contract:
 *   - Ring ticks and gcra_p2p_submit ticks form ONE tick sequence per rank.  Every rank submits every tick; a ring
 *     tick of 0 connections is a tick of 0 rows, and rank r's t-th tick may be a ring submit while rank s's is a
 *     gcra_p2p_submit.
 *   - Within a tick, rank r's rows precede rank r+1's, and a rank's rows are in its connection table's order.
 *   - Every connection takes what its protocol's host walk takes at the row cap of ITS OWN rank's slot (the ring
 *     contracts above); its replies are its protocol's formatter applied to the results decided in that order.
 *   - A refused submit enqueues nothing.  The caller must still submit that tick (e.g. again, or with 0 connections),
 *     or the peers' waits give up (gcra_p2p_error).
 * gcra_resp_ring_submit on such a ring is gcra_resp_ring_submit_route + gcra_resp_ring_submit_finish.  Engines of ONE
 * process (sharded.connect_local, one GPU or several) use the halves, as with gcra_p2p_submit_route / _finish: every
 * engine's route of a tick is enqueued before the first finish, and every engine's finish of a tick before the first
 * route of the next (a route may wait for the device while it makes room in the table, and the device then waits for
 * the finishes already enqueued; a missing one would leave a wait to give up).  Route validates and parses the slot
 * and routes its rows; finish decides this rank's inbox, brings the slot's results back and enqueues the replies and outcomes.  No
 * other tick may be routed on the engine between the two.  gcra_ring_wait / gcra_ring_poll complete the slot after
 * finish.  The engine's store sweep policy is not applied on these ticks (as on gcra_p2p_submit's). */
int32_t gcra_ring_p2p(gcra_engine *h, uint32_t on);
int32_t gcra_resp_ring_submit_route(gcra_engine *h, uint32_t slot, uint32_t n_conns, int64_t now_ns);
int32_t gcra_resp_ring_submit_finish(gcra_engine *h, uint32_t slot);

/* ---- ring metrics: the server's GET /metrics counts and top denied keys by name (metrics.rs:233-310) -------------
 * Only the rings know which transport a row came from, and they never hand key strings to the host.  With ring
 * metrics on, every ring submit (RESP, HTTP, gRPC or mixed ring, created before or after) launches one more kernel on
 * its reply stream, after the replies: it counts the slot's rows per transport by the reference's rules, and names
 * the denied keys of the denied-key table (gcra_track_denied) from the slot's input.
 *   - RESP ("redis"): a row is denied when its status is GCRA_OK and allowed is 0, else allowed -- an -ERR reply
 *     counts as allowed (redis/mod.rs:193-205).  RESP rows are never errors.
 *   - HTTP and gRPC: status != GCRA_OK is an error (the 500 response, grpc-status 13), else allowed or denied.
 *   - A denied row's key hash found in the denied table takes the row's key bytes as its name, once (the first row
 *     to name it wins); a key longer than GCRA_DENIED_NAME_MAX bytes is marked GCRA_NAME_TOO_LONG, as the reference
 *     never tracks such keys (metrics.rs:11,39-41).  A hash that found the table full has no entry to name.
 *   - gcra_top_denied's pruning keeps the surviving keys' names and forgets the rest.
 * Names cost GCRA_DENIED_NAME_MAX + 4 bytes per denied-table entry while both ring metrics and denied tracking are
 * on, so max_keys is then at most GCRA_RING_METRICS_MAX_KEYS (10,000, the reference's MAX_DENIED_KEYS_LIMIT, about
 * 68 MB): gcra_ring_metrics(h, 1) refuses while tracking runs with more, gcra_track_denied refuses more while ring
 * metrics are on.  Both return GCRA_INTERNAL and leave the engine as it was.  Every call here and gcra_top_denied
 * wait for the ring slots in flight and the engine's batches. */
typedef struct { uint64_t allowed, denied, errors; } gcra_transport_counts;
#define GCRA_DENIED_NAME_MAX 256u
#define GCRA_RING_METRICS_MAX_KEYS 10000u
#define GCRA_NAME_UNKNOWN  0xFFFFFFFFu   /* no ring row has named this hash */
#define GCRA_NAME_TOO_LONG 0xFFFFFFFEu   /* the key is longer than GCRA_DENIED_NAME_MAX bytes */
/* on: every later ring submit counts its rows per transport and names its denied keys; switching on zeroes the
 * counts and the names.  off: no kernel is launched and the parse kernels write no key positions; the counts stay
 * readable, the names are released. */
int32_t gcra_ring_metrics(gcra_engine *h, uint32_t on);
/* [0] RESP, [1] HTTP, [2] gRPC: the ring rows counted since ring metrics were switched on */
int32_t gcra_ring_transport_counts(gcra_engine *h, gcra_transport_counts out[3]);
/* for each of n hashes (from gcra_top_denied): lens[i] = its name's length, with the bytes at names + 256 i, or one of
 * the two markers (GCRA_NAME_UNKNOWN also for a hash not in the table, or while ring metrics are off).  Needs denied
 * tracking on.  With sharded ring metrics on (below) it reads that mode's name table instead, and needs no denied
 * tracking. */
int32_t gcra_denied_names(gcra_engine *h, uint32_t n, const uint64_t *key_hashes, char *names, uint32_t *lens);

/* ---- ring metrics for rings whose ticks may be peer-memory ticks (gcra_ring_p2p) ------------------------------------
 * On a peer-memory tick a denied request is counted on its key's owner (gcra_track_denied / gcra_top_denied on every
 * rank), but the key's bytes are only in the input of the rank that parsed the connection.  So this mode keeps three
 * things apart, and the caller joins them at a scrape:
 *   - counts per transport of THIS rank's ring slots (gcra_ring_transport_counts), by gcra_ring_metrics' rules;
 *   - names of the keys this rank's connections saw denied, in a name table of this rank keyed by key hash: a denied
 *     row inserts its key (linear probing from the denied table's home slot, at most 64 probes) and the first row to
 *     name it copies its bytes; a key over GCRA_DENIED_NAME_MAX bytes is marked GCRA_NAME_TOO_LONG.  A key that finds
 *     the table full is not stored, and every denied row of such a key is counted in `full` (rows, not keys: the
 *     table has no room to remember which keys it turned away, so a hot key left out counts once per denial);
 *   - the denied counts, on the owners.
 * Every ring submit runs the metrics kernel after the replies whether ring p2p is on or off (on a peer-memory tick,
 * once the results are back in the slot's row order).  gcra_ring_p2p(h, 1) is accepted in this mode.
 * gcra_ring_metrics(h, 1) and gcra_ring_metrics_sharded(h, 1, .) each refuse while the other is on, max_keys above
 * GCRA_RING_METRICS_MAX_KEYS is refused, and gcra_ring_metrics_sharded refuses between a slot's
 * gcra_resp_ring_submit_route and its _finish (the route decided whether key positions are written); every refusal
 * returns GCRA_INTERNAL and leaves the engine as it was.  Every
 * call here, and gcra_denied_names in this mode, waits for the ring slots in flight and the engine's batches: as with
 * gcra_top_denied, multi-GPU callers query between ticks, after every rank's gcra_ring_wait or join. */
/* on: counts per transport of this rank's slots, names of the keys this rank's connections saw denied in a name table
 * of as many entries as a denied table of max_keys (the power of two >= max(16 max_keys, 1024)); max_keys = 0 counts
 * without names.  Switching on zeroes the counts and empties the table.  off: no kernel is launched, the names are
 * released, the counts stay readable. */
int32_t gcra_ring_metrics_sharded(gcra_engine *h, uint32_t on, uint32_t max_keys);
/* keep the names of these hashes, forget every other (the table is rebuilt, and replaces the old one once complete:
 * a failed call leaves it as it was); *full = denied rows whose key found the table full since the last keep */
int32_t gcra_ring_names_keep(gcra_engine *h, uint32_t n, const uint64_t *key_hashes, uint64_t *full);

/* ---- the server: listeners and connections served through the engine's mixed ring ------------------------------
 * replaces throttlecrab-server's transports (transport/{redis,http,grpc}.rs, main.rs): one loop in the caller's
 * thread listens on up to three ports, reads every connection's bytes, and serves them through the engine's mixed ring
 * (gcra_mixed_ring_create, slot 0) with the caller's general path beside it.  It creates no thread and no process.
 *
 * gcra_server_create(h, listens, n, general, ctx, &srv): listens[0 .. n) give up to three (protocol, host, port), a
 * protocol at most once; port 0 binds an ephemeral port (gcra_server_port tells it).  The sockets are non-blocking,
 * SO_REUSEADDR, backlog 1024.  It refuses (GCRA_INTERNAL, nothing left open, gcra_last_error(h) says why) when the
 * engine's ring is not a mixed ring or its in_capacity is below GCRA_RESP_MAX_CONN_BYTES, a protocol is outside 1 .. 3
 * or listed twice, or a bind fails (e.g. the port is in use).  While the server exists the engine's ring slot 0 is
 * its own.
 *
 * gcra_server_read(srv, timeout_ms) waits up to timeout_ms for the sockets, accepts new connections (their ids are
 * 0, 1, 2, ... in accept order), and reads into each connection's pending bytes, at most GCRA_RESP_MAX_CONN_BYTES
 * (the rings' per-connection limit).  An EOF is recorded.  It sends pending output the sockets now take.
 *
 * gcra_server_serve(srv, now_ns) serves the pending bytes at one clock: exactly mixed.process_connections(conns,
 * limiter, now_ns, ring) over the open connections with pending bytes, in accept order -- the same rounds, submits
 * and general-path calls -- then sends what the sockets take.  Per connection afterwards:
 *   - a general path's close (QUIT, a RESP protocol error, HTTP/1.0 or Connection: close, a gRPC GOAWAY), or an EOF
 *     received before this serve: its replies are sent, then the socket closes; nothing more is read;
 *   - GCRA_RESP_MAX_CONN_BYTES pending bytes on which the serve made no progress (a request longer than the rings
 *     take): the connection closes (counters.full_closed);
 *   - more than GCRA_SERVER_READ_PAUSE bytes of unsent output: it is not read until they drain below (one serve adds at
 *     most the replies of 65,536 bytes of requests, so unsent output stays under GCRA_SERVER_OUT_BOUND); unsent
 *     output waits for the socket to take it.
 * A gRPC connection's ring state (gcra_grpc_conn: last_stream, send_window, init_window, class bytes) is kept here:
 * after a ring walk last_stream and send_window - data_sent, and the WINDOW_UPDATE and PING ACK frames appended after
 * its responses; after a general call, what the callback wrote into the row.
 *
 * The general callback runs inside serve, between ring submits, for a connection the ring stopped at a request that
 * is not plain (stop 2), or a gRPC connection that is not plain_ready: general(ctx, conn_id, protocol, data, len,
 * now_ns, grpc, out) with the connection's pending bytes; grpc = its gcra_grpc_conn row for a gRPC connection (read
 * last_stream and send_window from it, write the state back), else NULL.  It fills *out: consumed (<= len), out/out_len
 * (bytes to send, copied before the callback's next call), close, and for gRPC plain_ready.  Consuming nothing means
 * an incomplete request.  It returns 0; anything else, or consumed > len, closes that connection without its unsent
 * output, and serve finishes every other connection's work and then returns GCRA_INTERNAL ("the general path failed on
 * connection N").  When a connection that has had a general call closes, the callback is called once more with data
 * and out NULL: forget its state.
 *
 * gcra_server_poll = read, then serve.  gcra_server_destroy closes every socket and frees the server (the engine and
 * its ring stay).  Known differences from the reference: one clock per serve, where the reference stamps each request;
 * a request longer than 65,536 bytes is not taken (the connection closes), where the reference accepts larger frames.
 *
 * gcra_server_create_sharded(hs, world, listens, n, general, ctx, &srv): the same server over `world` engines of ONE
 * process that share one hash-sharded table (sharded.connect_local, on one GPU or several), hs[r] the engine of rank r.
 * Read, serve, poll, port, stats and destroy are the same calls.  Besides gcra_server_create's refusals it refuses
 * (GCRA_INTERNAL, nothing left open, gcra_last_error(hs[0]) says why, naming the rank) when world is 0, when any
 * engine's ring is not a mixed ring or its in_capacity is below GCRA_RESP_MAX_CONN_BYTES, when any engine is not
 * gcra_p2p_connect-ed with this world, when hs[r]'s peer-memory rank is not r, or when any engine's ring is not
 * switched to peer-memory ticks (gcra_ring_p2p(h, 1)).  While the server exists every engine's ring slot 0 is its own.
 *   - Placement: connection id (accept order, as above) belongs to rank id % world: its bytes go into that rank's slot
 *     0 input, and its replies come from that rank's output.
 *   - gcra_server_serve first runs gcra_policy_tick(hs[r], now_ns) on every rank, in rank order (peer-memory ticks do
 *     not sweep by themselves), then exactly mixed.process_connections_sharded(ranks, now_ns) with ranks[r] rank r's
 *     open connections with pending bytes, in accept order: every tick routes every rank before the first finish and
 *     finishes every rank before the next route; a rank whose connections do not all fit its slot leaves the later
 *     ranks empty ticks; the general paths run after a round's ticks, in the joined order.
 *   - A refused route (e.g. the table cannot grow) still owes the peers its tick: that rank routes 0 connections, every
 *     rank finishes and waits, the connections the other ranks placed get their replies, and serve returns the error.
 *     No connection loses pending bytes, and no peer's wait gives up.
 *   - counters.submits counts ticks.
 * Known differences from one engine: connections are placed round-robin by accept order; within a serve decisions run
 * rank-major (every connection of rank 0, then of rank 1, ...), where one engine decides in accept order; and each
 * engine applies the store's sweep policy to the keys it owns, so the adaptive and probabilistic stores count
 * operations per engine. */
#define GCRA_SERVER_READ_PAUSE (512u << 10)
#define GCRA_SERVER_OUT_BOUND (1u << 20)
typedef struct gcra_server gcra_server;
typedef struct {
    uint32_t protocol;                 /* GCRA_PROTO_RESP, _HTTP or _GRPC */
    uint16_t port;                     /* 0: an ephemeral port */
    uint16_t reserved;
    const char *host;                  /* numeric address, e.g. "0.0.0.0" or "127.0.0.1" */
} gcra_listen;
typedef struct {
    uint64_t consumed;                 /* bytes of data taken */
    const void *out;                   /* bytes to send */
    uint64_t out_len;
    uint32_t close;                    /* 1: close after out is sent */
    uint32_t plain_ready;              /* gRPC: 1 the ring may take the connection */
} gcra_server_general;
typedef int32_t (*gcra_server_general_fn)(void *ctx, uint64_t conn_id, uint32_t protocol, const void *data,
                                          uint64_t len, int64_t now_ns, gcra_grpc_conn *grpc,
                                          gcra_server_general *out);
typedef struct {
    uint64_t open, accepted, closed;   /* connections */
    uint64_t bytes_read, bytes_written;
    uint64_t rounds, submits, general_calls, general_errors;
    uint64_t full_closed;              /* closed with a full buffer on which a serve made no progress */
    uint64_t peak_unsent;              /* the most unsent output any connection held after a serve */
} gcra_server_counters;
int32_t gcra_server_create(gcra_engine *h, const gcra_listen *listens, uint32_t n, gcra_server_general_fn general,
                           void *ctx, gcra_server **out);
int32_t gcra_server_create_sharded(gcra_engine *const *hs, uint32_t world, const gcra_listen *listens, uint32_t n,
                                   gcra_server_general_fn general, void *ctx, gcra_server **out);
uint16_t gcra_server_port(gcra_server *srv, uint32_t protocol);      /* the bound port, 0 if not listening */
int32_t gcra_server_read(gcra_server *srv, int32_t timeout_ms);
int32_t gcra_server_serve(gcra_server *srv, int64_t now_ns);
int32_t gcra_server_poll(gcra_server *srv, int32_t timeout_ms, int64_t now_ns);
int32_t gcra_server_stats(gcra_server *srv, gcra_server_counters *out);
void gcra_server_destroy(gcra_server *srv);

#ifdef __cplusplus
}
#endif
#endif
