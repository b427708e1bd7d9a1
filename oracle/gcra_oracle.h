/*
 * gcra_oracle.h -- CPU restatement of throttlecrab's GCRA hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product:
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * `--impl reference` legs may load this library, and only as the checker or
 * as the timed CPU baseline.  The product path (throttlecrab_b200/) never
 * links, imports or calls it.
 *
 * What it restates (all paths relative to the reference checkout):
 *   throttlecrab/src/core/rate_limiter.rs:102-250      RateLimiter::rate_limit
 *   throttlecrab/src/core/rate/mod.rs:164-176          Rate::from_count_and_period
 *   throttlecrab/src/core/store/adaptive_cleanup.rs:138-278   AdaptiveStore
 *   throttlecrab/src/core/store/periodic.rs:128-209    PeriodicStore
 *   throttlecrab/src/core/store/probabilistic.rs:110-183  ProbabilisticStore
 *
 * Parity pin: the reference is Rust and no Rust toolchain exists in this
 * image, so the reference itself cannot be run.  The restatement is pinned by
 * the reference's own known-answer tests (core/tests.rs, store_test_suite.rs,
 * cleanup_test.rs, rate/tests.rs, redis_test.rs) transcribed as data in
 * tests/golden/ and replayed by tests/test_oracle_*.py.
 */
#ifndef GCRA_ORACLE_H
#define GCRA_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Same layout as gcra_request / gcra_result in include/gcra_b200.h so the
 * tests can hand the same numpy buffers to both sides. */
typedef struct {
    uint64_t key_id;      /* oracle: key string is "k:<key_id>" (decimal)   */
    int64_t max_burst;
    int64_t count_per_period;
    int64_t period;
    int64_t quantity;
    int64_t now_ns;
} ora_request;

typedef struct {
    int64_t remaining;
    int64_t reset_after_ns;
    int64_t retry_after_ns;
    int32_t status;       /* 0 ok, 1 NegativeQuantity, 2 InvalidRateLimit, 3 Internal */
    uint8_t allowed;
    uint8_t pad[3];
} ora_result;

enum { ORA_PERIODIC = 0, ORA_PROBABILISTIC = 1, ORA_ADAPTIVE = 2 };

typedef struct ora_store ora_store;

/* created_ns plays the role of SystemTime::now() inside the constructors
 * (adaptive_cleanup.rs:94, periodic.rs:107).  Pass param = 0 for the library
 * defaults: periodic interval 60 s, probabilistic modulo 1000, adaptive
 * (min 1 s, max 300 s, max_ops 100000). */
ora_store *ora_create(int kind, uint64_t capacity, int64_t created_ns,
                      uint64_t p0, uint64_t p1, uint64_t p2);
void ora_destroy(ora_store *s);

/* Store trait (core/store/mod.rs:85-133). */
int ora_get(ora_store *s, const char *key, uint64_t len, int64_t now_ns, int64_t *value);
int ora_cas(ora_store *s, const char *key, uint64_t len, int64_t old_v, int64_t new_v,
            uint64_t ttl_ns, int64_t now_ns);
int ora_set_nx(ora_store *s, const char *key, uint64_t len, int64_t value,
               uint64_t ttl_ns, int64_t now_ns);

/* Rate::from_count_and_period + the dvt product (rate_limiter.rs:120-122,154-155).
 * Returns 0, or 3 when the reference would panic in `Duration * u32`. */
int ora_derive(int64_t max_burst, int64_t count, int64_t period,
               int64_t *ei_ns, int64_t *dvt_ns);

/* RateLimiter::rate_limit.  Returns the status (also stored in out->status). */
int ora_rate_limit(ora_store *s, const char *key, uint64_t len, int64_t max_burst,
                   int64_t count_per_period, int64_t period, int64_t quantity,
                   int64_t now_ns, ora_result *out);

/* Replay n requests in index order; key string of request i is "k:<key_id>". */
void ora_replay(ora_store *s, uint64_t n, const ora_request *req, ora_result *out);

/* Same, but hash-sharded over `threads` independent stores (the "client-side
 * sharding" the reference docs recommend, README.md:247-249); request i goes to
 * shard key_id % threads, per-shard order = index order.  `stores` has
 * `threads` entries.  Returns wall seconds of the decision loops only. */
double ora_replay_sharded(ora_store **stores, int threads, uint64_t n,
                          const ora_request *req, ora_result *out);

/* Introspection (periodic.rs:113-126 test helpers, plus table state). */
uint64_t ora_len(ora_store *s);
uint64_t ora_expired_count(ora_store *s);
uint64_t ora_sweeps(ora_store *s);
/* writes over an existing, expired entry (set_if_not_exists_with_ttl that found one), every store kind, never reset:
 * what the engine counts as expired_hits */
uint64_t ora_expired_writes(ora_store *s);
/* returns 1 and fills tat / expiry (saturated to INT64_MAX) when the key has an entry */
int ora_entry(ora_store *s, const char *key, uint64_t len, int64_t *tat, int64_t *expiry_sat);
/* force retain(expiry > now) regardless of policy; returns removed */
uint64_t ora_force_sweep(ora_store *s, int64_t now_ns);

#ifdef __cplusplus
}
#endif
#endif
