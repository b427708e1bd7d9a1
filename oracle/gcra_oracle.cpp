/*
 * gcra_oracle.cpp -- CPU restatement of throttlecrab's GCRA hot path.
 * TEST INFRASTRUCTURE ONLY (see gcra_oracle.h for the rules and the parity pin).
 *
 * Every function cites the reference lines it follows.  Rust semantics mirrored:
 * i64 saturating add/sub/mul, `as` casts (f64->u64 saturating truncate, u128->i64
 * truncate, i64->u32 truncate, i64->u64 reinterpret), exact `Duration * u32`,
 * wrapping `+` in release builds, truncating `/`.
 */
#include "gcra_oracle.h"

#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <atomic>
#include <thread>
#include <pthread.h>
#include <sched.h>
#include <vector>

typedef unsigned __int128 u128;
typedef __int128 i128;

/* ---------------------------------------------------------------- i64 helpers */
static inline int64_t sat_add(int64_t a, int64_t b) {
    int64_t r;
    if (__builtin_add_overflow(a, b, &r)) return a < 0 ? INT64_MIN : INT64_MAX;
    return r;
}
static inline int64_t sat_sub(int64_t a, int64_t b) {
    int64_t r;
    if (__builtin_sub_overflow(a, b, &r)) return a < 0 ? INT64_MIN : INT64_MAX;
    return r;
}
static inline int64_t sat_mul(int64_t a, int64_t b) {
    int64_t r;
    if (__builtin_mul_overflow(a, b, &r)) return ((a < 0) != (b < 0)) ? INT64_MIN : INT64_MAX;
    return r;
}
static inline int64_t wrap_add(int64_t a, int64_t b) {
    return (int64_t)((uint64_t)a + (uint64_t)b);
}

/* ---------------------------------------------------------------- the key map
 * Stand-in for ahash::AHashMap<String,(i64,Option<SystemTime>)> over hashbrown
 * (adaptive_cleanup.rs:4-7,40): open addressing, one control byte per bucket
 * (EMPTY / DELETED / FULL+7 hash bits), power-of-two buckets, 7/8 load.  Hash
 * values never leak into results (no iteration order is observable), so the
 * hash function itself is not part of parity. */
struct Entry {
    std::string key;
    int64_t value;
    i128 expiry;  /* now + ttl, exact (SystemTime + Duration never saturates in domain) */
};

static inline uint64_t mix64(uint64_t x) {
    x ^= x >> 32; x *= 0xd6e8feb86659fd93ULL;
    x ^= x >> 32; x *= 0xd6e8feb86659fd93ULL;
    x ^= x >> 32;
    return x;
}
static inline uint64_t hash_bytes(const char *p, uint64_t n) {
    uint64_t h = 0x9E3779B97F4A7C15ULL ^ (n * 0xff51afd7ed558ccdULL);
    while (n >= 8) { uint64_t w; memcpy(&w, p, 8); h = mix64(h ^ w) ; p += 8; n -= 8; h = h * 0x100000001b3ULL + 0x632be59bd9b4e019ULL; }
    if (n) { uint64_t w = 0; memcpy(&w, p, n); h = mix64(h ^ w ^ (n << 56)); }
    return mix64(h);
}

enum : uint8_t { C_EMPTY = 0x80, C_DELETED = 0xFE };

struct Map {
    std::vector<uint8_t> ctrl;
    std::vector<Entry> slots;
    uint64_t mask = 0, items = 0, tombs = 0;

    static uint64_t buckets_for(uint64_t cap) {   /* hashbrown capacity_to_buckets */
        if (cap == 0) return 4;
        if (cap < 8) return cap < 4 ? 4 : 8;
        uint64_t adj = cap * 8 / 7, b = 1;
        while (b < adj) b <<= 1;
        return b;
    }
    uint64_t capacity() const {                   /* bucket_mask_to_capacity */
        uint64_t b = mask + 1;
        return b < 8 ? b - 1 : b / 8 * 7;
    }
    void init(uint64_t cap) {
        uint64_t b = buckets_for(cap);
        ctrl.assign(b, C_EMPTY); slots.clear(); slots.resize(b);
        mask = b - 1; items = 0; tombs = 0;
    }
    void rehash(uint64_t nb) {
        std::vector<uint8_t> oc; oc.swap(ctrl);
        std::vector<Entry> os; os.swap(slots);
        ctrl.assign(nb, C_EMPTY); slots.resize(nb); mask = nb - 1; tombs = 0;
        for (uint64_t i = 0; i < oc.size(); i++) {
            if (oc[i] & 0x80) continue;
            uint64_t h = hash_bytes(os[i].key.data(), os[i].key.size());
            uint64_t p = h & mask;
            while (ctrl[p] != C_EMPTY) p = (p + 1) & mask;
            ctrl[p] = (uint8_t)(h >> 57);
            slots[p] = std::move(os[i]);
        }
    }
    Entry *find(const char *k, uint64_t n, uint64_t h) {
        uint8_t tag = (uint8_t)(h >> 57);
        uint64_t p = h & mask;
        for (;;) {
            uint8_t c = ctrl[p];
            if (c == C_EMPTY) return nullptr;
            if (c == tag) {
                Entry &e = slots[p];
                if (e.key.size() == n && memcmp(e.key.data(), k, n) == 0) return &e;
            }
            p = (p + 1) & mask;
        }
    }
    /* HashMap::insert(key, v): replaces the value and drops the new String when the key exists */
    void insert(std::string &&key, uint64_t h, int64_t value, i128 expiry) {
        Entry *e = find(key.data(), key.size(), h);
        if (e) { e->value = value; e->expiry = expiry; return; /* `key` freed by caller scope */ }
        if (items + tombs + 1 > capacity()) {
            uint64_t nb = mask + 1;
            if (items + 1 > capacity() / 2) nb <<= 1;   /* grow, else rehash in place */
            rehash(nb);
        }
        uint8_t tag = (uint8_t)(h >> 57);
        uint64_t p = h & mask;
        while (!(ctrl[p] & 0x80)) p = (p + 1) & mask;
        if (ctrl[p] == C_DELETED) tombs--;
        ctrl[p] = tag;
        slots[p].key = std::move(key); slots[p].value = value; slots[p].expiry = expiry;
        items++;
    }
    /* HashMap::retain(|_, (_, exp)| exp > now) */
    uint64_t retain_live(i128 now) {
        uint64_t removed = 0;
        for (uint64_t p = 0; p <= mask; p++) {
            if (ctrl[p] & 0x80) continue;
            if (!(slots[p].expiry > now)) {
                uint64_t nx = (p + 1) & mask;
                if (ctrl[nx] == C_EMPTY) ctrl[p] = C_EMPTY; else { ctrl[p] = C_DELETED; tombs++; }
                std::string().swap(slots[p].key);
                items--; removed++;
            }
        }
        return removed;
    }
};

/* ---------------------------------------------------------------- the stores */
static const i128 NS = 1000000000;

struct ora_store {
    int kind;
    Map data;
    /* periodic.rs:40-46 / adaptive_cleanup.rs:39-53 / probabilistic.rs:40-44 */
    i128 next_cleanup = 0;
    i128 cleanup_interval = 0;                 /* periodic */
    i128 min_interval = 0, max_interval = 0, cur_interval = 0;   /* adaptive */
    uint64_t expired_count = 0;
    uint64_t ops_since_cleanup = 0, max_ops = 0;
    uint64_t last_removed = 0, last_total = 0;
    uint64_t ops_count = 0, cleanup_modulo = 0;   /* probabilistic */
    uint64_t sweeps = 0;
    uint64_t expired_writes = 0;                  /* not a reference field: see ora_expired_writes */
};

/* adaptive_cleanup.rs:138-171 */
static bool adaptive_should_clean(const ora_store *s, i128 now) {
    if (now >= s->next_cleanup) return true;
    if (s->ops_since_cleanup >= s->max_ops) return true;
    if (s->expired_count > 50) {
        uint64_t len = s->data.items ? s->data.items : 1;
        double ratio = (double)s->expired_count / (double)len;
        double threshold = (s->last_removed > s->last_total / 4) ? 0.2 / 2.0 : 0.2 * 1.25;
        if (ratio > threshold) return true;
    }
    if (s->data.items > s->data.capacity() * 3 / 4) return true;
    return false;
}
/* adaptive_cleanup.rs:173-203 */
static void adaptive_cleanup(ora_store *s, i128 now) {
    uint64_t initial = s->data.items;
    uint64_t removed = s->data.retain_live(now);
    s->sweeps++;
    if (removed == 0 && s->expired_count == 0) {
        i128 d = s->cur_interval * 2;
        s->cur_interval = d < s->max_interval ? d : s->max_interval;
    } else if ((double)removed > (double)initial * 0.5) {
        i128 d = s->cur_interval / 2;
        s->cur_interval = d > s->min_interval ? d : s->min_interval;
    }
    s->last_removed = removed; s->last_total = initial;
    s->next_cleanup = now + s->cur_interval;
    s->expired_count = 0; s->ops_since_cleanup = 0;
}
/* the `maybe_clean_expired` / `maybe_cleanup` each mutating op starts with */
static void maybe_clean(ora_store *s, i128 now) {
    switch (s->kind) {
    case ORA_PERIODIC:                                    /* periodic.rs:128-142 */
        if (now >= s->next_cleanup) {
            uint64_t before = s->data.items;
            s->data.retain_live(now); s->sweeps++;
            s->expired_count = before - s->data.items;
            s->next_cleanup = now + s->cleanup_interval;
        }
        break;
    case ORA_PROBABILISTIC: {                             /* probabilistic.rs:110-125 */
        s->ops_count += 1;
        uint64_t h = s->ops_count * 2654435761ULL;       /* wrapping_mul */
        if (h % s->cleanup_modulo == 0) { s->data.retain_live(now); s->sweeps++; }
        break;
    }
    default:                                              /* adaptive_cleanup.rs:205-211 */
        s->ops_since_cleanup += 1;
        if (adaptive_should_clean(s, now)) adaptive_cleanup(s, now);
    }
}

extern "C" ora_store *ora_create(int kind, uint64_t capacity, int64_t created_ns,
                                 uint64_t p0, uint64_t p1, uint64_t p2) {
    ora_store *s = new ora_store();
    s->kind = kind;
    /* with_capacity: HashMap::with_capacity((capacity as f64 * 1.3) as usize) */
    s->data.init((uint64_t)((double)capacity * 1.3));
    i128 created = created_ns;
    if (kind == ORA_PERIODIC) {
        s->cleanup_interval = (p0 ? (i128)p0 : 60) * NS;           /* periodic.rs:12 */
        s->next_cleanup = created + s->cleanup_interval;
    } else if (kind == ORA_PROBABILISTIC) {
        s->cleanup_modulo = p0 ? p0 : 1000;                        /* probabilistic.rs:12 */
    } else {
        s->min_interval = (p0 ? (i128)p0 : 1) * NS;                /* adaptive_cleanup.rs:12-15 */
        s->max_interval = (p1 ? (i128)p1 : 300) * NS;
        s->max_ops = p2 ? p2 : 100000;
        s->cur_interval = 5 * NS;
        s->next_cleanup = created + 5 * NS;
    }
    return s;
}
extern "C" void ora_destroy(ora_store *s) { delete s; }

/* Store::get -- adaptive_cleanup.rs:246-252 (periodic.rs:175-181, probabilistic.rs:157-163) */
extern "C" int ora_get(ora_store *s, const char *key, uint64_t len, int64_t now_ns, int64_t *value) {
    Entry *e = s->data.find(key, len, hash_bytes(key, len));
    if (e && e->expiry > (i128)now_ns) { *value = e->value; return 1; }
    return 0;
}
/* Store::compare_and_swap_with_ttl -- adaptive_cleanup.rs:221-244 */
extern "C" int ora_cas(ora_store *s, const char *key, uint64_t len, int64_t old_v, int64_t new_v,
                       uint64_t ttl_ns, int64_t now_ns) {
    i128 now = now_ns;
    maybe_clean(s, now);
    uint64_t h = hash_bytes(key, len);
    Entry *e = s->data.find(key, len, h);
    if (!e) return 0;
    if (e->expiry <= now) { if (s->kind == ORA_ADAPTIVE) s->expired_count++; return 0; }
    if (e->value != old_v) return 0;
    std::string owned(key, len);                       /* key.to_string() :238 */
    s->data.insert(std::move(owned), h, new_v, now + (i128)ttl_ns);
    return 1;
}
/* Store::set_if_not_exists_with_ttl -- adaptive_cleanup.rs:254-278 */
extern "C" int ora_set_nx(ora_store *s, const char *key, uint64_t len, int64_t value,
                          uint64_t ttl_ns, int64_t now_ns) {
    i128 now = now_ns;
    maybe_clean(s, now);
    uint64_t h = hash_bytes(key, len);
    Entry *e = s->data.find(key, len, h);
    if (e && e->expiry > now) return 0;
    if (e && s->kind == ORA_ADAPTIVE) s->expired_count++;           /* :267 */
    if (e) s->expired_writes++;
    std::string owned(key, len);                       /* key.to_string() :269,274 */
    s->data.insert(std::move(owned), h, value, now + (i128)ttl_ns);
    return 1;
}

/* rate/mod.rs:164-176 + rate_limiter.rs:120-122,154-155 */
extern "C" int ora_derive(int64_t max_burst, int64_t count, int64_t period,
                          int64_t *ei_ns, int64_t *dvt_ns) {
    double v = (double)period * 1000000000.0 / (double)count;       /* rate/mod.rs:172 */
    uint64_t ei;                                                    /* f64 as u64 */
    if (std::isnan(v) || v <= 0.0) ei = 0;
    else if (v >= 18446744073709551616.0) ei = UINT64_MAX;
    else ei = (uint64_t)v;
    uint32_t factor = (uint32_t)(uint64_t)(max_burst - 1);          /* (max_burst - 1) as u32 */
    u128 dvt = (u128)ei * (u128)factor;                             /* Duration * u32, exact */
    *ei_ns = (int64_t)ei;                                           /* as_nanos() as i64 */
    *dvt_ns = (int64_t)(uint64_t)dvt;
    /* Duration::mul panics when the whole seconds overflow u64 */
    if (dvt / (u128)1000000000 > (u128)UINT64_MAX) return 3;
    return 0;
}

/* rate_limiter.rs:102-250 */
extern "C" int ora_rate_limit(ora_store *s, const char *key, uint64_t len, int64_t max_burst,
                              int64_t count_per_period, int64_t period, int64_t quantity,
                              int64_t now_ns, ora_result *out) {
    memset(out, 0, sizeof(*out));
    if (quantity < 0) { out->status = 1; return 1; }                              /* :111-113 */
    if (max_burst <= 0 || count_per_period <= 0 || period <= 0) { out->status = 2; return 2; } /* :115-117 */
    int64_t ei, dvt;
    if (ora_derive(max_burst, count_per_period, period, &ei, &dvt)) { out->status = 3; return 3; }
    /* :126-144 -- a pre-epoch `now` makes the reference read the wall clock; outside the
     * deterministic domain, reported as Internal here and by the engine alike. */
    if (now_ns < 0) { out->status = 3; return 3; }

    int64_t stored;
    int have = ora_get(s, key, len, now_ns, &stored);                              /* :151 */
    int64_t tat = have ? std::max(stored, sat_sub(now_ns, dvt))                    /* :158-161 */
                       : sat_sub(now_ns, ei);                                      /* :162-166 */
    int64_t increment = sat_mul(ei, quantity);                                     /* :170 */
    int64_t new_tat = sat_add(tat, increment);                                     /* :171 */
    int64_t allow_at = sat_sub(new_tat, dvt);                                      /* :174 */
    bool allowed = now_ns >= allow_at;                                             /* :175 */
    if (allowed) {
        uint64_t ttl = (uint64_t)sat_add(sat_sub(new_tat, now_ns), dvt);           /* :179-183 */
        int ok = have ? ora_cas(s, key, len, stored, new_tat, ttl, now_ns)         /* :186-189 */
                      : ora_set_nx(s, key, len, new_tat, ttl, now_ns);             /* :190-195 */
        if (!ok) { out->status = 3; return 3; }   /* unreachable single-threaded (:197-204) */
    }
    int64_t cur = allowed ? new_tat : tat;                                         /* :208 */
    int64_t burst_limit = wrap_add(now_ns, dvt);                                   /* :217 */
    int64_t room = sat_sub(burst_limit, cur);                                      /* :218 */
    int64_t remaining = 0;
    if (ei > 0) { remaining = room / ei; if (remaining < 0) remaining = 0; }       /* :221-225 */
    int64_t reset = sat_add(sat_sub(cur, now_ns), dvt);                            /* :227-232 */
    if (reset < 0) reset = 0;
    int64_t retry = 0;
    if (!allowed) { retry = sat_sub(allow_at, now_ns); if (retry < 0) retry = 0; } /* :234-238 */
    out->remaining = remaining; out->reset_after_ns = reset; out->retry_after_ns = retry;
    out->allowed = allowed ? 1 : 0; out->status = 0;
    return 0;
}

static inline uint64_t fmt_key(char *buf, uint64_t id) {
    buf[0] = 'k'; buf[1] = ':';
    char tmp[24]; int n = 0;
    do { tmp[n++] = (char)('0' + id % 10); id /= 10; } while (id);
    for (int i = 0; i < n; i++) buf[2 + i] = tmp[n - 1 - i];
    return (uint64_t)(n + 2);
}

extern "C" void ora_replay(ora_store *s, uint64_t n, const ora_request *req, ora_result *out) {
    char buf[32];
    for (uint64_t i = 0; i < n; i++) {
        uint64_t len = fmt_key(buf, req[i].key_id);
        ora_rate_limit(s, buf, len, req[i].max_burst, req[i].count_per_period, req[i].period,
                       req[i].quantity, req[i].now_ns, &out[i]);
    }
}

extern "C" double ora_replay_sharded(ora_store **stores, int threads, uint64_t n,
                                     const ora_request *req, ora_result *out) {
    if (threads <= 1) {
        auto t0 = std::chrono::steady_clock::now();
        ora_replay(stores[0], n, req, out);
        return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    }
    /* pre-partition (untimed): shard t owns key_id % threads == t, index order kept */
    std::vector<std::vector<uint32_t>> idx(threads);
    for (uint64_t i = 0; i < n; i++) idx[req[i].key_id % (uint64_t)threads].push_back((uint32_t)i);
    /* one pinned thread per store; all threads start together, the clock runs from the common start to the
     * last join (thread creation is not timed) */
    std::vector<std::thread> th;
    std::atomic<int> ready{0};
    std::atomic<bool> go{false};
    cpu_set_t allowed;
    CPU_ZERO(&allowed);
    const bool have_mask = sched_getaffinity(0, sizeof(allowed), &allowed) == 0;
    std::vector<int> cpus;
    if (have_mask) for (int c = 0; c < CPU_SETSIZE; c++) if (CPU_ISSET(c, &allowed)) cpus.push_back(c);
    for (int t = 0; t < threads; t++) {
        th.emplace_back([&, t]() {
            if (!cpus.empty()) {
                cpu_set_t one;
                CPU_ZERO(&one);
                CPU_SET(cpus[t % cpus.size()], &one);
                pthread_setaffinity_np(pthread_self(), sizeof(one), &one);
            }
            ready.fetch_add(1);
            while (!go.load(std::memory_order_acquire)) { }
            char buf[32];
            ora_store *s = stores[t];
            for (uint32_t i : idx[t]) {
                uint64_t len = fmt_key(buf, req[i].key_id);
                ora_rate_limit(s, buf, len, req[i].max_burst, req[i].count_per_period,
                               req[i].period, req[i].quantity, req[i].now_ns, &out[i]);
            }
        });
    }
    while (ready.load() < threads) std::this_thread::yield();
    auto t0 = std::chrono::steady_clock::now();
    go.store(true, std::memory_order_release);
    for (auto &x : th) x.join();
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

extern "C" uint64_t ora_len(ora_store *s) { return s->data.items; }
extern "C" uint64_t ora_expired_count(ora_store *s) { return s->expired_count; }
extern "C" uint64_t ora_sweeps(ora_store *s) { return s->sweeps; }
extern "C" uint64_t ora_expired_writes(ora_store *s) { return s->expired_writes; }
extern "C" int ora_entry(ora_store *s, const char *key, uint64_t len, int64_t *tat, int64_t *expiry_sat) {
    Entry *e = s->data.find(key, len, hash_bytes(key, len));
    if (!e) return 0;
    *tat = e->value;
    *expiry_sat = e->expiry > (i128)INT64_MAX ? INT64_MAX : (int64_t)e->expiry;
    return 1;
}
extern "C" uint64_t ora_force_sweep(ora_store *s, int64_t now_ns) {
    s->sweeps++;
    return s->data.retain_live((i128)now_ns);
}
