// gcra_device.cuh -- table layout, exact i64 arithmetic and the GCRA decision (device side).
//
// Follows throttlecrab/src/core/rate_limiter.rs:102-250 (decision), core/rate/mod.rs:164-176
// (emission interval) and core/store/adaptive_cleanup.rs:221-278 (entry liveness / TTL).
#pragma once
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

namespace gcra {

typedef unsigned long long u64;
typedef long long i64;
typedef unsigned int u32;

constexpr u64 KEY_EMPTY = 0;   // slot never used / swept
constexpr u64 KEY_TOMB = 1;    // swept stash slot (stash probing continues past it)
constexpr i64 EXP_EMPTY = -1;  // (tat=0, off=-1): the slot holds no state (free slot, or a key without an entry)
constexpr i64 I64_MAX = 0x7fffffffffffffffLL;
constexpr i64 I64_MIN = (-0x7fffffffffffffffLL - 1);
// An entry's expiry is now + ttl, kept exact in the reference (SystemTime + Duration).  Past I64_MAX it never expires:
// stored as I64_MAX.  Exactly I64_MAX (live up to I64_MAX - 1) has the code EXP_AT_MAX instead, the one negative expiry
// that is an entry; every other negative expiry is "no state".  All readers go through has_state / live_at.
constexpr i64 EXP_AT_MAX = I64_MIN;

// Structure of arrays, one element per slot; a bucket = 4 consecutive slots:
//   keys[slot]   u64   mixed key hash (0 empty, 1 stash tombstone); a bucket's four keys are one
//                      32-byte sector, compared after two 128-bit loads
//   state[slot]  16 B  (tat_ns, burst_offset) -- always read and written together, so one decision is
//                      ONE 128-bit load + ONE 128-bit store, and the sweep streams this array densely
//                      (16 B per slot, coalesced 128-bit loads).  expiry code = tat + off (wrapping, see
//                      EXP_AT_MAX).
//   ei[slot]     i64   emission interval (ns) of the request that created the entry (informational)
// Layout history (profiles/r01_k1_summary.md): v1 kept all four columns of a bucket in one 128-byte
// line; ncu showed 64-byte DRAM fetch granules and a 44-54 %-of-peak sweep, and the probe (ingest
// kernel) and the state update (decide kernel) touch their sectors in different kernels anyway.
struct __align__(16) TatOff {
    i64 tat;   // theoretical arrival time, ns
    u64 off;   // burst offset: expiry - tat (wrapping)
};

enum Counter {
    C_OCCUPIED = 0,   // slots whose key word is taken (entries + keys without an entry)
    C_REAL,           // entries with state (HashMap::len)
    C_ALLOWED,
    C_DENIED,
    C_ERRORS,
    C_EXPIRED_HITS,   // writes over an expired entry (adaptive_cleanup.rs:233,267)
    C_STASH,          // keys living in the stash
    C_INSERT_FAIL,
    C_SWEPT,
    C_COUNT = 16
};

struct Table {
    u64 *keys;        // [slots]   main buckets (nb_main * 4 slots) followed by the stash slots
    TatOff *state;    // [slots]
    i64 *ei;          // [slots]
    u64 *mark;        // [slots]  index-order pipeline: (~batch epoch << 32 | first state-changing row) of the slot
    u32 nb_main;      // buckets addressed by the two hash choices
    u32 stash_slots;  // slots probed linearly when both buckets are full
    u32 null_slot;    // reserved id: "this request has no slot" (last slot of the allocation)
    u32 slot_bits;    // bits needed to sort by slot id
    u64 *counters;    // Counter[C_COUNT]
};

// ------------------------------------------------------------------ exact i64 arithmetic
// (host and device: the host expands 16-byte results with the same outputs_from as the kernels)
__host__ __device__ __forceinline__ i64 sat_add(i64 a, i64 b) {
    i64 r = (i64)((u64)a + (u64)b);
    if (((a ^ r) & (b ^ r)) < 0) r = a < 0 ? I64_MIN : I64_MAX;
    return r;
}
__host__ __device__ __forceinline__ i64 sat_sub(i64 a, i64 b) {
    i64 r = (i64)((u64)a - (u64)b);
    if (((a ^ b) & (a ^ r)) < 0) r = a < 0 ? I64_MIN : I64_MAX;
    return r;
}
__host__ __device__ __forceinline__ i64 sat_mul(i64 a, i64 b) {
    i64 lo = (i64)((u64)a * (u64)b);
#ifdef __CUDA_ARCH__
    i64 hi = __mul64hi(a, b);
#else
    i64 hi = (i64)(((__int128)a * b) >> 64);
#endif
    if (hi != (lo >> 63)) lo = ((a < 0) != (b < 0)) ? I64_MIN : I64_MAX;
    return lo;
}
__host__ __device__ __forceinline__ i64 wrap_add(i64 a, i64 b) { return (i64)((u64)a + (u64)b); }

// bijective mixer (splitmix64 finaliser): caller hashes may be poorly mixed
__host__ __device__ __forceinline__ u64 mix64(u64 x) {
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
    x ^= x >> 27; x *= 0x94d049bb133111ebULL;
    x ^= x >> 31;
    return x;
}
// inverse of mix64: the key hash a table's key word was made from (each xor-shift undone by repeating it until the
// shift passes 64 bits, each multiplier replaced by its inverse mod 2^64)
__host__ __device__ __forceinline__ u64 unmix64(u64 x) {
    x ^= (x >> 31) ^ (x >> 62);
    x *= 0x319642b2d24d8ec3ULL;
    x ^= (x >> 27) ^ (x >> 54);
    x *= 0x96de1b173f119089ULL;
    x ^= (x >> 30) ^ (x >> 60);
    return x;
}
__host__ __device__ __forceinline__ u64 stored_key(u64 key_hash) {
    u64 k = mix64(key_hash);
    return k < 2 ? k + 2 : k;   // 0 / 1 are the empty / tombstone marks
}

// ------------------------------------------------------------------ key bytes -> key hash
// The two key hashes of the string-keyed entry points, ONE definition for the host (gcra_hash_key,
// gcra_hash_key_seeded) and the hash pass (hash_keys_kernel).  Both read a key as little-endian 64-bit words and a
// tail of 0..7 bytes through a byte source: word(i) = the 8 bytes at i, tail(i, r) = the r < 8 bytes at i,
// zero-extended.  A source never reads outside the key.
struct KeyBytes {
    const unsigned char *p;
    __host__ __device__ __forceinline__ u64 word(u64 i) const { u64 w; memcpy(&w, p + i, 8); return w; }
    __host__ __device__ __forceinline__ u64 tail(u64 i, u32 r) const {
        u64 w = 0;
        for (u32 j = 0; j < r; j++) w |= (u64)p[i + j] << (8 * j);
        return w;
    }
};

// unkeyed: for trusted / synthetic key universes (see "KEY IDENTITY" in gcra_b200.h)
template <class Src>
__host__ __device__ __forceinline__ u64 hash_key_unkeyed(const Src &src, u64 len) {
    u64 h = 0x2545F4914F6CDD1DULL ^ (len * 0x9E3779B97F4A7C15ULL);
    u64 i = 0;
    for (; len - i >= 8; i += 8) h = mix64(h ^ src.word(i)) + 0xD1B54A32D192ED03ULL;
    const u32 r = (u32)(len & 7);
    if (r) h = mix64(h ^ src.tail(i, r) ^ ((u64)r << 56));
    return mix64(h);
}

__host__ __device__ __forceinline__ u64 rotl64(u64 x, int b) { return (x << b) | (x >> (64 - b)); }

// SipHash-2-4 (Aumasson & Bernstein), 64-bit output: the keyed hash for keys an adversary may choose
template <class Src>
__host__ __device__ __forceinline__ u64 hash_key_siphash(const Src &src, u64 len, u64 k0, u64 k1) {
    u64 v0 = 0x736f6d6570736575ULL ^ k0, v1 = 0x646f72616e646f6dULL ^ k1;
    u64 v2 = 0x6c7967656e657261ULL ^ k0, v3 = 0x7465646279746573ULL ^ k1;
#define GCRA_SIPROUND                                                                 \
    do {                                                                              \
        v0 += v1; v1 = rotl64(v1, 13); v1 ^= v0; v0 = rotl64(v0, 32);                \
        v2 += v3; v3 = rotl64(v3, 16); v3 ^= v2;                                      \
        v0 += v3; v3 = rotl64(v3, 21); v3 ^= v0;                                      \
        v2 += v1; v1 = rotl64(v1, 17); v1 ^= v2; v2 = rotl64(v2, 32);                \
    } while (0)
    u64 i = 0;
    for (; len - i >= 8; i += 8) {
        const u64 m = src.word(i);
        v3 ^= m; GCRA_SIPROUND; GCRA_SIPROUND; v0 ^= m;
    }
    const u64 b = (len << 56) | src.tail(i, (u32)(len & 7));
    v3 ^= b; GCRA_SIPROUND; GCRA_SIPROUND; v0 ^= b;
    v2 ^= 0xff;
    GCRA_SIPROUND; GCRA_SIPROUND; GCRA_SIPROUND; GCRA_SIPROUND;
#undef GCRA_SIPROUND
    return v0 ^ v1 ^ v2 ^ v3;
}

// The hash pass's copy of the arena bytes [keys + lo, keys + lo + ext) into a warp's staging (hash_keys_kernel):
// 16-byte chunks from the first byte rounded down to 16 up to the last rounded up (the staging holds chunk_end(...) -
// chunk_begin(...) bytes); one lane takes chunks first, first + step, ...  A chunk wholly inside the arena
// [keys, keys + keys_len) is one 16-byte load, wide(address, staging offset); of any other chunk only the bytes inside
// [keys + lo, keys + lo + ext) are copied, one at a time, narrow(address, staging offset) -- so nothing outside the
// arena is read, not even up to a 16-byte boundary.  (A CPU test runs this with recording callbacks.)
__host__ __device__ __forceinline__ uintptr_t chunk_begin(uintptr_t keys, u32 lo) { return (keys + lo) & ~(uintptr_t)15; }
__host__ __device__ __forceinline__ uintptr_t chunk_end(uintptr_t keys, u32 lo, u32 ext) {
    return (keys + lo + ext + 15) & ~(uintptr_t)15;
}
template <class Wide, class Narrow>
__host__ __device__ __forceinline__ void stage_key_span(uintptr_t keys, u64 keys_len, u32 lo, u32 ext, u32 first,
                                                        u32 step, Wide &&wide, Narrow &&narrow) {
    const uintptr_t g0 = chunk_begin(keys, lo), g1 = chunk_end(keys, lo, ext);
    const uintptr_t a_hi = keys + keys_len, k_lo = keys + lo, k_hi = k_lo + ext;
    for (uintptr_t c = g0 + 16 * (uintptr_t)first; c < g1; c += 16 * (uintptr_t)step) {
        if (c >= keys && c + 16 <= a_hi) {
            wide(c, (u32)(c - g0));
        } else {
            const uintptr_t b1 = c + 16 < k_hi ? c + 16 : k_hi;
            for (uintptr_t b = c > k_lo ? c : k_lo; b < b1; b++) narrow(b, (u32)(b - g0));
        }
    }
}

// the identity an engine gives a key: SipHash-2-4 under its seed, the unkeyed hash when the seed is (0,0)
template <class Src>
__host__ __device__ __forceinline__ u64 hash_key_engine(const Src &src, u64 len, u64 k0, u64 k1) {
    return (k0 | k1) ? hash_key_siphash(src, len, k0, k1) : hash_key_unkeyed(src, len);
}

// ------------------------------------------------------------------ parameter derivation
// Rate::from_count_and_period (rate/mod.rs:172) + `emission_interval * (max_burst-1) as u32`
// (rate_limiter.rs:122) + the `as i64` casts (rate_limiter.rs:154-155).  IEEE double multiply
// and divide, round-to-nearest, then Rust's saturating-truncating `as u64`.
__host__ __device__ __forceinline__ int derive_params(i64 max_burst, i64 count, i64 period,
                                                      i64 *ei_ns, i64 *dvt_ns) {
#ifdef __CUDA_ARCH__
    double v = __ddiv_rn(__dmul_rn(__ll2double_rn(period), 1000000000.0), __ll2double_rn(count));
#else
    double v = (double)period * 1000000000.0 / (double)count;
#endif
    u64 ei;
    if (!(v > 0.0)) ei = 0;
    else if (v >= 18446744073709551616.0) ei = ~0ULL;
    else ei = (u64)v;
    u64 factor = (u64)(u32)(u64)(max_burst - 1);
    u64 lo = ei * factor;
#ifdef __CUDA_ARCH__
    u64 hi = __umul64hi(ei, factor);
#else
    u64 hi = (u64)(((unsigned __int128)ei * factor) >> 64);
#endif
    *ei_ns = (i64)ei;
    *dvt_ns = (i64)lo;
    // Duration * u32 panics when whole seconds overflow u64: (hi*2^64+lo)/1e9 > u64::MAX <=> hi >= 1e9
    return hi >= 1000000000ULL ? 3 : 0;
}

// ------------------------------------------------------------------ expiry codes
__host__ __device__ __forceinline__ bool has_state(i64 exp) { return exp >= 0 || exp == EXP_AT_MAX; }
// Store::get shows the entry at `now` (adaptive_cleanup.rs:248: expiry > now); now >= 0
__host__ __device__ __forceinline__ bool live_at(i64 exp, i64 now) {
    return exp > now || exp == I64_MAX || (exp == EXP_AT_MAX && now != I64_MAX);
}
// the expiry code of now + ttl (now >= 0; a negative ttl has wrapped to a huge u64)
__host__ __device__ __forceinline__ i64 expiry_code(i64 now, u64 ttl) {
    const u64 e = (u64)now + ttl;
    return (e < ttl || e > (u64)I64_MAX) ? I64_MAX : e == (u64)I64_MAX ? EXP_AT_MAX : (i64)e;
}
// the expiry an entry reports (gcra_peek), clamped to I64_MAX as the oracle reports it
__host__ __device__ __forceinline__ i64 expiry_value(i64 exp) { return exp == EXP_AT_MAX ? I64_MAX : exp; }

// ------------------------------------------------------------------ the decision
struct Req { i64 now, ei, dvt, q; };   // 32 bytes: the derived request the decide kernel gathers

struct Decision {
    i64 tat;       // TAT the request starts from (rate_limiter.rs:158-166)
    i64 new_tat;   // :171
    i64 allow_at;  // :174
    i64 new_exp;   // expiry code of now + ttl (adaptive_cleanup.rs:237,268,273)
    bool allowed;  // :175
    bool live;     // stored entry visible to Store::get (adaptive_cleanup.rs:248)
};

// No operation of a decision can saturate or wrap when the clock, the parameters and the stored TAT are
// "ordinary": 0 <= now < 2^61, 0 <= ei, dvt < 2^60, 0 <= q, ei * q < 2^60 and |tat| < 2^61 keep every
// intermediate below 2^63 in magnitude, so the saturating forms equal plain two's-complement arithmetic there.
__device__ __forceinline__ bool ordinary_request(const Req &r, i64 *inc) {
    const u64 hi = __umul64hi((u64)r.ei, (u64)r.q);
    const u64 lo = (u64)r.ei * (u64)r.q;
    *inc = (i64)lo;
    return (((u64)r.now >> 61) | ((u64)r.ei >> 60) | ((u64)r.dvt >> 60) | ((u64)r.q >> 60) | hi | (lo >> 60)) == 0;
}

__device__ __forceinline__ Decision decide(i64 s_tat, i64 s_exp, const Req &r) {
    Decision d;
    d.live = live_at(s_exp, r.now);
    i64 inc;
#ifdef GCRA_NO_FASTPATH
    if (false) {
#else
    if (ordinary_request(r, &inc) && (!d.live || (s_tat > -(1LL << 61) && s_tat < (1LL << 61)))) {
#endif
        // fast path: the same sequence (rate_limiter.rs:158-183) in plain 64-bit arithmetic
        d.tat = d.live ? max(s_tat, r.now - r.dvt) : r.now - r.ei;
        d.new_tat = d.tat + inc;
        d.allow_at = d.new_tat - r.dvt;
        d.allowed = r.now >= d.allow_at;
        const u64 ttl = (u64)((d.new_tat - r.now) + r.dvt);          // negative wraps (:179-183)
        d.new_exp = expiry_code(r.now, ttl);
        return d;
    }
    d.tat = d.live ? max(s_tat, sat_sub(r.now, r.dvt)) : sat_sub(r.now, r.ei);
    d.new_tat = sat_add(d.tat, sat_mul(r.ei, r.q));
    d.allow_at = sat_sub(d.new_tat, r.dvt);
    d.allowed = r.now >= d.allow_at;
    u64 ttl = (u64)sat_add(sat_sub(d.new_tat, r.now), r.dvt);   // negative wraps (:179-183)
    d.new_exp = expiry_code(r.now, ttl);
    return d;
}

struct Outputs { i64 remaining, reset_after, retry_after; };

// rate_limiter.rs:208-238: the three outputs of a decision from `cur` (:208: new_tat if allowed, else the tat the
// request started from), the verdict, allow_at (:174, read only when denied) and the request.  The ONE definition:
// the kernels call it through outputs_of, the host through outputs_from_cur (gcra_expand_results16).
__host__ __device__ __forceinline__ Outputs outputs_from(i64 cur, bool allowed, i64 allow_at, const Req &r) {
    Outputs o;
    // ordinary magnitudes (see ordinary_request; cur is then within +-2^62): nothing below saturates
#ifdef GCRA_NO_FASTPATH
    const bool plain = false;
#else
    const bool plain = ((((u64)r.now >> 61) | ((u64)r.dvt >> 60)) == 0) && cur > -(1LL << 62) && cur < (1LL << 62);
#endif
    i64 room = plain ? (r.now + r.dvt) - cur : sat_sub(wrap_add(r.now, r.dvt), cur);
    // remaining = max(room / ei, 0) for ei > 0 (truncating).  room <= 0 gives 0.  Device: both operands below 2^53
    // (always, away from saturation corners): one IEEE double division, exact after a +-1 correction; otherwise the
    // 64-bit integer division.  Host: the integer division (the same exact quotient).
    i64 rem = 0;
    if (r.ei > 0 && room > 0) {
#ifdef __CUDA_ARCH__
        if ((u64)(room | r.ei) < (1ULL << 53)) {
            i64 q = (i64)__ddiv_rn(__ll2double_rn(room), __ll2double_rn(r.ei));
            i64 rr = room - q * r.ei;
            if (rr < 0) q--; else if (rr >= r.ei) q++;
            rem = q;
        } else {
            rem = room / r.ei;
        }
#else
        rem = room / r.ei;
#endif
    }
    o.remaining = rem;
    i64 reset = plain ? (cur - r.now) + r.dvt : sat_add(sat_sub(cur, r.now), r.dvt);
    o.reset_after = reset < 0 ? 0 : reset;
    i64 retry = 0;
    if (!allowed) {
        // allow_at = new_tat - dvt stays within +-2^63 on the plain path (|new_tat| < 2^62 + 2^60)
        retry = (plain && allow_at > -(1LL << 62) && allow_at < (1LL << 62)) ? allow_at - r.now : sat_sub(allow_at, r.now);
        if (retry < 0) retry = 0;
    }
    o.retry_after = retry;
    return o;
}

// The same from `cur` alone.  A denied request left the state alone, so cur is the tat it started from and
// allow_at = (cur + ei * q) - dvt (rate_limiter.rs:170-174), saturating as decide() computes it.
__host__ __device__ __forceinline__ Outputs outputs_from_cur(i64 cur, bool allowed, const Req &r) {
    const i64 allow_at = allowed ? 0 : sat_sub(sat_add(cur, sat_mul(r.ei, r.q)), r.dvt);
    return outputs_from(cur, allowed, allow_at, r);
}

__device__ __forceinline__ Outputs outputs_of(const Decision &d, const Req &r) {
    return outputs_from(d.allowed ? d.new_tat : d.tat, d.allowed, d.allow_at, r);
}

// ------------------------------------------------------------------ key -> slot
__device__ __forceinline__ u32 mulhi32(u32 a, u32 b) { return __umulhi(a, b); }

__device__ __forceinline__ void bucket_choices(const Table &t, u64 k, u32 &b1, u32 &b2) {
    b1 = mulhi32((u32)k, t.nb_main);
    b2 = mulhi32((u32)(k >> 32), t.nb_main);
    if (b2 == b1) { b2 = b1 + 1; if (b2 == t.nb_main) b2 = 0; }
}

__device__ __forceinline__ void load_keys(const u64 *bucket, u64 k[4]) {
    // L2-coherent 128-bit loads: other CTAs claim slots with CAS during the same kernel
    ulonglong2 a = __ldcg(reinterpret_cast<const ulonglong2 *>(bucket));
    ulonglong2 b = __ldcg(reinterpret_cast<const ulonglong2 *>(bucket + 2));
    k[0] = a.x; k[1] = a.y; k[2] = b.x; k[3] = b.y;
}

__device__ __forceinline__ u32 stash_start(const Table &t, u64 k) {
    return mulhi32((u32)(k >> 17) * 0x9E3779B1u, t.stash_slots);
}

// lookup only; returns null_slot when the key has no slot
__device__ __forceinline__ u32 find_slot(const Table &t, u64 k) {
    u32 b1, b2;
    bucket_choices(t, k, b1, b2);
    u64 kk[4];
    load_keys(t.keys + (size_t)b1 * 4, kk);
#pragma unroll
    for (int j = 0; j < 4; j++) if (kk[j] == k) return b1 * 4 + j;
    load_keys(t.keys + (size_t)b2 * 4, kk);
#pragma unroll
    for (int j = 0; j < 4; j++) if (kk[j] == k) return b2 * 4 + j;
    if (__ldcg(&t.counters[C_STASH]) != 0) {
        u32 s = stash_start(t, k);
        for (u32 i = 0; i < t.stash_slots; i++) {
            u32 slot = t.nb_main * 4 + s;
            u64 v = __ldcg(&t.keys[slot]);
            if (v == k) return slot;
            if (v == KEY_EMPTY) break;
            if (++s == t.stash_slots) s = 0;
        }
    }
    return t.null_slot;
}

__device__ __forceinline__ bool claim_in_bucket(const Table &t, u32 b, u64 kk[4], u64 k, u32 &slot,
                                                bool &fresh) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
        if (kk[j] != KEY_EMPTY) continue;
        u64 old = atomicCAS(&t.keys[(size_t)b * 4 + j], KEY_EMPTY, k);
        if (old == KEY_EMPTY) { slot = b * 4 + j; fresh = true; return true; }
        if (old == k) { slot = b * 4 + j; fresh = false; return true; }
    }
    return false;
}

// Both bucket sectors of a key through L1.  Slots only fill while a kernel runs (nothing empties them), so a
// key SEEN in a possibly stale L1 line is really there; a key not seen proves nothing and the caller goes on with
// L2-coherent loads.  This keeps the hottest keys of a batch (thousands of requests on ONE sector) out of L2:
// an LTS slice serves requests to one sector one after another.
__device__ __forceinline__ u32 find_in_buckets_cached(const Table &t, u64 k, u32 b1, u32 b2) {
    const ulonglong2 *p1 = reinterpret_cast<const ulonglong2 *>(t.keys + (size_t)b1 * 4);
    const ulonglong2 a = p1[0], b = p1[1];
    if (a.x == k) return b1 * 4;
    if (a.y == k) return b1 * 4 + 1;
    if (b.x == k) return b1 * 4 + 2;
    if (b.y == k) return b1 * 4 + 3;
    return t.null_slot;
}

// Lookup, claiming a slot when the key is absent.  Placement rule: first empty slot of bucket 1,
// else of bucket 2, else the stash.  The rule only depends on state that is monotone during a
// kernel (slots fill, never empty), so concurrent claimers of the SAME key always agree on one slot.
__device__ __forceinline__ u32 find_or_claim_coherent(const Table &t, u64 k, u32 b1, u32 b2, bool &fresh);

__device__ __forceinline__ u32 find_or_claim(const Table &t, u64 k, bool &fresh) {
    fresh = false;
    u32 b1, b2;
    bucket_choices(t, k, b1, b2);
    const u32 hit = find_in_buckets_cached(t, k, b1, b2);
    if (hit != t.null_slot) return hit;
    return find_or_claim_coherent(t, k, b1, b2, fresh);
}

// the L2-coherent lookup / claim (everything find_or_claim does after the cached look at bucket 1)
__device__ __forceinline__ u32 find_or_claim_coherent(const Table &t, u64 k, u32 b1, u32 b2, bool &fresh) {
    fresh = false;
    u64 k1[4], k2[4];
    load_keys(t.keys + (size_t)b1 * 4, k1);
#pragma unroll
    for (int j = 0; j < 4; j++) if (k1[j] == k) return b1 * 4 + j;
    load_keys(t.keys + (size_t)b2 * 4, k2);
#pragma unroll
    for (int j = 0; j < 4; j++) if (k2[j] == k) return b2 * 4 + j;
    // stash lookup (remember the first reusable stash slot on the way)
    u32 s0 = stash_start(t, k);
    if (__ldcg(&t.counters[C_STASH]) != 0) {
        u32 s = s0;
        for (u32 i = 0; i < t.stash_slots; i++) {
            u32 slot = t.nb_main * 4 + s;
            u64 v = __ldcg(&t.keys[slot]);
            if (v == k) return slot;
            if (v == KEY_EMPTY) break;
            if (++s == t.stash_slots) s = 0;
        }
    }
    u32 slot;
    if (claim_in_bucket(t, b1, k1, k, slot, fresh)) return slot;
    if (claim_in_bucket(t, b2, k2, k, slot, fresh)) return slot;
    // both buckets full: linear probing in the stash, reusing tombstones
    u32 s = s0;
    for (u32 i = 0; i < t.stash_slots; i++) {
        slot = t.nb_main * 4 + s;
        u64 *p = &t.keys[slot];
        u64 v = __ldcg(p);
        while (v == KEY_EMPTY || v == KEY_TOMB) {
            u64 old = atomicCAS(p, v, k);
            if (old == v) { fresh = true; atomicAdd(&t.counters[C_STASH], 1ULL); return slot; }
            v = old;
        }
        if (v == k) return slot;
        if (++s == t.stash_slots) s = 0;
    }
    return t.null_slot;   // table and stash full
}

}  // namespace gcra
