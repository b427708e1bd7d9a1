// gcra_kernels.cuh -- the sm_90a (H100) kernels of the batched GCRA engine.
//
//   K1a ingest  : bulk-async (TMA, UBLKCP) staging of a request tile into shared memory, per-request
//                 validation + parameter derivation (rate_limiter.rs:111-122), key -> slot probe/claim
//   K1b order   : stable LSD radix sort of (slot, index) so that requests on one key are adjacent and
//                 in index order -- the reference applies requests strictly one at a time
//                 (throttlecrab-server/src/actor.rs:217-236)
//   K1c decide  : warp-cooperative GCRA compare-and-update (rate_limiter.rs:150-248); duplicates of a
//                 key inside a batch are resolved exactly by speculate-and-commit over warp ballots
//   K2  sweep   : HashMap::retain(expiry > now) (adaptive_cleanup.rs:176-182) as a streaming scan
//   K3  route   : stable partition of a batch by owner shard for the multi-GPU all-to-all
#pragma once
#include <cooperative_groups.h>

#include "gcra_device.cuh"
#include "../../include/gcra_b200.h"

namespace gcra {

constexpr int TILE_THREADS = 256;

// ---------------------------------------------------------------------------------------------
// mbarrier + 1-D bulk async copy (TMA) helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ u32 smem_u32(const void *p) {
    return (u32)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(u64 *bar, u32 count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(u64 *bar, u32 bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, u32 bytes, u64 *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void mbar_wait(u64 *bar, u32 parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// ---------------------------------------------------------------------------------------------
// K1a: ingest
// ---------------------------------------------------------------------------------------------
struct PolicyDerived { i64 ei, dvt; int status; int pad; };

__device__ __forceinline__ void write_result(gcra_result *out, i64 remaining, i64 reset, i64 retry,
                                             int status, int allowed) {
    longlong2 a = make_longlong2(remaining, reset);
    longlong2 b;
    b.x = retry;
    b.y = (i64)(u32)status | ((i64)(allowed & 0xff) << 32);
    reinterpret_cast<longlong2 *>(out)[0] = a;
    reinterpret_cast<longlong2 *>(out)[1] = b;
}

// 16-byte result of a compact request: `cur` (rate_limiter.rs:208) instead of the three outputs derived from it;
// the host expands it (gcra_expand_results16 -> outputs_from_cur)
__device__ __forceinline__ void write_result16(gcra_result16 *out, i64 cur, int status, int allowed) {
    *reinterpret_cast<longlong2 *>(out) = make_longlong2(cur, (i64)(u32)status | ((i64)(allowed & 0xff) << 32));
}

// Row format of a batch, request bytes / result bytes.  16-byte results exist for compact requests only (the host
// re-derives the outputs from the policy table), and only for single-segment batches.
enum RowFmt { FMT_48_32 = 0, FMT_16_32 = 1, FMT_16_16 = 2, FMT_COUNT };

// Everything a row format decides, defined once.  COMPACT: a request names a policy of the engine's table
// (gcra_request16) instead of carrying its parameters (gcra_request).  R16: a result is `cur` (gcra_result16)
// instead of the three outputs (gcra_result).
template <int FMT>
struct Rows {
    static constexpr bool COMPACT = FMT != FMT_48_32;
    static constexpr bool R16 = FMT == FMT_16_16;
    static constexpr u32 REQ_BYTES = COMPACT ? 16 : 48;
    static constexpr u32 RES_BYTES = R16 ? 16 : 32;
};
static_assert(Rows<FMT_48_32>::REQ_BYTES == sizeof(gcra_request) && Rows<FMT_16_32>::REQ_BYTES == sizeof(gcra_request16),
              "request rows are the ABI's request structs");
static_assert(Rows<FMT_48_32>::RES_BYTES == sizeof(gcra_result) && Rows<FMT_16_16>::RES_BYTES == sizeof(gcra_result16),
              "result rows are the ABI's result structs");

// the row sizes of a format known at run time only (the host's copies and buffers)
__host__ __device__ constexpr u32 req_bytes(int fmt) {
    return fmt == FMT_16_16 ? Rows<FMT_16_16>::REQ_BYTES : fmt == FMT_16_32 ? Rows<FMT_16_32>::REQ_BYTES : Rows<FMT_48_32>::REQ_BYTES;
}
__host__ __device__ constexpr u32 res_bytes(int fmt) {
    return fmt == FMT_16_16 ? Rows<FMT_16_16>::RES_BYTES : fmt == FMT_16_32 ? Rows<FMT_16_32>::RES_BYTES : Rows<FMT_48_32>::RES_BYTES;
}

// an error row (validation failed, table full, refused residue) in the batch's result format
template <int FMT>
__device__ __forceinline__ void write_error(gcra_result *out, u32 i, int status) {
    if (Rows<FMT>::R16) write_result16(reinterpret_cast<gcra_result16 *>(out) + i, 0, status, 0);
    else write_result(out + i, 0, 0, 0, status, 0);
}

// validation (rate_limiter.rs:111-117) + parameter derivation of ONE request record (shared or global memory):
// returns the status the reference would return before touching the store, fills the key hash and the
// derived request.
template <bool COMPACT>
__device__ __forceinline__ int parse_request(const unsigned char *rec, const PolicyDerived *__restrict__ pol, u32 npol,
                                             i64 now_batch, u64 &key_hash, Req &r) {
    int status = 0;
    if (COMPACT) {
        ulonglong2 w = *reinterpret_cast<const ulonglong2 *>(rec);
        key_hash = w.x;
        int qty = (int)(u32)(w.y & 0xffffffffULL);
        u32 p = (u32)(w.y >> 32);
        r.q = qty;
        r.now = now_batch;
        r.ei = 0;
        r.dvt = 0;
        if (qty < 0) status = GCRA_NEGATIVE_QUANTITY;          // rate_limiter.rs:111-113
        else if (p >= npol) status = GCRA_INTERNAL;
        else {
            PolicyDerived pd = pol[p];
            status = pd.status;
            r.ei = pd.ei;
            r.dvt = pd.dvt;
        }
    } else {
        const ulonglong2 *q = reinterpret_cast<const ulonglong2 *>(rec);
        ulonglong2 w0 = q[0], w1 = q[1], w2 = q[2];
        key_hash = w0.x;
        i64 max_burst = (i64)w0.y, count = (i64)w1.x, period = (i64)w1.y;
        r.q = (i64)w2.x;
        r.now = (i64)w2.y;
        r.ei = 0;
        r.dvt = 0;
        if (r.q < 0) status = GCRA_NEGATIVE_QUANTITY;          // :111-113
        else if (max_burst <= 0 || count <= 0 || period <= 0) status = GCRA_INVALID_RATE_LIMIT;  // :115-117
        else status = derive_params(max_burst, count, period, &r.ei, &r.dvt);
    }
    // a pre-epoch `now` makes the reference read the wall clock (:128-143): not reproducible
    if (status == 0 && r.now < 0) status = GCRA_INTERNAL;
    return status;
}

// validation, parameter derivation, key probe/claim for ONE request whose record sits at `rec` (shared or
// global memory).  Writes the derived request, the error result if any, and returns the sort key
// (slot << 32 | i).  Must be called by all 32 lanes of a warp (warp-aggregated counters).
template <int FMT>
__device__ __forceinline__ u64 ingest_one(const Table &t, const unsigned char *rec, bool in_range,
                                          const PolicyDerived *__restrict__ pol, u32 npol, i64 now_batch, u32 i,
                                          Req *__restrict__ drec, gcra_result *__restrict__ out) {
    int status = 0;
    u64 key_hash = 0;
    Req r = {0, 0, 0, 0};
    if (in_range) status = parse_request<Rows<FMT>::COMPACT>(rec, pol, npol, now_batch, key_hash, r);
    u32 slot = t.null_slot;
    bool fresh = false;
    if (in_range && status == 0) {
        slot = find_or_claim(t, stored_key(key_hash), fresh);
        if (slot == t.null_slot) status = GCRA_INTERNAL;   // table full
    }
    if (in_range) {
        reinterpret_cast<longlong2 *>(drec + i)[0] = make_longlong2(r.now, r.ei);
        reinterpret_cast<longlong2 *>(drec + i)[1] = make_longlong2(r.dvt, r.q);
        if (status != 0) write_error<FMT>(out, i, status);
    }
    // warp-aggregated counters
    u32 mf = __ballot_sync(0xffffffffu, fresh);
    u32 me = __ballot_sync(0xffffffffu, in_range && status != 0);
    if ((threadIdx.x & 31) == 0) {
        if (mf) atomicAdd(&t.counters[C_OCCUPIED], (u64)__popc(mf));
        if (me) atomicAdd(&t.counters[C_ERRORS], (u64)__popc(me));
    }
    return ((u64)slot << 32) | i;
}

template <int FMT>
__global__ void __launch_bounds__(TILE_THREADS)
ingest_kernel(Table t, const void *__restrict__ req_base, const PolicyDerived *__restrict__ pol,
              u32 npol, i64 now_batch, u32 n, Req *__restrict__ drec, u64 *__restrict__ sortkeys,
              gcra_result *__restrict__ out) {
    using Row = Rows<FMT>;
    __shared__ __align__(128) unsigned char stage[TILE_THREADS * Row::REQ_BYTES];
    __shared__ __align__(8) u64 bar;

    const u32 base = blockIdx.x * TILE_THREADS;
    const u32 cnt = min((u32)TILE_THREADS, n - base);
    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar, cnt * Row::REQ_BYTES);
        bulk_g2s(stage, (const unsigned char *)req_base + (size_t)base * Row::REQ_BYTES, cnt * Row::REQ_BYTES, &bar);
    }
    mbar_wait(&bar, 0);

    const u32 i = base + threadIdx.x;
    const bool in_range = threadIdx.x < cnt;
    const u64 key = ingest_one<FMT>(t, stage + (size_t)threadIdx.x * Row::REQ_BYTES, in_range, pol, npol, now_batch, i, drec, out);
    if (in_range) sortkeys[i] = key;
}

// ---------------------------------------------------------------------------------------------
// K1b: stable LSD radix sort on the slot bits of (slot << 32 | index), one sweep per pass
// ---------------------------------------------------------------------------------------------
// One launch counts the digits of every pass (the multiset of digits of a pass does not depend on the order the
// earlier passes leave), then one launch per pass ranks a tile of keys, takes the tile's global offset of each
// digit from the tiles before it (decoupled look-back on per-(tile, digit) status words) and writes the tile back
// in digit order: 1 + passes launches, one read of the keys for the counts and one read + one write per pass.
#ifndef GCRA_SORT_ITEMS
#define GCRA_SORT_ITEMS 16
#endif
constexpr int SORT_ITEMS = GCRA_SORT_ITEMS;                // items per thread
constexpr int SORT_TILE = TILE_THREADS * SORT_ITEMS;       // 4096 keys per tile
constexpr int SORT_MAX_BITS = 9;
constexpr int SORT_MAX_DIGITS = 1 << SORT_MAX_BITS;
constexpr int SORT_MAX_PASSES = (32 + SORT_MAX_BITS - 1) / SORT_MAX_BITS;   // slot ids are 32 bits
static_assert(SORT_MAX_DIGITS == 2 * TILE_THREADS, "the sweep handles two digits per thread");

// Work space of one sort, zeroed once per batch: the tile tickets of the passes, the digit counts of every pass,
// then one status word per (pass, tile, digit); a pass's tiles are `status_tiles` apart (the tiles of the largest
// count the batch can sort).
constexpr u32 SW_TICKETS = 0, SW_HIST = 32, SW_STATUS = SW_HIST + SORT_MAX_PASSES * SORT_MAX_DIGITS;
__host__ __device__ constexpr size_t sort_ws_words(u32 passes, u32 status_tiles) {
    return SW_STATUS + (size_t)passes * status_tiles * SORT_MAX_DIGITS;
}

// digit bits of pass p when `bits` slot bits are sorted in `passes` passes (the low passes take the odd bits)
__host__ __device__ constexpr u32 sort_pass_bits(u32 bits, u32 passes, u32 p) { return bits / passes + (p < bits % passes ? 1 : 0); }

// status word of one (tile, digit): 0 = not yet published, else a flag and a count of keys (< 2^30, max_batch is
// at most that): AGG = this tile's keys of the digit, INC = those of this tile and of every tile before it, plus
// the keys of all smaller digits (the digit's base in the output)
constexpr u32 SS_AGG = 1u << 30, SS_INC = 2u << 30, SS_COUNT = SS_AGG - 1;
constexpr u32 SORT_MAX_COUNT = SS_COUNT;

// block-wide exclusive scan of one value per thread (warp shuffles + one shared-memory hop);
// returns the exclusive prefix, the block total in *total
__device__ __forceinline__ u32 block_exclusive_scan(u32 v, u32 *part, u32 *total) {
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        u32 t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (u32)o) inc += t;
    }
    if (lane == 31) part[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        u32 w = lane < TILE_THREADS / 32 ? part[lane] : 0;
#pragma unroll
        for (int o = 1; o < TILE_THREADS / 32; o <<= 1) {
            u32 t = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= (u32)o) w += t;
        }
        if (lane < TILE_THREADS / 32) part[lane] = w;          // inclusive over warps
    }
    __syncthreads();
    const u32 before = warp > 0 ? part[warp - 1] : 0;
    *total = part[TILE_THREADS / 32 - 1];
    return before + inc - v;
}

// Both kernels take the element count either from the host (`n`) or -- when `n_dev` is given -- from device
// memory: the residue of the index-order pipeline is only known on the device, its sort has a fixed grid.
__device__ __forceinline__ u32 sort_count(u32 n, const u32 *__restrict__ n_dev) { return n_dev ? *n_dev : n; }

// digit counts of all passes: shared-memory bins, then one posted add per nonzero bin per CTA (persistent grid)
__global__ void __launch_bounds__(TILE_THREADS)
sort_digits_kernel(const u64 *__restrict__ in, u32 n_host, const u32 *__restrict__ n_dev, u32 bits, u32 passes,
                   u32 *__restrict__ ws) {
    __shared__ u32 h[SORT_MAX_PASSES * SORT_MAX_DIGITS];
    for (u32 d = threadIdx.x; d < passes * SORT_MAX_DIGITS; d += TILE_THREADS) h[d] = 0;
    __syncthreads();
    const u32 n = sort_count(n_host, n_dev);
    u32 shift[SORT_MAX_PASSES], mask[SORT_MAX_PASSES];
    u32 s = 0;
#pragma unroll
    for (int p = 0; p < SORT_MAX_PASSES; p++) {
        const u32 pb = (u32)p < passes ? sort_pass_bits(bits, passes, p) : 0;
        shift[p] = s;
        mask[p] = (1u << pb) - 1;
        s += pb;
    }
    const u32 stride = gridDim.x * TILE_THREADS;
#pragma unroll 4
    for (u32 i = blockIdx.x * TILE_THREADS + threadIdx.x; i < n; i += stride) {
        const u32 slot = (u32)(in[i] >> 32);
#pragma unroll
        for (int p = 0; p < SORT_MAX_PASSES; p++)
            if ((u32)p < passes) atomicAdd(&h[p * SORT_MAX_DIGITS + ((slot >> shift[p]) & mask[p])], 1u);
    }
    __syncthreads();
    for (u32 d = threadIdx.x; d < passes * SORT_MAX_DIGITS; d += TILE_THREADS)
        if (h[d]) atomicAdd(&ws[SW_HIST + d], h[d]);
}

// the status words of digits d and d + 1 (d even) of one tile, in one 8-byte access
__device__ __forceinline__ uint2 ld_status2(const u32 *p) {
    uint2 v;
    asm volatile("ld.volatile.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_status2(u32 *p, u32 a, u32 b) {
    asm volatile("st.volatile.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}

// Exclusive prefixes of digits d and d + 1 (d even) over the tiles before `tile`, digit bases included: walks back
// from tile - 1, LB tiles per round trip, until each digit meets an inclusive prefix (tile 0 publishes them at once).
// Every earlier tile was handed to a CTA that runs already (ticket), so each wait ends.
__device__ __forceinline__ uint2 sort_lookback2(const u32 *status, u32 tile, u32 d) {
    constexpr int LB = 8;
    u32 sum0 = 0, sum1 = 0;
    bool open0 = true, open1 = true;
    for (int j = (int)tile - 1; open0 || open1; j -= LB) {
        uint2 v[LB];
#pragma unroll
        for (int i = 0; i < LB; i++)
            v[i] = j - i >= 0 ? ld_status2(status + (size_t)(j - i) * SORT_MAX_DIGITS + d) : make_uint2(SS_INC, SS_INC);
#pragma unroll
        for (int i = 0; i < LB; i++) {
            while ((open0 && v[i].x == 0) || (open1 && v[i].y == 0)) v[i] = ld_status2(status + (size_t)(j - i) * SORT_MAX_DIGITS + d);
            if (open0) { sum0 += v[i].x & SS_COUNT; open0 = !(v[i].x & SS_INC); }
            if (open1) { sum1 += v[i].y & SS_COUNT; open1 = !(v[i].y & SS_INC); }
        }
    }
    return make_uint2(sum0, sum1);
}

struct SortSweepSmem {
    union {
        u32 cnt[TILE_THREADS / 32][SORT_MAX_DIGITS];   // per-warp digit counters -> per-warp offsets
        u64 keys[SORT_TILE];                           // the tile in digit order
    } x;
    u32 tile_ex[SORT_MAX_DIGITS];                      // first position of each digit in the tile
    u32 gofs[SORT_MAX_DIGITS];                         // output position - tile position, per digit
    u32 part[TILE_THREADS / 32];
    u32 tile;
};

// One pass.  CTAs take tiles by ticket until the tiles of the count run out.  Warp w ranks tile elements
// [w * 32 ITEMS, (w + 1) * 32 ITEMS) in index order (item k, lane l -> w * 32 ITEMS + 32 k + l), so equal digits
// keep their order: within a warp by MATCH.ANY, across warps and tiles by the prefix sums.
__global__ void __launch_bounds__(TILE_THREADS)
sort_sweep_kernel(const u64 *__restrict__ in, u64 *__restrict__ outk, u32 n_host, const u32 *__restrict__ n_dev,
                  u32 shift, u32 bits, const u32 *__restrict__ hist, u32 *__restrict__ ticket,
                  u32 *__restrict__ status) {
    constexpr int NW = TILE_THREADS / 32;
    __shared__ SortSweepSmem sm;
    const u32 n = sort_count(n_host, n_dev);
    const u32 num_tiles = (n + SORT_TILE - 1) / SORT_TILE;
    const u32 nd = 1u << bits, mask = nd - 1;
    const u32 w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 lt = (1u << lane) - 1;
    const u32 d0 = 2 * threadIdx.x, d1 = d0 + 1;       // this thread's digits in the per-digit steps
    if (blockIdx.x >= num_tiles) return;               // (the CTAs below take every tile)
    for (;;) {
        if (threadIdx.x == 0) sm.tile = atomicAdd(ticket, 1u);
        for (u32 d = threadIdx.x; d < nd; d += TILE_THREADS) {
#pragma unroll
            for (int x = 0; x < NW; x++) sm.x.cnt[x][d] = 0;
        }
        __syncthreads();
        const u32 tile = sm.tile;
        if (tile >= num_tiles) break;                  // uniform over the CTA
        const u32 tile0 = tile * SORT_TILE;
        const u32 tcount = min((u32)SORT_TILE, n - tile0);
        const u32 base = tile0 + w * (32 * SORT_ITEMS);
        u64 key[SORT_ITEMS];
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; k++) {
            const u32 i = base + k * 32 + lane;
            key[k] = i < n ? in[i] : 0;
        }
        u32 rank[SORT_ITEMS];
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; k++) {
            const bool valid = base + k * 32 + lane < n;
            const u32 dig = (u32)(key[k] >> shift) & mask;
            const u32 peers = __match_any_sync(0xffffffffu, valid ? dig : (0x80000000u | lane));
            const u32 before = valid ? sm.x.cnt[w][dig] : 0;
            rank[k] = before + __popc(peers & lt);
            __syncwarp();
            if (valid && (peers & lt) == 0) sm.x.cnt[w][dig] = before + __popc(peers);
            __syncwarp();
        }
        __syncthreads();
        // per digit: exclusive scan over the warps -> the tile's count of the digit
        u32 t0 = 0, t1 = 0;
        if (d1 < nd) {                                 // (nd is even: a thread has both digits or none)
#pragma unroll
            for (int x = 0; x < NW; x++) {
                const u32 a = sm.x.cnt[x][d0], b = sm.x.cnt[x][d1];
                sm.x.cnt[x][d0] = t0;
                sm.x.cnt[x][d1] = t1;
                t0 += a;
                t1 += b;
            }
            if (tile > 0) st_status2(status + (size_t)tile * SORT_MAX_DIGITS + d0, SS_AGG | t0, SS_AGG | t1);
        }
        u32 total;
        const u32 ex = block_exclusive_scan(t0 + t1, sm.part, &total);
        u32 g0, g1;                                    // output position of the tile's first key of d0 / d1
        if (tile == 0) {
            // the digit bases: exclusive scan of the pass's digit counts, once per pass
            const u32 h0 = d1 < nd ? hist[d0] : 0, h1 = d1 < nd ? hist[d1] : 0;
            __syncthreads();                           // (part is reused)
            g0 = block_exclusive_scan(h0 + h1, sm.part, &total);
            g1 = g0 + h0;
        } else {
            const uint2 g = d1 < nd ? sort_lookback2(status, tile, d0) : make_uint2(0, 0);
            g0 = g.x;
            g1 = g.y;
        }
        if (d1 < nd) {
            st_status2(status + (size_t)tile * SORT_MAX_DIGITS + d0, SS_INC | (g0 + t0), SS_INC | (g1 + t1));
            sm.tile_ex[d0] = ex;
            sm.tile_ex[d1] = ex + t0;
            sm.gofs[d0] = g0 - ex;
            sm.gofs[d1] = g1 - ex - t0;
        }
        __syncthreads();
        u32 pos[SORT_ITEMS];
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; k++) {
            const u32 dig = (u32)(key[k] >> shift) & mask;
            pos[k] = sm.tile_ex[dig] + sm.x.cnt[w][dig] + rank[k];
        }
        __syncthreads();                               // (the counters and the keys share memory)
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; k++)
            if (base + k * 32 + lane < n) sm.x.keys[pos[k]] = key[k];
        __syncthreads();
        // consecutive threads write consecutive positions of one digit's range
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; k++) {
            const u32 j = k * TILE_THREADS + threadIdx.x;
            if (j < tcount) {
                const u64 v = sm.x.keys[j];
                outk[sm.gofs[(u32)(v >> shift) & mask] + j] = v;
            }
        }
        __syncthreads();                               // the shared memory is reused by the next tile
    }
}

// ---------------------------------------------------------------------------------------------
// A batch as the kernels see it: one segment of n rows (host-known count), or -- multi-GPU, rows written
// by peer GPUs straight into this GPU's inbox -- up to MAX_SEGS segments whose row counts live in device
// memory.  Row id = (segment << cap_shift) | row-in-segment; results of a row go to its segment's result
// array (for a peer's segment that is a peer-mapped pointer: the result travels back over NVLink as it is
// written).
// ---------------------------------------------------------------------------------------------
constexpr int MAX_SEGS = 16;
struct SegDesc {
    const unsigned char *req;
    gcra_result *res;
};
struct BatchView {
    const unsigned char *req0;   // nseg == 1
    gcra_result *res0;
    const SegDesc *segs;         // device array [nseg], nseg > 1
    const u32 *dev_counts;       // device array [nseg], nseg > 1
    u32 n;                       // nseg == 1: number of rows
    u32 nseg;
    u32 cap_shift;               // nseg > 1: log2 of the per-segment row capacity

    __device__ __forceinline__ gcra_result *res_at(u32 i) const {
        if (nseg == 1) return res0 + i;
        return (gcra_result *)__ldg((const u64 *)&segs[i >> cap_shift].res) + (i & ((1u << cap_shift) - 1));
    }
    // batches with 16-byte results (always one segment): res0 holds gcra_result16 rows
    __device__ __forceinline__ gcra_result16 *res16_at(u32 i) const { return reinterpret_cast<gcra_result16 *>(res0) + i; }
    __device__ __forceinline__ const unsigned char *req_at(u32 i, u32 rsz) const {
        if (nseg == 1) return req0 + (size_t)i * rsz;
        return (const unsigned char *)__ldg((const u64 *)&segs[i >> cap_shift].req) + (size_t)(i & ((1u << cap_shift) - 1)) * rsz;
    }
};

// What the payload `i` of a sorted key stands for.  Sort pipeline: the batch index -- the derived request is
// drec[i], the result goes to out + i.  Residue of the index-order pipeline: the row id -- the request is parsed
// from the batch itself (req_at(i)), the result goes to the row's own place (res_at(i)).
struct OutMap {
    gcra_result *out;
    int by_row;                  // 0: sort pipeline, 1: residue of the index-order pipeline
    int compact;                 // by_row: the batch holds gcra_request16 rows
    BatchView view;
    const PolicyDerived *pol;
    u32 npol;
    i64 now_batch;
    template <bool BY_ROW>
    __device__ __forceinline__ gcra_result *at(u32 i) const { return BY_ROW ? view.res_at(i) : out + i; }
    template <bool BY_ROW>
    __device__ __forceinline__ gcra_result16 *at16(u32 i) const {
        return BY_ROW ? view.res16_at(i) : reinterpret_cast<gcra_result16 *>(out) + i;
    }

    // the result row of a finished decision: R16 (16-byte results) stores `cur` alone, else the 32-byte result
    template <bool BY_ROW, bool R16>
    __device__ __forceinline__ void write(u32 i, const Decision &d, const Req &r) const {
        if (R16) {
            write_result16(at16<BY_ROW>(i), d.allowed ? d.new_tat : d.tat, 0, d.allowed ? 1 : 0);
        } else {
            const Outputs o = outputs_of(d, r);
            write_result(at<BY_ROW>(i), o.remaining, o.reset_after, o.retry_after, 0, d.allowed ? 1 : 0);
        }
    }
};

// ---------------------------------------------------------------------------------------------
// K1c: decide -- the GCRA theoretical-arrival-time compare-and-update
// ---------------------------------------------------------------------------------------------
// Sorted positions are cut into chunks of 32, one warp per chunk.  A run of equal slots (all
// requests of one key, in index order) is owned by the warp whose chunk holds the run's first
// element; when a run crosses the chunk end that warp keeps walking it chunk by chunk, carrying
// the key's state in registers, and the warps of the following chunks skip those lanes.
//
// Inside a chunk every lane evaluates its request against the state its run currently has.
// A request that is denied (or leaves the entry bit-for-bit unchanged) does not alter what later
// requests see, so all lanes up to and including the first state-changing lane of a run are final;
// that lane's new state is shuffled to the lanes behind it and only they re-evaluate.  The loop
// runs (state changes in the busiest run of the chunk + 1) times, and yields exactly the results
// of applying the requests one after another.
struct RunState { i64 tat, exp, ei; };   // ei: informational column only, never part of a decision

__device__ __forceinline__ void run_chunk(u32 lane, bool mine, u32 gmask, const Req &r, RunState &s,
                                          Decision &fin, bool &changed_any, u32 &n_exp_hits) {
    // on return: fin = this lane's decision; s = state after this lane (its run's state)
    const u32 lt = (1u << lane) - 1;
    bool pending = mine;
    bool mflag = false;
    for (;;) {
        Decision d;
        bool mut = false;
        i64 so_tat = s.tat, so_exp = s.exp;
        if (pending) {
            d = decide(s.tat, s.exp, r);
            if (d.allowed) {
                so_tat = d.new_tat; so_exp = d.new_exp;
                mut = (so_tat != s.tat) | (so_exp != s.exp);
            }
        }
        const u32 M = __ballot_sync(0xffffffffu, pending && mut);
        const u32 prior = M & gmask & lt;                  // state-changing lanes of my run before me
        const bool final_now = pending && prior == 0;
        const u32 behind = __ballot_sync(0xffffffffu, pending && prior != 0);
        if (final_now) {
            fin = d;
            // a write over an entry that exists but is expired (adaptive_cleanup.rs:233,267)
            if (d.allowed && !d.live && has_state(s.exp)) n_exp_hits++;
            if (mut) { s.tat = so_tat; s.exp = so_exp; mflag = true; }
            pending = false;
        }
        if (behind == 0) break;                            // common case: one pass, no shuffles
        const int src = prior ? (__ffs(prior) - 1) : (int)lane;
        const i64 sn_tat = __shfl_sync(0xffffffffu, so_tat, src);
        const i64 sn_exp = __shfl_sync(0xffffffffu, so_exp, src);
        if (pending) { s.tat = sn_tat; s.exp = sn_exp; }
    }
    changed_any = mflag;
}

// A run of LONG_RUN_MIN or more requests on one key (a hot key) is not walked by its warp: the warp
// appends (first position, length) to a work list and decide_long_kernel gives it a whole CTA.
#ifndef GCRA_LONG_MIN
#define GCRA_LONG_MIN 256
#endif
#ifndef GCRA_GIANT_MIN
#define GCRA_GIANT_MIN 4096
#endif
#ifndef GCRA_CLUSTER
#define GCRA_CLUSTER 8
#endif
constexpr u32 LONG_RUN_MIN = GCRA_LONG_MIN;     // >= this: one CTA per run (decide_runs_kernel<1>)
constexpr u32 GIANT_RUN_MIN = GCRA_GIANT_MIN;   // >= this: one cluster per run (decide_runs_kernel<CLUSTER_CTAS>)
// 256 threads of ~110 registers: a hot-run CTA leaves room on its SM for a decide_kernel or a sort_sweep_kernel CTA,
// so that the hot runs are decided beside those kernels (DESIGN §4.2)
constexpr int LONG_THREADS = 256;
constexpr int CLUSTER_CTAS = GCRA_CLUSTER;
struct LongRun { u32 start, len; };

template <bool BY_ROW>
__device__ __forceinline__ void load_req(const Req *__restrict__ drec, const OutMap &om, u32 idx, Req &r) {
    if (BY_ROW) {
        // (rows in the residue passed validation in pass A: the status is 0)
        u64 key_hash;
        if (om.compact) parse_request<true>(om.view.req_at(idx, sizeof(gcra_request16)), om.pol, om.npol, om.now_batch, key_hash, r);
        else parse_request<false>(om.view.req_at(idx, sizeof(gcra_request)), nullptr, 0, 0, key_hash, r);
        return;
    }
    longlong2 a = reinterpret_cast<const longlong2 *>(drec + idx)[0];
    longlong2 b = reinterpret_cast<const longlong2 *>(drec + idx)[1];
    r.now = a.x; r.ei = a.y; r.dvt = b.x; r.q = b.y;
}

// first position >= lo whose slot differs from run_slot; sorted[lo] is known to be in the run.
// Warp-cooperative 32-ary search (all lanes call it; result uniform).
__device__ __forceinline__ u32 run_end(const u64 *__restrict__ sorted, u32 n, u32 lo, u32 run_slot, u32 lane) {
    u32 hi = n;   // sorted[hi] (if any) is outside the run
    while (hi - lo > 1) {
        u32 p = lo + (u32)(((u64)(hi - lo) * (lane + 1)) / 33);
        bool in = (u32)(sorted[p] >> 32) == run_slot;    // lo <= p < hi <= n
        u32 m = __ballot_sync(0xffffffffu, in);          // monotone: a prefix of lanes
        int k = __popc(m);
        u32 plo = __shfl_sync(0xffffffffu, p, k > 0 ? k - 1 : 0);
        u32 phi = __shfl_sync(0xffffffffu, p, k < 32 ? k : 31);
        if (k > 0) lo = plo;
        if (k < 32) hi = phi;
    }
    return hi;
}

__device__ __forceinline__ void load_state(const Table &t, u32 slot, RunState &s) {
    const longlong2 v = *reinterpret_cast<const longlong2 *>(&t.state[slot]);   // LDG.128
    s.tat = v.x;
    s.exp = (i64)((u64)v.x + (u64)v.y);
    s.ei = 0;
}

__device__ __forceinline__ void store_state(const Table &t, u32 slot, const RunState &s, bool created) {
    *reinterpret_cast<longlong2 *>(&t.state[slot]) =
        make_longlong2(s.tat, (i64)((u64)s.exp - (u64)s.tat));                                 // STG.128
    if (created) t.ei[slot] = s.ei;
}

#ifndef GCRA_DECIDE_THREADS
#define GCRA_DECIDE_THREADS 256
#endif
constexpr int DECIDE_THREADS = GCRA_DECIDE_THREADS;   // warps are independent: the CTA size only sets scheduling granularity

// one warp, one chunk of 32 sorted positions (see the comment above run_chunk); BY_ROW: the sorted payload is a row
// id of the batch (residue of the index-order pipeline), else a batch index into drec / out; R16: 16-byte results
template <bool BY_ROW, bool R16>
__device__ __forceinline__ void decide_chunk(const Table &t, const u64 *sorted, const Req *__restrict__ drec, u32 n,
                                             const OutMap &out, LongRun *__restrict__ long_runs,
                                             LongRun *__restrict__ giant_runs, u32 *__restrict__ long_count,
                                             u32 warp_global, u32 lane, bool list_runs = false) {
    // list_runs: only find the hot runs and append them to the work lists; else decide everything but the hot runs
    // (a list_runs launch before wrote the lists, the hot-run kernels work on them).  Both walk the same run
    // boundaries below, so the runs that are listed and the runs that are skipped are the same.
    const u32 base = warp_global * 32;
    if (base >= n) return;   // whole warp

    const u32 pos = base + lane;
    const u64 e = pos < n ? sorted[pos] : ~0ULL;
    const u32 slot = (u32)(e >> 32);
    const bool valid = pos < n && slot != t.null_slot;
    // slot of the element just before this chunk, and just after it
    const u32 prev_last = base > 0 ? (u32)(sorted[base - 1] >> 32) : 0xffffffffu;
    const u32 next_first = base + 32 < n ? (u32)(sorted[base + 32] >> 32) : 0xffffffffu;
    u32 prev = __shfl_up_sync(0xffffffffu, slot, 1);
    if (lane == 0) prev = prev_last;
    // lanes continuing a run that started in an earlier chunk belong to that chunk's warp
    const u32 slot0 = __shfl_sync(0xffffffffu, slot, 0);
    const u32 same0 = __ballot_sync(0xffffffffu, valid && slot == slot0);   // sorted => a prefix
    const u32 foreign = (base > 0 && slot0 == prev_last) ? same0 : 0;
    bool mine = valid && !((foreign >> lane) & 1);
    const bool head = mine && slot != prev;
    const u32 heads = __ballot_sync(0xffffffffu, head);
    const u32 le = (lane == 31) ? 0xffffffffu : ((2u << lane) - 1);
    const int hl = mine ? (31 - __clz(heads & le)) : (int)lane;
    // lanes of my run: from my head lane up to (not including) the next head, among `mine` lanes
    u32 gmask = 1u << lane;
    {
        const u32 mine_m = __ballot_sync(0xffffffffu, mine);
        if (mine) {
            const u32 above = heads & ~((hl == 31) ? 0xffffffffu : ((2u << hl) - 1));   // heads after mine
            const u32 upto = above ? ((1u << (__ffs(above) - 1)) - 1) : 0xffffffffu;     // lanes below the next head
            gmask = mine_m & upto & ~((1u << hl) - 1);
        }
    }

    // does the chunk's last run continue past the chunk?  (uniform)
    const u32 slot31 = __shfl_sync(0xffffffffu, slot, 31);
    const bool mine31 = __shfl_sync(0xffffffffu, mine ? 1 : 0, 31) != 0;
    bool cont = mine31 && next_first == slot31;
    const u32 gmask31 = __shfl_sync(0xffffffffu, gmask, 31);
    if (cont) {
        const u32 run_start = base + (u32)(__ffs(gmask31) - 1);
        // sorted, so a run is contiguous: it is hot iff its LONG_RUN_MIN-th request is on the same key.  Only the
        // listing searches a hot run's end (from there).
        const u32 hot_at = run_start + LONG_RUN_MIN - 1;   // > base + 32
        if (hot_at < n && (u32)(sorted[hot_at] >> 32) == slot31) {
            // hot key: hand the whole run (including its lanes here) to the hot-run kernels
            if (list_runs) {
                const u32 end = run_end(sorted, n, hot_at, slot31, lane);
                if (lane == 0) {
                    const bool giant = end - run_start >= GIANT_RUN_MIN;
                    u32 w = atomicAdd(long_count + (giant ? 1 : 0), 1u);
                    LongRun *dst = giant ? giant_runs : long_runs;
                    dst[w].start = run_start;
                    dst[w].len = end - run_start;
                }
            }
            if ((gmask31 >> lane) & 1) mine = false;
            cont = false;
        }
    }
    if (list_runs) return;

    Req r = {0, 0, 0, 0};
    const u32 idx = (u32)e;
    if (mine) load_req<BY_ROW>(drec, out, idx, r);
    // run heads read the entry; the run's lanes get it by shuffle
    RunState s = {0, EXP_EMPTY, 0};
    if (head && mine) load_state(t, slot, s);
    s.tat = __shfl_sync(0xffffffffu, s.tat, hl);
    s.exp = __shfl_sync(0xffffffffu, s.exp, hl);
    const bool was_phantom = !has_state(s.exp);              // the key has no entry yet (same for every lane of the run)

    Decision fin;
    bool changed = false;
    u32 exp_hits = 0;
    run_chunk(lane, mine, gmask, r, s, fin, changed, exp_hits);

    u32 n_allowed = 0, n_denied = 0;
    if (mine) {
        out.template write<BY_ROW, R16>(idx, fin, r);
        n_allowed += fin.allowed ? 1 : 0;
        n_denied += fin.allowed ? 0 : 1;
    }
    // run tails: last lane of each run inside this chunk writes the run's state back
    const u32 run_changed_mask = __ballot_sync(0xffffffffu, mine && changed);
    const bool run_changed = (run_changed_mask & gmask) != 0;
    const u32 next_slot_in = __shfl_down_sync(0xffffffffu, slot, 1);
    const u32 mine_mask = __ballot_sync(0xffffffffu, mine);
    const bool next_mine = lane < 31 && ((mine_mask >> (lane + 1)) & 1);
    const bool tail = mine && (!next_mine || next_slot_in != slot);

    u32 real_inc = 0;
    // informational ei column: emission interval of the run's first request in the creating batch
    s.ei = __shfl_sync(0xffffffffu, r.ei, hl);
    if (tail && !(cont && lane == 31) && run_changed) {
        store_state(t, slot, s, was_phantom);
        if (was_phantom) real_inc++;
    }

    if (cont) {
        // walk the rest of lane 31's run (< LONG_RUN_MIN requests), next chunk prefetched
        RunState cs;
        cs.tat = __shfl_sync(0xffffffffu, s.tat, 31);
        cs.exp = __shfl_sync(0xffffffffu, s.exp, 31);
        cs.ei = __shfl_sync(0xffffffffu, s.ei, 31);   // (set below: ei of the run's first request)
        bool c_changed = __shfl_sync(0xffffffffu, run_changed ? 1 : 0, 31) != 0;
        const bool c_phantom = __shfl_sync(0xffffffffu, was_phantom ? 1 : 0, 31) != 0;
        u32 b2 = base + 32;
        u64 e2 = b2 + lane < n ? sorted[b2 + lane] : ~0ULL;
        bool in_run = (u32)(e2 >> 32) == slot31 && b2 + lane < n;
        Req r2 = {0, 0, 0, 0};
        if (in_run) load_req<BY_ROW>(drec, out, (u32)e2, r2);
        for (;;) {
            const u32 rm = __ballot_sync(0xffffffffu, in_run);   // a prefix (sorted)
            if (rm == 0) break;
            // prefetch the following chunk while this one is decided
            const u32 b3 = b2 + 32;
            u64 e3 = ~0ULL;
            bool in3 = false;
            Req r3 = {0, 0, 0, 0};
            if (rm == 0xffffffffu) {
                e3 = b3 + lane < n ? sorted[b3 + lane] : ~0ULL;
                in3 = (u32)(e3 >> 32) == slot31 && b3 + lane < n;
                if (in3) load_req<BY_ROW>(drec, out, (u32)e3, r3);
            }
            RunState s2 = cs;
            Decision f2;
            bool ch2 = false;
            run_chunk(lane, in_run, rm, r2, s2, f2, ch2, exp_hits);
            if (in_run) {
                out.template write<BY_ROW, R16>((u32)e2, f2, r2);
                n_allowed += f2.allowed ? 1 : 0;
                n_denied += f2.allowed ? 0 : 1;
            }
            c_changed |= __ballot_sync(0xffffffffu, in_run && ch2) != 0;
            const int last = 31 - __clz(rm);
            cs.tat = __shfl_sync(0xffffffffu, s2.tat, last);
            cs.exp = __shfl_sync(0xffffffffu, s2.exp, last);
            if (rm != 0xffffffffu) break;
            b2 = b3; e2 = e3; in_run = in3; r2 = r3;
        }
        cs.ei = __shfl_sync(0xffffffffu, s.ei, 31);
        if (lane == 31 && c_changed) {
            store_state(t, slot31, cs, c_phantom);
            if (c_phantom) real_inc++;
        }
    }

    // warp-aggregated counters
    n_allowed = __reduce_add_sync(0xffffffffu, n_allowed);
    n_denied = __reduce_add_sync(0xffffffffu, n_denied);
    real_inc = __reduce_add_sync(0xffffffffu, real_inc);
    exp_hits = __reduce_add_sync(0xffffffffu, exp_hits);
    if (lane == 0) {
        if (n_allowed) atomicAdd(&t.counters[C_ALLOWED], (u64)n_allowed);
        if (n_denied) atomicAdd(&t.counters[C_DENIED], (u64)n_denied);
        if (real_inc) atomicAdd(&t.counters[C_REAL], (u64)real_inc);
        if (exp_hits) atomicAdd(&t.counters[C_EXPIRED_HITS], (u64)exp_hits);
    }
}

// Resident threads per SM the register budget is sized for: 512 (97 registers, no spills; 2 CTAs of 256 per SM).
// At 1024 the cap of 64 registers spilled ~200 B per thread to local memory, and on H100 the Zipf ticks ran ~5 %
// slower (bench.py, 400 W): the run walk is latency-bound on its state loads, and spill traffic competes with them.
#ifndef GCRA_DECIDE_MINBLOCKS
#define GCRA_DECIDE_MINBLOCKS (512 / GCRA_DECIDE_THREADS)
#endif
template <bool BY_ROW, bool R16>
__global__ void __launch_bounds__(DECIDE_THREADS, GCRA_DECIDE_MINBLOCKS)
decide_kernel(Table t, const u64 *__restrict__ sorted, const Req *__restrict__ drec, u32 n_host,
              const u32 *__restrict__ n_dev, OutMap out) {
    const u32 n = sort_count(n_host, n_dev);
    const u32 warps_total = gridDim.x * (DECIDE_THREADS / 32);
    for (u32 wg = (blockIdx.x * DECIDE_THREADS + threadIdx.x) >> 5; wg * 32 < n; wg += warps_total)
        decide_chunk<BY_ROW, R16>(t, sorted, drec, n, out, nullptr, nullptr, nullptr, wg, threadIdx.x & 31);
}

// The hot runs of a sorted batch, into the work lists of the hot-run kernels: decide_chunk's run boundaries without
// its decisions (which it leaves to decide_kernel), in a kernel of few registers that fills the SMs.
__global__ void __launch_bounds__(DECIDE_THREADS)
list_runs_kernel(Table t, const u64 *__restrict__ sorted, u32 n_host, const u32 *__restrict__ n_dev,
                 LongRun *__restrict__ long_runs, LongRun *__restrict__ giant_runs, u32 *__restrict__ long_count) {
    const u32 n = sort_count(n_host, n_dev);
    const u32 warps_total = gridDim.x * (DECIDE_THREADS / 32);
    for (u32 wg = (blockIdx.x * DECIDE_THREADS + threadIdx.x) >> 5; wg * 32 < n; wg += warps_total)
        decide_chunk<false, false>(t, sorted, nullptr, n, OutMap{}, long_runs, giant_runs, long_count, wg, threadIdx.x & 31, true);
}

// Small batches (n < LONG_RUN_MIN, e.g. one RateLimiter::rate_limit call or a lightly loaded actor): ONE CTA
// does everything -- ingest, a bitonic sort of the (slot, index) keys in shared memory, and the warp-chunk
// compare-and-update -- instead of the sort pipeline's 4-7 launches and 2 memsets.  No run can reach LONG_RUN_MIN, so no work list is produced.
constexpr u32 SMALL_MAX = 255;
static_assert(SMALL_MAX < GCRA_LONG_MIN && SMALL_MAX < TILE_THREADS, "small path must not create long runs");

template <int FMT>
__global__ void __launch_bounds__(TILE_THREADS)
small_batch_kernel(Table t, const void *__restrict__ req_base, const PolicyDerived *__restrict__ pol, u32 npol,
                   i64 now_batch, u32 n, Req *__restrict__ drec, gcra_result *__restrict__ out) {
    __shared__ u64 keys[TILE_THREADS];
    const u32 tid = threadIdx.x;
    const bool in_range = tid < n;
    const u64 key = ingest_one<FMT>(t, (const unsigned char *)req_base + (size_t)(in_range ? tid : 0) * Rows<FMT>::REQ_BYTES,
                                    in_range, pol, npol, now_batch, tid, drec, out);
    keys[tid] = in_range ? key : ~0ULL;
    __syncthreads();
    // bitonic sort of 256 keys; (slot << 32 | index) is a total order, so equal slots stay in index order
    for (u32 k = 2; k <= TILE_THREADS; k <<= 1) {
        for (u32 j = k >> 1; j > 0; j >>= 1) {
            const u32 partner = tid ^ j;
            if (partner > tid) {
                const u64 a = keys[tid], b = keys[partner];
                const bool up = (tid & k) == 0;
                if ((a > b) == up) { keys[tid] = b; keys[partner] = a; }
            }
            __syncthreads();
        }
    }
    __threadfence_block();   // drec / state written above are read below by other warps of this CTA
    OutMap om;
    om.out = out;
    om.by_row = 0;
    decide_chunk<false, Rows<FMT>::R16>(t, keys, drec, n, om, nullptr, nullptr, nullptr, tid >> 5, tid & 31);
}

// ---------------------------------------------------------------------------------------------
// Hot keys: runs of >= LONG_RUN_MIN requests get one CTA, runs of >= GIANT_RUN_MIN one 8-CTA cluster.
// ---------------------------------------------------------------------------------------------
// The run is consumed in strides (one request per thread of the group).  Two kinds of round:
//
//  * plain round: every pending thread evaluates its request against the run's current state; the
//    group finds the first state-changing request (min-reduction); everything up to it is final and
//    its new state becomes current.  One round per state change -- fine while changes are rare.
//
//  * finite-state round (after FSM_AFTER state changes in the run): some keys flip between a few
//    states all the time (max_burst = 1: every zero-quantity request toggles the entry, SURVEY V8), which
//    would cost one round per flip.  The threads keep the last K distinct states of the run as
//    candidates, each request becomes a map "candidate in -> candidate out" (a nibble per candidate,
//    0xF = leaves the candidate set), the maps are composed with an inclusive prefix scan (shuffles,
//    shared memory, distributed shared memory across the cluster), and every request reads its TRUE
//    input state off the scan.  A round is only repeated when a request creates a state that is not a
//    candidate yet.  Still exact: each decision is decide(true input state, request).
constexpr int FSM_K = 4;
constexpr u32 FSM_NEW = 0xF;
constexpr u32 FSM_IDENT = 0x3210;
constexpr u32 FSM_AFTER = 4;

__device__ __forceinline__ u32 fsm_compose(u32 f, u32 g) {   // first f, then g
    const u64 gg = (u64)g | (0xFULL << 60);
    u32 r = 0;
#pragma unroll
    for (int c = 0; c < FSM_K; c++) {
        const u32 x = (f >> (4 * c)) & 0xF;
        r |= ((u32)(gg >> (4 * x)) & 0xF) << (4 * c);
    }
    return r;
}

struct Cands {
    i64 tat[FSM_K], exp[FSM_K];
    __device__ __forceinline__ void get(u32 i, i64 &t, i64 &e) const {
        t = tat[0]; e = exp[0];
#pragma unroll
        for (int c = 1; c < FSM_K; c++) if (i == (u32)c) { t = tat[c]; e = exp[c]; }
    }
    __device__ __forceinline__ void set(u32 i, i64 t, i64 e) {
#pragma unroll
        for (int c = 0; c < FSM_K; c++) if (i == (u32)c) { tat[c] = t; exp[c] = e; }
    }
    __device__ __forceinline__ u32 find(u32 nc, i64 t, i64 e) const {
        u32 j = FSM_NEW;
#pragma unroll
        for (int c = 0; c < FSM_K; c++) if ((u32)c < nc && tat[c] == t && exp[c] == e) j = c;
        return j;
    }
};

struct PubState { i64 tat, exp; };

template <int CTAS, bool BY_ROW, bool R16>
__global__ void __launch_bounds__(LONG_THREADS, 2)
decide_runs_kernel(Table t, const u64 *__restrict__ sorted, const Req *__restrict__ drec,
                   OutMap out, const LongRun *__restrict__ runs,
                   const u32 *__restrict__ count_ptr) {
    namespace cg = cooperative_groups;
    constexpr int NW = LONG_THREADS / 32;
    constexpr u32 STRIDE = CTAS * LONG_THREADS;
    __shared__ u32 sm_warp[2][NW];       // per-warp first-change position / composed map
    __shared__ u32 sm_cta[2];            // this CTA's value, read by the other CTAs of the cluster
    __shared__ PubState sm_pub[2];       // state created in this round (written into every CTA)
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    u32 rank = 0, group_id = blockIdx.x, num_groups = gridDim.x;
    if (CTAS > 1) {
        rank = cg::this_cluster().block_rank();
        group_id = blockIdx.x / CTAS;
        num_groups = gridDim.x / CTAS;
    }
    auto group_sync = [&]() {
        if (CTAS > 1) cg::this_cluster().sync(); else __syncthreads();
    };
    const u32 gpos = rank * LONG_THREADS + tid;          // position inside a stride
    const u32 count = *count_ptr;
    u32 n_allowed = 0, n_denied = 0, exp_hits = 0, real_inc = 0;
    u32 par = 0;
    for (u32 item = group_id; item < count; item += num_groups) {
        const u32 start = runs[item].start, len = runs[item].len;
        const u32 slot = (u32)(sorted[start] >> 32);
        RunState s0;
        load_state(t, slot, s0);
        const bool was_phantom = !has_state(s0.exp);           // the key has no entry yet
        Cands cd;
#pragma unroll
        for (int c = 0; c < FSM_K; c++) { cd.tat[c] = s0.tat; cd.exp[c] = s0.exp; }
        u32 nc = 1, cur = 0, victim = 0, n_changes = 0;
        // software pipeline: the next stride's request is loaded while this one is decided
        bool active = gpos < len;
        u32 idx = 0;
        Req r = {0, 0, 0, 0};
        if (active) { idx = (u32)sorted[start + gpos]; load_req<BY_ROW>(drec, out, idx, r); }
        for (u32 off = 0; off < len; off += STRIDE) {
            const u32 noff = off + STRIDE;
            const bool nactive = noff + gpos < len;
            u32 nidx = 0;
            Req nr = {0, 0, 0, 0};
            if (nactive) { nidx = (u32)sorted[start + noff + gpos]; load_req<BY_ROW>(drec, out, nidx, nr); }
            bool pending = active;
            for (;;) {
                const bool fsm = n_changes >= FSM_AFTER;
                u32 in_idx = cur;            // candidate this thread's request really starts from
                bool has_new;                // some request of this round created a new state
                u32 total = FSM_IDENT;       // composed map of the whole round (fsm rounds)
                u32 my_map = FSM_IDENT;
                if (!fsm) {
                    // ---- plain round: first state-changing request by min-reduction
                    i64 ct, ce;
                    cd.get(cur, ct, ce);
                    bool mut = false;
                    if (pending) {
                        const Decision d = decide(ct, ce, r);
                        mut = d.allowed && ((d.new_tat != ct) | (d.new_exp != ce));
                    }
                    const u32 wmin = __reduce_min_sync(0xffffffffu, (pending && mut) ? gpos : 0xffffffffu);
                    if (lane == 0) sm_warp[par][warp] = wmin;
                    __syncthreads();
                    u32 first = __reduce_min_sync(0xffffffffu, lane < NW ? sm_warp[par][lane] : 0xffffffffu);
                    if (CTAS > 1) {
                        if (tid == 0) sm_cta[par] = first;
                        cg::this_cluster().sync();
                        u32 v = 0xffffffffu;
                        if (lane < CTAS) v = *cg::this_cluster().map_shared_rank(&sm_cta[par], lane);
                        first = __reduce_min_sync(0xffffffffu, v);
                    }
                    has_new = first != 0xffffffffu;
                    if (pending && gpos > first) in_idx = FSM_NEW;       // behind the change: retry
                    if (pending && gpos == first) my_map = (FSM_IDENT & ~(0xFu << (4 * cur))) | (FSM_NEW << (4 * cur));
                } else {
                    // ---- finite-state round
                    if (pending) {
                        my_map = 0;
#pragma unroll
                        for (int c = 0; c < FSM_K; c++) {
                            u32 o = FSM_NEW;
                            if ((u32)c < nc) {
                                const Decision d = decide(cd.tat[c], cd.exp[c], r);
                                o = c;
                                if (d.allowed && ((d.new_tat != cd.tat[c]) | (d.new_exp != cd.exp[c])))
                                    o = cd.find(nc, d.new_tat, d.new_exp);
                            }
                            my_map |= o << (4 * c);
                        }
                    }
                    u32 incl = my_map;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        const u32 o = __shfl_up_sync(0xffffffffu, incl, d);
                        if (lane >= (u32)d) incl = fsm_compose(o, incl);
                    }
                    u32 lane_excl = __shfl_up_sync(0xffffffffu, incl, 1);
                    if (lane == 0) lane_excl = FSM_IDENT;
                    if (lane == 31) sm_warp[par][warp] = incl;
                    __syncthreads();
                    u32 wt = lane < NW ? sm_warp[par][lane] : FSM_IDENT;
#pragma unroll
                    for (int d = 1; d < NW; d <<= 1) {
                        const u32 o = __shfl_up_sync(0xffffffffu, wt, d);
                        if (lane >= (u32)d) wt = fsm_compose(o, wt);
                    }
                    u32 cta_total = __shfl_sync(0xffffffffu, wt, NW - 1);
                    u32 excl = __shfl_sync(0xffffffffu, wt, warp > 0 ? warp - 1 : 0);
                    if (warp == 0) excl = FSM_IDENT;
                    total = cta_total;
                    if (CTAS > 1) {
                        if (tid == 0) sm_cta[par] = cta_total;
                        cg::this_cluster().sync();
                        u32 ctv = FSM_IDENT;
                        if (lane < CTAS) ctv = *cg::this_cluster().map_shared_rank(&sm_cta[par], lane);
#pragma unroll
                        for (int d = 1; d < CTAS; d <<= 1) {
                            const u32 o = __shfl_up_sync(0xffffffffu, ctv, d);
                            if (lane >= (u32)d) ctv = fsm_compose(o, ctv);
                        }
                        total = __shfl_sync(0xffffffffu, ctv, CTAS - 1);
                        u32 cexcl = __shfl_sync(0xffffffffu, ctv, rank > 0 ? rank - 1 : 0);
                        if (rank == 0) cexcl = FSM_IDENT;
                        excl = fsm_compose(cexcl, excl);
                    }
                    excl = fsm_compose(excl, lane_excl);
                    in_idx = (excl >> (4 * cur)) & 0xF;
                    has_new = ((total >> (4 * cur)) & 0xF) == FSM_NEW;
                }
                // ---- finalize every pending request whose true input state is known
                if (pending && in_idx != FSM_NEW) {
                    i64 ct, ce;
                    cd.get(in_idx, ct, ce);
                    const Decision d = decide(ct, ce, r);
                    out.template write<BY_ROW, R16>(idx, d, r);
                    n_allowed += d.allowed ? 1 : 0;
                    n_denied += d.allowed ? 0 : 1;
                    if (d.allowed && !d.live && has_state(ce)) exp_hits++;
                    pending = false;
                    if (((my_map >> (4 * in_idx)) & 0xF) == FSM_NEW) {
                        // this request created a state outside the candidate set: publish it
                        PubState ps = {d.new_tat, d.new_exp};
                        if (CTAS > 1) {
                            for (int c = 0; c < CTAS; c++) *cg::this_cluster().map_shared_rank(&sm_pub[par], c) = ps;
                        } else {
                            sm_pub[par] = ps;
                        }
                    }
                }
                if (!has_new) {
                    if (fsm) cur = (total >> (4 * cur)) & 0xF;
                    par ^= 1;
                    break;                                   // uniform over the group: stride done
                }
                group_sync();
                const PubState ps = sm_pub[par];
                par ^= 1;
                u32 v = cd.find(nc, ps.tat, ps.exp);          // plain rounds may return to a known state
                if (v == FSM_NEW) {
                    if (nc < FSM_K) { v = nc; nc++; }
                    else { v = victim; victim = (victim + 1) % FSM_K; }
                    cd.set(v, ps.tat, ps.exp);
                }
                cur = v;
                n_changes++;
            }
            active = nactive; idx = nidx; r = nr;
        }
        if (rank == 0 && tid == 0) {
            RunState fs;
            cd.get(cur, fs.tat, fs.exp);
            if (fs.tat != s0.tat || fs.exp != s0.exp) {
                Req first;
                load_req<BY_ROW>(drec, out, (u32)sorted[start], first);
                fs.ei = first.ei;
                store_state(t, slot, fs, was_phantom);
                if (was_phantom) real_inc++;
            }
        }
        __syncthreads();
    }
    if (CTAS > 1) cg::this_cluster().sync();   // nobody leaves while its shared memory may be accessed remotely
    n_allowed = __reduce_add_sync(0xffffffffu, n_allowed);
    n_denied = __reduce_add_sync(0xffffffffu, n_denied);
    real_inc = __reduce_add_sync(0xffffffffu, real_inc);
    exp_hits = __reduce_add_sync(0xffffffffu, exp_hits);
    if (lane == 0) {
        if (n_allowed) atomicAdd(&t.counters[C_ALLOWED], (u64)n_allowed);
        if (n_denied) atomicAdd(&t.counters[C_DENIED], (u64)n_denied);
        if (real_inc) atomicAdd(&t.counters[C_REAL], (u64)real_inc);
        if (exp_hits) atomicAdd(&t.counters[C_EXPIRED_HITS], (u64)exp_hits);
    }
}

// ---------------------------------------------------------------------------------------------
// K2: sweep -- retain(expiry > now)
// ---------------------------------------------------------------------------------------------
// One thread per slot: a coalesced 128-bit load of the (tat, off) pair (L1 bypass), expiry = tat + off, and
// only the slots whose entry has expired are touched again: the pair is reset to the empty pattern with one
// 128-bit store into the sector that was just read.  The KEY word is left in place (no scattered 8-byte
// writes into sectors the sweep never reads): a key without an entry behaves exactly like an absent key
// (Store::get sees nothing, the next allowed request creates the entry), it just keeps its slot -- which is
// what a key that comes back wants anyway.  purge_kernel reclaims such slots when the table gets crowded.
__device__ __forceinline__ ulonglong2 ld_stream(const void *p) {
    ulonglong2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
    return v;
}

constexpr int SWEEP_UNROLL = 4;

// One thread per 32-byte SECTOR of the state array (two slots): two 128-bit loads, and when either entry has
// expired the whole sector is written back (two 128-bit stores), so DRAM only ever sees full-sector writes.
// `mode` (tuning, GCRA_SWEEP_MODE): 0 plain stores; 1 streaming stores (st.global.cs: the reset pairs are not read
// again soon, they need not displace the scan's lines in L2); 2 only the expired 16-byte pair is written.
__device__ __forceinline__ void st_stream(void *p, longlong2 v) {
    asm volatile("st.global.cs.v2.s64 [%0], {%1, %2};" ::"l"(p), "l"(v.x), "l"(v.y) : "memory");
}

__global__ void __launch_bounds__(TILE_THREADS)
sweep_kernel(Table t, u64 total_slots, i64 now, int mode) {
    u32 removed = 0;
    const u64 total_pairs = total_slots >> 1;            // the slot count is a power of two >= 64
    const u64 stride = (u64)gridDim.x * TILE_THREADS;
    u64 i = (u64)blockIdx.x * TILE_THREADS + threadIdx.x;
    while (i < total_pairs) {
        ulonglong2 a[SWEEP_UNROLL], b[SWEEP_UNROLL];
#pragma unroll
        for (int u = 0; u < SWEEP_UNROLL; u++) {
            const u64 p = i + (u64)u * stride;
            a[u] = make_ulonglong2(0, (u64)EXP_EMPTY);
            b[u] = a[u];
            if (p < total_pairs) { a[u] = ld_stream(&t.state[2 * p]); b[u] = ld_stream(&t.state[2 * p + 1]); }
        }
#pragma unroll
        for (int u = 0; u < SWEEP_UNROLL; u++) {
            const u64 p = i + (u64)u * stride;
            const i64 ea = (i64)(a[u].x + a[u].y), eb = (i64)(b[u].x + b[u].y);
            const bool xa = has_state(ea) && !live_at(ea, now), xb = has_state(eb) && !live_at(eb, now);   // entries Store::get no longer shows
            if (xa | xb) {
                longlong2 *dst = reinterpret_cast<longlong2 *>(&t.state[2 * p]);
                const longlong2 va = xa ? make_longlong2(0, EXP_EMPTY) : make_longlong2((i64)a[u].x, (i64)a[u].y);
                const longlong2 vb = xb ? make_longlong2(0, EXP_EMPTY) : make_longlong2((i64)b[u].x, (i64)b[u].y);
                if (mode == 1) { st_stream(dst, va); st_stream(dst + 1, vb); }
                else if (mode == 2) { if (xa) dst[0] = va; if (xb) dst[1] = vb; }
                else { dst[0] = va; dst[1] = vb; }
                removed += (xa ? 1 : 0) + (xb ? 1 : 0);
            }
        }
        i += (u64)SWEEP_UNROLL * stride;
    }
    removed = __reduce_add_sync(0xffffffffu, removed);
    if ((threadIdx.x & 31) == 0 && removed) {
        atomicAdd(&t.counters[C_REAL], (u64)(0 - (u64)removed));
        atomicAdd(&t.counters[C_SWEPT], (u64)removed);
    }
}

// Reclaim the slots of keys that hold no entry (swept, or only ever denied): exclusive pass run by the host
// before it would otherwise grow the table.  Reads key + state of every slot, clears such keys
// (stash: tombstone, so probing continues past them).
__global__ void __launch_bounds__(TILE_THREADS)
purge_kernel(Table t, u64 total_slots) {
    u32 freed = 0, freed_stash = 0;
    const u64 stride = (u64)gridDim.x * TILE_THREADS;
    for (u64 k = (u64)blockIdx.x * TILE_THREADS + threadIdx.x; k < total_slots; k += stride) {
        const ulonglong2 v = ld_stream(&t.state[k]);
        if (has_state((i64)(v.x + v.y))) continue;
        if (t.keys[k] < 2) continue;
        const bool stash = k >= (u64)t.nb_main * 4;
        t.keys[k] = stash ? KEY_TOMB : KEY_EMPTY;
        freed++;
        if (stash) freed_stash++;
    }
    freed = __reduce_add_sync(0xffffffffu, freed);
    freed_stash = __reduce_add_sync(0xffffffffu, freed_stash);
    if ((threadIdx.x & 31) == 0 && freed) {
        atomicAdd(&t.counters[C_OCCUPIED], (u64)(0 - (u64)freed));
        if (freed_stash) atomicAdd(&t.counters[C_STASH], (u64)(0 - (u64)freed_stash));
    }
}

// fill slots [first, first+count) with the empty pattern (also resets an emptied stash)
__global__ void __launch_bounds__(TILE_THREADS)
clear_slots_kernel(Table t, u64 first, u64 count) {
    const u64 stride = (u64)gridDim.x * TILE_THREADS;
    for (u64 i = (u64)blockIdx.x * TILE_THREADS + threadIdx.x; i < count; i += stride) {
        t.keys[first + i] = KEY_EMPTY;
        *reinterpret_cast<longlong2 *>(&t.state[first + i]) = make_longlong2(0, EXP_EMPTY);
        t.ei[first + i] = 0;
    }
}

// re-insert every entry of `src` into the (empty, larger) table `dst` -- HashMap growth
__global__ void __launch_bounds__(TILE_THREADS)
rehash_kernel(Table src, u64 src_slots, Table dst) {
    const u64 stride = (u64)gridDim.x * TILE_THREADS;
    for (u64 i = (u64)blockIdx.x * TILE_THREADS + threadIdx.x; i < src_slots; i += stride) {
        u64 k = src.keys[i];
        if (k < 2) continue;
        TatOff st = src.state[i];
        if (!has_state((i64)((u64)st.tat + st.off))) continue;   // keys without an entry are not carried over
        bool fresh;
        u32 s = find_or_claim(dst, k, fresh);
        if (s == dst.null_slot) { atomicAdd(&dst.counters[C_INSERT_FAIL], 1ULL); continue; }
        dst.state[s] = st;
        dst.ei[s] = src.ei[i];
        atomicAdd(&dst.counters[C_OCCUPIED], 1ULL);
        atomicAdd(&dst.counters[C_REAL], 1ULL);
    }
}

// ---------------------------------------------------------------------------------------------
// Store-trait single operations (core/store/mod.rs:85-133): one thread, results in `res`
// ---------------------------------------------------------------------------------------------
struct StoreOpResult { i64 value; int flag; int status; };

// op: 0 get (adaptive_cleanup.rs:246-252), 1 cas (:221-244), 2 set_nx (:254-278),
//     3 peek (entry as stored: res[0].value = tat, res[1].value = expiry)

__global__ void store_op_kernel(Table t, int op, u64 key, i64 a, i64 b, u64 ttl, i64 now,
                                StoreOpResult *res) {
    StoreOpResult r = {0, 0, 0};
    if (op == 2) {
        bool fresh;
        u32 s = find_or_claim(t, key, fresh);
        if (s == t.null_slot) {
            r.status = GCRA_INTERNAL;
        } else {
            TatOff *l = t.state + s;
            if (fresh) atomicAdd(&t.counters[C_OCCUPIED], 1ULL);
            i64 ex = (i64)((u64)l->tat + l->off);   // EXP_EMPTY for a fresh or entry-less key
            if (live_at(ex, now)) {
                r.flag = 0;                                  // live entry: :264-265
            } else {
                l->tat = a;
                l->off = (u64)expiry_code(now, ttl) - (u64)a;
                r.flag = 1;
                atomicAdd(&t.counters[C_ALLOWED], 1ULL);     // one mutating op
                if (!has_state(ex)) atomicAdd(&t.counters[C_REAL], 1ULL);
                else atomicAdd(&t.counters[C_EXPIRED_HITS], 1ULL);   // :267
            }
        }
    } else {
        u32 s = find_slot(t, key);
        if (s != t.null_slot) {
            TatOff *l = t.state + s;
            i64 tat = l->tat;
            i64 ex = (i64)((u64)tat + l->off);
            if (op == 3) {
                if (has_state(ex)) { r.flag = 1; r.value = tat; res[1].value = expiry_value(ex); }
            } else if (live_at(ex, now)) {
                if (op == 0) { r.flag = 1; r.value = tat; }
                else if (tat == a) {                         // :236-240
                    l->tat = b;
                    l->off = (u64)expiry_code(now, ttl) - (u64)b;
                    r.flag = 1;
                    atomicAdd(&t.counters[C_ALLOWED], 1ULL);
                }
            } else if (op == 1 && has_state(ex)) {
                atomicAdd(&t.counters[C_EXPIRED_HITS], 1ULL);        // :232-235
            }
        }
    }
    res[0] = r;
}

// ---------------------------------------------------------------------------------------------
// K3: routing for the hash-sharded multi-GPU engine -- stable partition by owner shard
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ u32 owner_of(u64 key_hash, u32 n_shards) {
    // bits independent of the in-table bucket choices (those use mix64's low/high words directly)
    u64 m = mix64(key_hash ^ 0xA24BAED4963EE407ULL);
    return (u32)(((m >> 32) * (u64)n_shards) >> 32);
}

constexpr int ROUTE_MAX_SHARDS = 16;

// (tiles at or past n count zero rows: route_count_dev_kernel sizes its grid from a bound of the device count)
__device__ __forceinline__ void route_count_tile(const gcra_request *__restrict__ req, u32 n, u32 n_shards,
                                                 u32 num_tiles, u32 *__restrict__ tile_counts) {
    __shared__ u32 c[ROUTE_MAX_SHARDS];
    if (threadIdx.x < ROUTE_MAX_SHARDS) c[threadIdx.x] = 0;
    __syncthreads();
    u32 i = blockIdx.x * TILE_THREADS + threadIdx.x;
    if (i < n) atomicAdd(&c[owner_of(req[i].key_hash, n_shards)], 1u);
    __syncthreads();
    if (threadIdx.x < n_shards) tile_counts[threadIdx.x * num_tiles + blockIdx.x] = c[threadIdx.x];
}

__global__ void __launch_bounds__(TILE_THREADS)
route_count_kernel(const gcra_request *__restrict__ req, u32 n, u32 n_shards, u32 num_tiles,
                   u32 *__restrict__ tile_counts) {
    route_count_tile(req, n, n_shards, num_tiles, tile_counts);
}

// the row count on the device (a ring slot's parsed rows): min(*dev_n, n_bound) rows, grid sized from n_bound
__global__ void __launch_bounds__(TILE_THREADS)
route_count_dev_kernel(const gcra_request *__restrict__ req, u32 n_bound, const u32 *__restrict__ dev_n, u32 n_shards,
                       u32 num_tiles, u32 *__restrict__ tile_counts) {
    route_count_tile(req, min(*dev_n, n_bound), n_shards, num_tiles, tile_counts);
}

// single CTA: exclusive scan of tile_counts in (shard, tile) order; per-shard totals to counts
__global__ void __launch_bounds__(TILE_THREADS)
route_scan_kernel(u32 *__restrict__ tile_counts, u32 n_shards, u32 num_tiles, u32 *__restrict__ counts) {
    __shared__ u32 part[TILE_THREADS];
    __shared__ u32 carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (u32 s = 0; s < n_shards; s++) {
        u32 shard_start = carry;
        u32 *row = tile_counts + s * num_tiles;
        for (u32 b = 0; b < num_tiles; b += TILE_THREADS) {
            u32 i = b + threadIdx.x;
            u32 v = i < num_tiles ? row[i] : 0;
            part[threadIdx.x] = v;
            __syncthreads();
            for (u32 off = 1; off < TILE_THREADS; off <<= 1) {
                u32 x = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
                __syncthreads();
                part[threadIdx.x] += x;
                __syncthreads();
            }
            if (i < num_tiles) row[i] = carry + part[threadIdx.x] - v;
            __syncthreads();
            if (threadIdx.x == 0) carry += part[TILE_THREADS - 1];
            __syncthreads();
        }
        if (threadIdx.x == 0) counts[s] = carry - shard_start;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(TILE_THREADS)
route_scatter_kernel(const gcra_request *__restrict__ req, u32 n, u32 n_shards, u32 num_tiles,
                     const u32 *__restrict__ tile_offsets, gcra_request *__restrict__ out,
                     u32 *__restrict__ src_index) {
    constexpr int NW = TILE_THREADS / 32;
    __shared__ u32 wc[NW][ROUTE_MAX_SHARDS];
    const u32 w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x < NW * ROUTE_MAX_SHARDS) (&wc[0][0])[threadIdx.x] = 0;
    __syncthreads();
    u32 i = blockIdx.x * TILE_THREADS + threadIdx.x;
    bool valid = i < n;
    u32 own = valid ? owner_of(req[i].key_hash, n_shards) : 0;
    u32 peers = __match_any_sync(0xffffffffu, valid ? own : (0x80000000u | lane));
    u32 rank = __popc(peers & ((1u << lane) - 1));
    if (valid && rank == 0) wc[w][own] = __popc(peers);
    __syncthreads();
    if (threadIdx.x < n_shards) {
        u32 acc = 0;
        for (int x = 0; x < NW; x++) { u32 v = wc[x][threadIdx.x]; wc[x][threadIdx.x] = acc; acc += v; }
    }
    __syncthreads();
    if (valid) {
        u32 pos = tile_offsets[own * num_tiles + blockIdx.x] + wc[w][own] + rank;
        const ulonglong2 *s = reinterpret_cast<const ulonglong2 *>(req + i);
        ulonglong2 *d = reinterpret_cast<ulonglong2 *>(out + pos);
        d[0] = s[0]; d[1] = s[1]; d[2] = s[2];
        src_index[pos] = i;
    }
}

__global__ void __launch_bounds__(TILE_THREADS)
route_unpermute_kernel(const gcra_result *__restrict__ routed, const u32 *__restrict__ src_index, u32 n,
                       gcra_result *__restrict__ out) {
    u32 i = blockIdx.x * TILE_THREADS + threadIdx.x;
    if (i < n) {
        const ulonglong2 *s = reinterpret_cast<const ulonglong2 *>(routed + i);
        ulonglong2 *d = reinterpret_cast<ulonglong2 *>(out + src_index[i]);
        d[0] = s[0]; d[1] = s[1];
    }
}

// ---------------------------------------------------------------------------------------------
// snapshot restore (gcra_snapshot_restore): one staged chunk of a snapshot file's key, state and ei sections
// ---------------------------------------------------------------------------------------------
// An entry is carried when its key word is >= 2 and its state is a real entry (has_state(tat + off), expired or
// not, as rehash_kernel keeps them), and shard `rank` of `world` owns it: owner_of(unmix64(key word)).  The key hashes
// whose mix64 is 0 or 1 share the key words 2 and 3 with those whose mix64 is 2 or 3 (stored_key); such a shared entry
// goes to the owner of the unmixed key word, i.e. of the latter.
// COUNT adds the chunk's carried entries to out[0].  INSERT claims their keys through find_or_claim (the placement
// rule of traffic) and writes tat, off and ei verbatim -- unless the key already holds a real entry here, which
// stays (out[2], a conflict); out[1] = inserted, out[3] = keys that found the table full.
enum { RESTORE_OWNED = 0, RESTORE_INSERTED, RESTORE_CONFLICTS, RESTORE_FAILED, RESTORE_COUNTS };

template <bool INSERT>
__global__ void __launch_bounds__(TILE_THREADS)
restore_kernel(Table t, const u64 *__restrict__ keys, const TatOff *__restrict__ state, const i64 *__restrict__ ei,
               u64 n, u32 rank, u32 world, u64 *__restrict__ out) {
    u32 owned = 0, inserted = 0, fresh_n = 0, conflicts = 0, failed = 0;
    const u64 stride = (u64)gridDim.x * TILE_THREADS;
    for (u64 i = (u64)blockIdx.x * TILE_THREADS + threadIdx.x; i < n; i += stride) {
        const ulonglong2 v = ld_stream(&state[i]);
        if (!has_state((i64)(v.x + v.y))) continue;
        const u64 k = keys[i];
        if (k < 2 || owner_of(unmix64(k), world) != rank) continue;
        if (!INSERT) { owned++; continue; }
        bool fresh;
        const u32 s = find_or_claim(t, k, fresh);
        if (s == t.null_slot) { failed++; continue; }
        if (!fresh) {
            const TatOff cur = t.state[s];
            if (has_state((i64)((u64)cur.tat + cur.off))) { conflicts++; continue; }
        }
        *reinterpret_cast<ulonglong2 *>(&t.state[s]) = v;
        t.ei[s] = ei[i];
        inserted++;
        fresh_n += fresh ? 1 : 0;
    }
    owned = __reduce_add_sync(0xffffffffu, owned);
    inserted = __reduce_add_sync(0xffffffffu, inserted);
    fresh_n = __reduce_add_sync(0xffffffffu, fresh_n);
    conflicts = __reduce_add_sync(0xffffffffu, conflicts);
    failed = __reduce_add_sync(0xffffffffu, failed);
    if ((threadIdx.x & 31) == 0) {
        if (owned) atomicAdd(&out[RESTORE_OWNED], (u64)owned);
        if (inserted) {
            atomicAdd(&out[RESTORE_INSERTED], (u64)inserted);
            atomicAdd(&t.counters[C_REAL], (u64)inserted);
        }
        if (fresh_n) atomicAdd(&t.counters[C_OCCUPIED], (u64)fresh_n);
        if (conflicts) atomicAdd(&out[RESTORE_CONFLICTS], (u64)conflicts);
        if (failed) atomicAdd(&out[RESTORE_FAILED], (u64)failed);
    }
}

// ---------------------------------------------------------------------------------------------
// background snapshot (gcra_snapshot_begin): the carried entries of the table, compacted in slot order
// ---------------------------------------------------------------------------------------------
// Carries exactly what restore_kernel and rehash_kernel carry: key word >= 2 and has_state(tat + off), expired but
// unswept entries included.  Persistent CTAs take tiles of SNAP_TILE slots by ticket; a tile's entries go to
// [exclusive prefix, + count) of the three output sections (keys | (tat, off) pairs | ei), the prefix found by a
// decoupled look-back over the tiles' status words.  Every earlier tile was handed to a CTA that runs already, so each
// wait ends.  Positions at or past `cap` are not written; ctrl[SC_ENTRIES] receives the whole count, so a count above
// `cap` tells the host that the output was cut short.  ctrl is zeroed before the launch.
constexpr u32 SNAP_ROWS = 4;                               // rows of 2 x TILE_THREADS slots per tile
constexpr u32 SNAP_TILE = SNAP_ROWS * 2 * TILE_THREADS;
enum { SC_TICKET = 0, SC_ENTRIES, SC_STATUS };             // ctrl words; tile t's status word is ctrl[SC_STATUS + t]
constexpr u64 SC_AGG = 1ULL << 62, SC_INC = 1ULL << 63, SC_COUNT = SC_AGG - 1;

__device__ __forceinline__ u64 ld_volatile_u64(const u64 *p) {
    u64 v;
    asm volatile("ld.volatile.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile_u64(u64 *p, u64 v) {
    asm volatile("st.volatile.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__global__ void __launch_bounds__(TILE_THREADS)
snapshot_capture_kernel(Table t, u64 total_slots, u64 *__restrict__ ctrl, u64 *__restrict__ out_keys,
                        TatOff *__restrict__ out_state, i64 *__restrict__ out_ei, u64 cap) {
    constexpr u32 NW = TILE_THREADS / 32;
    static_assert(SNAP_ROWS * NW == 32, "one warp scans the tile's (row, warp) counts");
    __shared__ u32 wofs[SNAP_ROWS * NW];     // entries of each (row, warp), then their offset in the tile
    __shared__ u64 s_base;
    __shared__ u32 s_tile;
    const u32 w = threadIdx.x >> 5, lane = threadIdx.x & 31, lt = (1u << lane) - 1;
    const u64 num_tiles = (total_slots + SNAP_TILE - 1) / SNAP_TILE;
    for (;;) {
        if (threadIdx.x == 0) s_tile = (u32)atomicAdd(&ctrl[SC_TICKET], 1ULL);
        __syncthreads();
        const u32 tile = s_tile;
        if (tile >= num_tiles) break;                      // uniform over the CTA
        // row r, thread i: slots s and s + 1 (the slot count is a power of two >= 64: both exist or neither)
        const u64 first = (u64)tile * SNAP_TILE + 2 * threadIdx.x;
        ulonglong2 key[SNAP_ROWS], sa[SNAP_ROWS], sb[SNAP_ROWS], ei[SNAP_ROWS];
#pragma unroll
        for (u32 r = 0; r < SNAP_ROWS; r++) {
            const u64 s = first + (u64)r * 2 * TILE_THREADS;
            key[r] = make_ulonglong2(0, 0);
            sa[r] = sb[r] = make_ulonglong2(0, (u64)EXP_EMPTY);
            ei[r] = make_ulonglong2(0, 0);
            if (s < total_slots) {
                key[r] = ld_stream(&t.keys[s]);
                sa[r] = ld_stream(&t.state[s]);
                sb[r] = ld_stream(&t.state[s + 1]);
                ei[r] = ld_stream(&t.ei[s]);
            }
        }
        bool k0[SNAP_ROWS], k1[SNAP_ROWS];
        u32 rank[SNAP_ROWS];
#pragma unroll
        for (u32 r = 0; r < SNAP_ROWS; r++) {
            k0[r] = key[r].x >= 2 && has_state((i64)(sa[r].x + sa[r].y));
            k1[r] = key[r].y >= 2 && has_state((i64)(sb[r].x + sb[r].y));
            const u32 b0 = __ballot_sync(0xffffffffu, k0[r]), b1 = __ballot_sync(0xffffffffu, k1[r]);
            if (lane == 0) wofs[r * NW + w] = __popc(b0) + __popc(b1);
            rank[r] = __popc(b0 & lt) + __popc(b1 & lt);
        }
        __syncthreads();
        if (w == 0) {
            // (row, warp) counts in slot order -> exclusive offsets and the tile's count
            const u32 v = wofs[lane];
            u32 inc = v;
#pragma unroll
            for (u32 o = 1; o < 32; o <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += y;
            }
            wofs[lane] = inc - v;
            const u64 total = __shfl_sync(0xffffffffu, inc, 31);
            u64 excl = 0;
            if (tile > 0) {
                if (lane == 0) st_volatile_u64(&ctrl[SC_STATUS + tile], SC_AGG | total);
                // lane l reads tile j - l; the walk ends at the nearest inclusive prefix (tile 0 publishes one at once)
                for (long long j = (long long)tile - 1;; j -= 32) {
                    const long long idx = j - (long long)lane;
                    u64 st = SC_INC;
                    if (idx >= 0) {
                        do st = ld_volatile_u64(&ctrl[SC_STATUS + idx]); while (st == 0);
                    }
                    const u32 incs = __ballot_sync(0xffffffffu, (st & SC_INC) != 0);
                    const u32 stop = incs ? __ffs(incs) - 1 : 31;
                    u64 part = lane <= stop ? (st & SC_COUNT) : 0;
#pragma unroll
                    for (u32 o = 16; o; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
                    excl += part;
                    if (incs) break;
                }
            }
            if (lane == 0) {
                st_volatile_u64(&ctrl[SC_STATUS + tile], SC_INC | (excl + total));
                if (tile == num_tiles - 1) ctrl[SC_ENTRIES] = excl + total;
                s_base = excl;
            }
        }
        __syncthreads();
        const u64 base = s_base;
#pragma unroll
        for (u32 r = 0; r < SNAP_ROWS; r++) {
            u64 pos = base + wofs[r * NW + w] + rank[r];
            if (k0[r]) {
                if (pos < cap) {
                    out_keys[pos] = key[r].x;
                    *reinterpret_cast<ulonglong2 *>(&out_state[pos]) = sa[r];
                    out_ei[pos] = (i64)ei[r].x;
                }
                pos++;
            }
            if (k1[r] && pos < cap) {
                out_keys[pos] = key[r].y;
                *reinterpret_cast<ulonglong2 *>(&out_state[pos]) = sb[r];
                out_ei[pos] = (i64)ei[r].y;
            }
        }
        __syncthreads();                                   // (s_tile, wofs and s_base are reused by the next tile)
    }
}


// ---------------------------------------------------------------------------------------------
// metrics bridge: denied requests per key, from the kernels' own outputs
// ---------------------------------------------------------------------------------------------
// The reference counts denials per key string in a HashMap and keeps the top N (throttlecrab-server/src/
// metrics.rs:24-64,162-173).  Here a pass over a finished batch (request rows + result rows) counts the denied rows
// per key hash: every 256-row tile aggregates in a shared-memory hash set, then adds each distinct key's count to an
// open-addressed table in HBM -- a key already in the table costs a load and a posted add, only a new key a CAS.
// A full table drops new keys (counted); gcra_top_denied prunes it to the top entries like the reference's cleanup.
struct DeniedTable {
    u64 *keys;      // 0 = empty
    u64 *counts;
    u32 mask;       // capacity - 1
    u64 *dropped;
};
constexpr u32 DENIED_HASH = 512;

// one denied row of key `k` into the tile's shared-memory hash set
__device__ __forceinline__ void denied_tile_add(u64 *hkey, u32 *hcnt, u64 k) {
    if (k == 0) k = 1;                                                              // 0 marks an empty entry
    u32 h = (u32)(mix64(k) >> 55);                                                  // 9 bits
    for (;;) {
        const u64 old = atomicCAS(&hkey[h], 0ULL, k);
        if (old == 0 || old == k) { atomicAdd(&hcnt[h], 1u); break; }
        h = (h + 1) & (DENIED_HASH - 1);
    }
}

// the tile's distinct keys into the table (after a __syncthreads that follows the tile's adds)
__device__ __forceinline__ void denied_tile_flush(const u64 *hkey, const u32 *hcnt, const DeniedTable &t) {
    for (u32 e = threadIdx.x; e < DENIED_HASH; e += TILE_THREADS) {
        const u64 k = hkey[e];
        if (k == 0) continue;
        u32 h = (u32)(mix64(k ^ 0x9E3779B97F4A7C15ULL)) & t.mask;
        bool done = false;
        for (u32 probe = 0; probe < 64 && !done; probe++) {
            u64 cur = t.keys[h];                                    // (a stale L1 line shows "empty": then the CAS decides)
            if (cur == 0) { const u64 old = atomicCAS(&t.keys[h], 0ULL, k); cur = old == 0 ? k : old; }
            if (cur == k) { atomicAdd(&t.counts[h], (u64)hcnt[e]); done = true; }
            else h = (h + 1) & t.mask;
        }
        if (!done) atomicAdd(t.dropped, (u64)hcnt[e]);
    }
}

// single-segment batch: one CTA per 256-row tile
template <int FMT>
__global__ void __launch_bounds__(TILE_THREADS)
denied_count_kernel(const unsigned char *__restrict__ req, const gcra_result *__restrict__ res, u32 n, DeniedTable t) {
    __shared__ u64 hkey[DENIED_HASH];
    __shared__ u32 hcnt[DENIED_HASH];
    for (u32 i = threadIdx.x; i < DENIED_HASH; i += TILE_THREADS) { hkey[i] = 0; hcnt[i] = 0; }
    __syncthreads();
    const u32 i = blockIdx.x * TILE_THREADS + threadIdx.x;
    if (i < n) {
        // (retry_after | cur_tat_ns), status | allowed << 32: the second half of a 32-byte row, a whole 16-byte row
        const longlong2 tail = Rows<FMT>::R16 ? reinterpret_cast<const longlong2 *>(res)[i]
                                              : reinterpret_cast<const longlong2 *>(res + i)[1];
        const bool denied = (u32)tail.y == GCRA_OK && ((tail.y >> 32) & 0xff) == 0;
        if (denied) denied_tile_add(hkey, hcnt, *reinterpret_cast<const u64 *>(req + (size_t)i * Rows<FMT>::REQ_BYTES));
    }
    __syncthreads();
    denied_tile_flush(hkey, hcnt, t);
}

// Segmented batch (the peer-memory tick: 48-byte requests in this GPU's inbox, 32-byte results in the senders'
// outboxes, one segment per sender).  The segments' row counts exist only on the device, and the row-id space
// (nseg << cap_shift) is mostly empty, so a persistent grid turns a dense tile index into (segment, tile) with a
// prefix over the counts and takes tiles until the real rows run out.  Per tile: as denied_count_kernel.
__global__ void __launch_bounds__(TILE_THREADS)
denied_count_seg_kernel(BatchView v, DeniedTable t) {
    __shared__ u64 hkey[DENIED_HASH];
    __shared__ u32 hcnt[DENIED_HASH];
    __shared__ u32 s_cnt[MAX_SEGS], s_tile0[MAX_SEGS + 1];     // rows of segment s, its first dense tile
    if (threadIdx.x < MAX_SEGS) s_cnt[threadIdx.x] = threadIdx.x < v.nseg ? min(v.dev_counts[threadIdx.x], 1u << v.cap_shift) : 0;
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 acc = 0;
        for (u32 s = 0; s < MAX_SEGS; s++) { s_tile0[s] = acc; acc += (s_cnt[s] + TILE_THREADS - 1) / TILE_THREADS; }
        s_tile0[MAX_SEGS] = acc;
    }
    __syncthreads();
    const u32 n_tiles = s_tile0[MAX_SEGS];
    for (u32 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        for (u32 i = threadIdx.x; i < DENIED_HASH; i += TILE_THREADS) { hkey[i] = 0; hcnt[i] = 0; }
        u32 s = 0;
        while (tile >= s_tile0[s + 1]) s++;                     // (uniform over the CTA: s < nseg)
        const u32 j = (tile - s_tile0[s]) * TILE_THREADS + threadIdx.x;
        __syncthreads();
        if (j < s_cnt[s]) {
            const u32 row = (s << v.cap_shift) | j;
            const longlong2 tail = reinterpret_cast<const longlong2 *>(v.res_at(row))[1];      // as above, 32-byte rows
            const bool denied = (u32)tail.y == GCRA_OK && ((tail.y >> 32) & 0xff) == 0;
            if (denied) denied_tile_add(hkey, hcnt, *reinterpret_cast<const u64 *>(v.req_at(row, sizeof(gcra_request))));
        }
        __syncthreads();
        denied_tile_flush(hkey, hcnt, t);
        __syncthreads();                                        // (the hash set is cleared for the next tile)
    }
}

// ---------------------------------------------------------------------------------------------
// K0 hash pass: key references -> key hashes, in place
// ---------------------------------------------------------------------------------------------
// A row's key_hash field (offset 0 in both request formats) holds GCRA_KEY_REF(off, len): the key is the bytes
// [off, off + len) of the caller's arena.  One lane per row.  A warp stages the span its 32 keys cover into shared
// memory with aligned 16-byte loads when the span fits HASH_STAGE (consecutive rows' keys lie close together, as a
// ring slot or the RESP parser lays them out); otherwise every lane reads its own key from global memory.  Both
// paths feed the same hash (gcra_device.cuh), so a key's hash does not depend on the layout.  Nothing outside
// [keys, keys + keys_len) is read: a 16-byte chunk of the staging that is not wholly inside the arena is copied
// byte by byte.
constexpr u32 HASH_STAGE = 2048;                   // bytes a warp stages: 32 keys of up to ~60 bytes
constexpr u32 HASH_WARPS = TILE_THREADS / 32;

// a key in a warp's staging: 64-bit words from aligned 32-bit shared loads and funnel shifts (the staging is padded
// by 16 bytes, so a word read for the last bytes of a key stays inside it)
struct StagedBytes {
    const u32 *base;                               // the warp's staging
    u32 pos;                                       // the key's first byte in it
    __device__ __forceinline__ u64 word(u64 i) const {
        const u32 a = pos + (u32)i, sh = (a & 3) * 8;
        const u32 *w = base + (a >> 2);
        const u32 w0 = w[0], w1 = w[1], w2 = w[2];
        return (u64)__funnelshift_r(w0, w1, sh) | ((u64)__funnelshift_r(w1, w2, sh) << 32);
    }
    __device__ __forceinline__ u64 tail(u64 i, u32 r) const { return r ? word(i) & ((1ULL << (8 * r)) - 1) : 0; }
};

__global__ void __launch_bounds__(TILE_THREADS)
hash_keys_kernel(unsigned char *rows, u32 n, u32 row_bytes, const unsigned char *keys, u64 keys_len, u64 k0, u64 k1) {
    __shared__ __align__(16) u32 stage[HASH_WARPS][(HASH_STAGE + 16) / 4];
    const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const u64 i = (u64)blockIdx.x * TILE_THREADS + threadIdx.x;
    const bool active = i < n;
    u64 *row = reinterpret_cast<u64 *>(rows + i * row_bytes);
    const u64 ref = active ? row[0] : 0;
    const u32 off = (u32)ref, len = (u32)(ref >> 32);
    const bool ok = active && (u64)off + len <= keys_len;
    // the warp's span [lo, lo + ext) over its in-arena keys with at least one byte
    const bool used = ok && len > 0;
    const u32 lo = __reduce_min_sync(0xffffffffu, used ? off : 0xffffffffu);
    const u32 ext = __reduce_max_sync(0xffffffffu, used ? (u32)min((u64)off + len - lo, 0xffffffffULL) : 0u);
    const uintptr_t g0 = chunk_begin((uintptr_t)keys, lo);
    const bool staged = ext > 0 && chunk_end((uintptr_t)keys, lo, ext) - g0 <= HASH_STAGE;   // (uniform over the warp)
    if (staged) {
        unsigned char *sb = reinterpret_cast<unsigned char *>(stage[wid]);
        stage_key_span((uintptr_t)keys, keys_len, lo, ext, lane, 32,
                       [&](uintptr_t src, u32 dst) {
                           *reinterpret_cast<uint4 *>(sb + dst) = __ldg(reinterpret_cast<const uint4 *>(src));
                       },
                       [&](uintptr_t src, u32 dst) { sb[dst] = *reinterpret_cast<const unsigned char *>(src); });
        __syncwarp();
    }
    if (!active) return;
    if (!ok) {
        // a reference that leaves the arena: a row the decide kernels answer GCRA_INTERNAL without touching an entry
        row[0] = 0;
        if (row_bytes == sizeof(gcra_request)) row[5] = ~0ULL;                           // now_ns = -1 (pre-epoch)
        else reinterpret_cast<u32 *>(row)[3] = 0xffffffffu;                              // policy >= any npol
        return;
    }
    row[0] = staged && len > 0
        ? hash_key_engine(StagedBytes{stage[wid], (u32)((uintptr_t)keys + off - g0)}, len, k0, k1)
        : hash_key_engine(KeyBytes{keys + off}, len, k0, k1);
}

}  // namespace gcra
