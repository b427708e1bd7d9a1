// gcra_index_path.cuh -- the index-order K1 pipeline (large batches).
//
// The sort path (gcra_kernels.cuh: ingest -> radix sort by slot -> warp-cooperative decide) groups ALL
// requests of a batch by key before a single decision is made; every request then pays a gather and a scatter
// by batch index.  Most requests do not need that.  The reference applies requests one at a time
// (throttlecrab-server/src/actor.rs:217-236), and a request that is denied -- or that leaves the entry
// bit-for-bit unchanged -- does not alter what later requests on its key observe (rate_limiter.rs:186-204: only
// an allowed request writes).  So, with S0 = the state of a key when the batch starts and i1 < i2 < ... its
// requests in batch order, let m be the FIRST request whose decision against S0 changes the state.  Then every
// request up to and including m is decided exactly by decide(S0, request) -- independently of all the others,
// in any order, on any thread -- and only the requests BEHIND m need the state m leaves.  Three streaming
// passes in batch-index order (coalesced request reads and result writes; the only random accesses are the key
// sector and the 16-byte state pair), then the sort path on the residue only:
//
//   A  probe_kernel          TMA-staged request tile, validation, key -> slot probe/claim (gcra_device.cuh);
//                            writes slot[i]; counts every slot in hashed batch counters (>= 2: the key is shared)
//   B  decide_index_kernel   decide(S0, request) for every request, result written in place.  A request whose
//                            slot was seen once is alone on its key: its new state is committed right away.
//                            A state-changing request on a shared slot records its index with
//                            atomicMin(mark[slot]) (epoch-tagged, so marks never need clearing)
//   C  resolve_kernel        requests on shared slots: before the first state change -> final; the first state
//                            change itself -> commits its state; behind it -> appended, in batch order
//                            (decoupled look-back compaction), to the residue
//   residue                  the sort path over the residue only: it starts from the states C committed and
//                            applies the rest one after another (speculate-and-commit / finite-state rounds)
//
// The three stages (A+A' | B+C | residue) of consecutive batches run on three streams.  So that B+C of batch
// j+1 may overlap the residue of batch j, pass C leaves a PEND bit for every key it sends to the residue in the
// NEXT batch's pend bitmap: batch j+1 does not evaluate requests on such keys in pass B, it defers them to its own
// residue (residues run strictly one after another).
//
// In the steady state of a rate limiter the hot keys are saturated (0-1 state changes per tick), so the
// residue is the handful of keys that toggle state (max_burst = 1 with zero-quantity requests, SURVEY V8); a
// 60 K-request run on the hottest key is decided by 60 K independent threads in pass B.
#pragma once
#include "gcra_kernels.cuh"

namespace gcra {

struct TileRef {
    u32 row0;                    // row id of the tile's first row
    u32 cnt;                     // rows in the tile (1..TILE_THREADS)
    const unsigned char *req;    // the tile's first request record
};

// tile `t` of the batch in row-id order; false past the last tile (uniform over the CTA)
__device__ __forceinline__ bool tile_lookup(const BatchView &b, u32 t, u32 rsz, TileRef &r) {
    if (b.nseg == 1) {
        const u64 row0 = (u64)t * TILE_THREADS;
        if (row0 >= b.n) return false;
        r.row0 = (u32)row0;
        r.cnt = min((u32)TILE_THREADS, b.n - (u32)row0);
        r.req = b.req0 + (size_t)row0 * rsz;
        return true;
    }
    const u32 cap = 1u << b.cap_shift;
    for (u32 s = 0; s < b.nseg; s++) {
        const u32 c = min(__ldg(&b.dev_counts[s]), cap);
        const u32 tiles = (c + TILE_THREADS - 1) / TILE_THREADS;
        if (t < tiles) {
            const u32 j0 = t * TILE_THREADS;
            r.row0 = (s << b.cap_shift) | j0;
            r.cnt = min((u32)TILE_THREADS, c - j0);
            r.req = (const unsigned char *)__ldg((const u64 *)&b.segs[s].req) + (size_t)j0 * rsz;
            return true;
        }
        t -= tiles;
    }
    return false;
}

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// stage one request tile into shared memory with ONE 1-D bulk async copy (SASS: UBLKCP) and wait for it
__device__ __forceinline__ void stage_tile(unsigned char *stage, u64 *bar, const TileRef &tr, u32 rsz, u32 &parity) {
    if (threadIdx.x == 0) {
        fence_proxy_async();          // the previous tile's generic-proxy reads are ordered before this write
        mbar_expect_tx(bar, tr.cnt * rsz);
        bulk_g2s(stage, tr.req, tr.cnt * rsz, bar);
    }
    mbar_wait(bar, parity);
    parity ^= 1;
}

// Batch-local knowledge about slots, both hashed by (slot & mask) -- a hashed index only merges slots, and a false
// "shared" / "pending" verdict costs time, never exactness:
//   counters  32 bits per entry: how often the entry's slots occur in THIS batch, as far as that matters: pass A
//             finds the distinct slots of every 256-row tile with a hash set in shared memory and adds
//             min(count in the tile, 2) per distinct slot with ONE posted RED (no global atomic ever returns a
//             value: returning atomics are throttled by the few that an SM can keep in flight).  >= 2 <=> shared.
//             A tile adds at most its row count (256) to an entry, whatever slots share the entry, so an entry
//             never exceeds the batch's rows -- below INDEX_MAX_ROWS, which a 32-bit counter holds.  (16-bit
//             counters would wrap: one key in every row of a 2^23-row multi-GPU tick adds 2 x 32768 = 65536.)
//   pend      1 bit per entry, written by the PREVIOUS batch's pass C: a slot of the entry still has residue
//             requests in that batch's sorted tail, which may run concurrently with this batch's passes B and C;
//             this batch's requests on such a slot are deferred to its own tail (tails run one after another)
// Row ids of an index-order batch: a single batch has at most 2^21 rows (use_index_path), a multi-GPU tick spans
// world x cap_rows < 2^31 row ids (gcra_p2p_prepare).
constexpr u64 INDEX_MAX_ROWS = 1ULL << 31;
static_assert(INDEX_MAX_ROWS - 1 <= 0xFFFFFFFFull, "a 32-bit batch counter holds the row count of any index-order batch");
__device__ __forceinline__ u32 counter_of(const u32 *__restrict__ cnt, u32 mask, u32 slot) {
    return __ldg(cnt + (slot & mask));
}
__device__ __forceinline__ bool pend_of(const u32 *__restrict__ pend, u32 mask, u32 slot) {
    const u32 e = slot & mask;
    return (__ldg(pend + (e >> 5)) >> (e & 31)) & 1;
}

// ---------------------------------------------------------------------------------------------
// pass A: probe
// ---------------------------------------------------------------------------------------------
// Persistent CTAs over the tiles, software-pipelined one tile deep: while tile t is probed, the request tile t+1
// already sits in the second stage buffer (bulk async copy) and its rows' first-choice key sectors are in
// flight into registers -- a row's DRAM round trip overlaps the work of a whole tile instead of stalling it.
constexpr u32 NOTE_HASH_BITS = 9, NOTE_HASH = 1u << NOTE_HASH_BITS;   // hash set of one 256-row tile (load <= 1/2)

struct KeyProbe {
    u64 k;            // stored key
    u32 b1, b2;       // bucket choices
    ulonglong2 a, b;  // the four keys of bucket 1 (through L1, see find_in_buckets_cached)
};

__device__ __forceinline__ void probe_start(const Table &t, const unsigned char *rec, bool in_range, KeyProbe &kp) {
    kp.k = 0; kp.b1 = 0; kp.b2 = 0;
    kp.a = make_ulonglong2(0, 0); kp.b = kp.a;
    if (!in_range) return;
    kp.k = stored_key(*reinterpret_cast<const u64 *>(rec));      // both request formats start with the key hash
    bucket_choices(t, kp.k, kp.b1, kp.b2);
    const ulonglong2 *p1 = reinterpret_cast<const ulonglong2 *>(t.keys + (size_t)kp.b1 * 4);
    kp.a = p1[0];
    kp.b = p1[1];
}

__device__ __forceinline__ u32 probe_finish(const Table &t, const KeyProbe &kp, bool &fresh) {
    fresh = false;
    if (kp.a.x == kp.k) return kp.b1 * 4;
    if (kp.a.y == kp.k) return kp.b1 * 4 + 1;
    if (kp.b.x == kp.k) return kp.b1 * 4 + 2;
    if (kp.b.y == kp.k) return kp.b1 * 4 + 3;
    return find_or_claim_coherent(t, kp.k, kp.b1, kp.b2, fresh);
}

__device__ __forceinline__ void issue_tile(unsigned char *stage, u64 *bar, const TileRef &tr, u32 rsz) {
    fence_proxy_async();          // earlier generic-proxy reads of this buffer are ordered before the async write
    mbar_expect_tx(bar, tr.cnt * rsz);
    bulk_g2s(stage, tr.req, tr.cnt * rsz, bar);
}

template <int FMT>
__global__ void __launch_bounds__(TILE_THREADS)
probe_kernel(Table t, BatchView b, const PolicyDerived *__restrict__ pol, u32 npol, i64 now_batch,
             u32 *__restrict__ slot_arr, u32 *__restrict__ counters, u32 bm_mask, int prefetch_state) {
    using Row = Rows<FMT>;
    __shared__ __align__(128) unsigned char stage[2][TILE_THREADS * Row::REQ_BYTES];
    __shared__ __align__(8) u64 bar[2];
    // the distinct slots of the current tile and how often each occurs (see "counters" above)
    __shared__ u32 hkey[NOTE_HASH];
    __shared__ u32 hcnt[NOTE_HASH];
    for (u32 i = threadIdx.x; i < NOTE_HASH; i += TILE_THREADS) { hkey[i] = 0xFFFFFFFFu; hcnt[i] = 0; }
    if (threadIdx.x == 0) {
        mbar_init(&bar[0], 1);
        mbar_init(&bar[1], 1);
        fence_barrier_init();
    }
    __syncthreads();
    const u32 G = gridDim.x;
    u32 tile = blockIdx.x;
    TileRef cur, nxt;
    if (!tile_lookup(b, tile, Row::REQ_BYTES, cur)) return;
    bool has_nxt = tile_lookup(b, tile + G, Row::REQ_BYTES, nxt);
    if (threadIdx.x == 0) {
        issue_tile(stage[0], &bar[0], cur, Row::REQ_BYTES);
        if (has_nxt) issue_tile(stage[1], &bar[1], nxt, Row::REQ_BYTES);
    }
    u32 par = 0;                 // phase parity of the two barriers, one bit each
    u32 buf = 0;
    mbar_wait(&bar[0], 0);
    par ^= 1;
    KeyProbe kc;
    probe_start(t, stage[0] + (size_t)threadIdx.x * Row::REQ_BYTES, threadIdx.x < cur.cnt, kc);
    u32 n_fresh = 0, n_err = 0;
    for (;;) {
        KeyProbe kn;
        if (has_nxt) {
            mbar_wait(&bar[buf ^ 1], (par >> (buf ^ 1)) & 1);
            par ^= 1u << (buf ^ 1);
            probe_start(t, stage[buf ^ 1] + (size_t)threadIdx.x * Row::REQ_BYTES, threadIdx.x < nxt.cnt, kn);
        }
        const bool in_range = threadIdx.x < cur.cnt;
        const u32 row = cur.row0 + threadIdx.x;
        if (in_range) {
            u64 key_hash = 0;
            Req r = {0, 0, 0, 0};
            int status = parse_request<Row::COMPACT>(stage[buf] + (size_t)threadIdx.x * Row::REQ_BYTES, pol, npol, now_batch, key_hash, r);
            u32 slot = t.null_slot;
            if (status == 0) {
                bool fresh;
                slot = probe_finish(t, kc, fresh);
                n_fresh += fresh ? 1 : 0;
                if (slot == t.null_slot) status = GCRA_INTERNAL;   // table full
            }
            slot_arr[row] = slot;
            if (status != 0) {
                if (Row::R16) write_result16(b.res16_at(row), 0, status, 0);
                else write_result(b.res_at(row), 0, 0, 0, status, 0);
                n_err++;
            }
            else {
                // the state pair is what pass B touches next: optionally pull its sector into L2 now
                if (prefetch_state) asm volatile("prefetch.global.L2 [%0];" ::"l"(&t.state[slot]));
                u32 h = (slot * 0x9E3779B1u) >> (32 - NOTE_HASH_BITS);
                for (;;) {
                    const u32 old = atomicCAS(&hkey[h], 0xFFFFFFFFu, slot);
                    if (old == 0xFFFFFFFFu || old == slot) { atomicAdd(&hcnt[h], 1u); break; }
                    h = (h + 1) & (NOTE_HASH - 1);
                }
            }
        }
        __syncthreads();   // everybody is done with stage[buf]; the tile's hash set is complete
        // one posted add per distinct slot of the tile (result unused: RED.ADD), and the set is empty again
        for (u32 i = threadIdx.x; i < NOTE_HASH; i += TILE_THREADS) {
            const u32 sl = hkey[i];
            if (sl == 0xFFFFFFFFu) continue;
            atomicAdd(counters + (sl & bm_mask), min(hcnt[i], 2u));
            hkey[i] = 0xFFFFFFFFu;
            hcnt[i] = 0;
        }
        __syncthreads();
        if (!has_nxt) break;
        tile += G;
        cur = nxt;
        kc = kn;
        has_nxt = tile_lookup(b, tile + G, Row::REQ_BYTES, nxt);
        if (has_nxt && threadIdx.x == 0) issue_tile(stage[buf], &bar[buf], nxt, Row::REQ_BYTES);
        buf ^= 1;
    }
    n_fresh = __reduce_add_sync(0xffffffffu, n_fresh);
    n_err = __reduce_add_sync(0xffffffffu, n_err);
    if ((threadIdx.x & 31) == 0) {
        if (n_fresh) atomicAdd(&t.counters[C_OCCUPIED], (u64)n_fresh);
        if (n_err) atomicAdd(&t.counters[C_ERRORS], (u64)n_err);
    }
}

constexpr int RES_ROWS = 4;                                  // rows per thread (note, resolve)
constexpr int RES_TILE = TILE_THREADS * RES_ROWS;            // rows per CTA tile: a whole number of probe tiles

// tile `t` of RES_TILE rows in row-id order (segments are padded to whole tiles in the row-id space)
__device__ __forceinline__ bool res_tile_lookup(const BatchView &b, u32 t, u32 &row0, u32 &cnt) {
    if (b.nseg == 1) {
        const u64 r0 = (u64)t * RES_TILE;
        if (r0 >= b.n) return false;
        row0 = (u32)r0;
        cnt = min((u32)RES_TILE, b.n - row0);
        return true;
    }
    const u32 cap = 1u << b.cap_shift;
    for (u32 s = 0; s < b.nseg; s++) {
        const u32 c = min(__ldg(&b.dev_counts[s]), cap);
        const u32 tiles = (c + RES_TILE - 1) / RES_TILE;
        if (t < tiles) {
            row0 = (s << b.cap_shift) | (t * RES_TILE);
            cnt = min((u32)RES_TILE, c - t * RES_TILE);
            return true;
        }
        t -= tiles;
    }
    return false;
}

// ---------------------------------------------------------------------------------------------
// pass B: decide every request against the state its key had when the batch started
// ---------------------------------------------------------------------------------------------
constexpr unsigned char F_ALLOWED = 1, F_MUTATES = 2, F_EXP_HIT = 4, F_DEFER = 8, F_SHARED = 16;

__device__ __forceinline__ u64 mark_value(u32 epoch, u32 row) { return ((u64)(~epoch) << 32) | row; }

#ifndef GCRA_B_MINBLOCKS
#define GCRA_B_MINBLOCKS 1
#endif
// Persistent CTAs, software-pipelined: while tile t is decided, tile t+1's requests sit in the second stage buffer,
// its rows' state pairs, counters and pend bits are in flight into registers, and tile t+2's slots are being read.
template <int FMT>
__global__ void __launch_bounds__(TILE_THREADS, GCRA_B_MINBLOCKS)
decide_index_kernel(Table t, BatchView b, const PolicyDerived *__restrict__ pol, u32 npol, i64 now_batch,
                    const u32 *__restrict__ slot_arr, const u32 *__restrict__ counters, const u32 *__restrict__ pend,
                    u32 bm_mask, unsigned char *__restrict__ flags, u32 epoch, u32 honour_pend, u32 dbg) {
    using Row = Rows<FMT>;
    constexpr u32 PIECES = Row::RES_BYTES / 16;       // 16-byte pieces per result row
    __shared__ __align__(128) unsigned char stage[2][TILE_THREADS * Row::REQ_BYTES];
    __shared__ __align__(8) u64 bar[2];
    // results leave through shared memory: a tile's 256 results are written out as 256 x PIECES consecutive 16-byte
    // pieces (a warp store covers 512 contiguous bytes: 16 rows of 32 bytes, 32 rows of 16).  A segment's result array
    // may be a peer GPU's outbox: a lane storing the two halves of its own row would put 16-byte packets on NVLink.
    __shared__ __align__(16) longlong2 rstage[2][TILE_THREADS * PIECES];
    __shared__ unsigned char rwrite[2][TILE_THREADS];
    if (threadIdx.x == 0) {
        mbar_init(&bar[0], 1);
        mbar_init(&bar[1], 1);
        fence_barrier_init();
    }
    __syncthreads();
    const u32 G = gridDim.x;
    u32 tile = blockIdx.x;
    TileRef cur, nxt, nn;
    if (!tile_lookup(b, tile, Row::REQ_BYTES, cur)) return;
    bool has_nxt = tile_lookup(b, tile + G, Row::REQ_BYTES, nxt);
    if (threadIdx.x == 0) {
        issue_tile(stage[0], &bar[0], cur, Row::REQ_BYTES);
        if (has_nxt) issue_tile(stage[1], &bar[1], nxt, Row::REQ_BYTES);
    }
    u32 par = 0;                 // phase parity of the two barriers, one bit each
    u32 buf = 0;
    u32 slot_c = threadIdx.x < cur.cnt ? slot_arr[cur.row0 + threadIdx.x] : t.null_slot;
    u32 slot_n = (has_nxt && threadIdx.x < nxt.cnt) ? slot_arr[nxt.row0 + threadIdx.x] : t.null_slot;
    RunState s_c = {0, EXP_EMPTY, 0};
    u32 bits_c = 0;
    // bits: F_SHARED (the batch holds the key at least twice) | F_DEFER (the previous batch's tail owns it)
    if (slot_c != t.null_slot) {
        if (!(dbg & 16)) load_state(t, slot_c, s_c);
        if (!(dbg & 32)) bits_c = (counter_of(counters, bm_mask, slot_c) >= 2 ? F_SHARED : 0) |
                                  ((honour_pend && pend_of(pend, bm_mask, slot_c)) ? F_DEFER : 0);
    }
    u32 n_allowed = 0, n_denied = 0, exp_hits = 0, real_inc = 0;
    for (;;) {
        // next tile: the random accesses go out now, their data is used one iteration later
        RunState s_n = {0, EXP_EMPTY, 0};
        u32 bits_n = 0;
        if (slot_n != t.null_slot) {
            if (!(dbg & 16)) load_state(t, slot_n, s_n);
            if (!(dbg & 32)) bits_n = (counter_of(counters, bm_mask, slot_n) >= 2 ? F_SHARED : 0) |
                                      ((honour_pend && pend_of(pend, bm_mask, slot_n)) ? F_DEFER : 0);
        }
        // the tile after that: its slots
        const bool has_nn = has_nxt && tile_lookup(b, tile + 2 * G, Row::REQ_BYTES, nn);
        const u32 slot_nn = (has_nn && threadIdx.x < nn.cnt) ? slot_arr[nn.row0 + threadIdx.x] : t.null_slot;

        mbar_wait(&bar[buf], (par >> buf) & 1);
        par ^= 1u << buf;
        const u32 row = cur.row0 + threadIdx.x;
        const u32 slot = slot_c;
        const RunState s = s_c;
        const u32 bits = bits_c;
        rwrite[buf][threadIdx.x] = 0;
        if (slot != t.null_slot && (bits & F_DEFER)) {
            // the previous batch still works on this key (or on one sharing its entry): not evaluated here, the
            // whole key goes to this batch's sorted tail
            flags[row] = F_DEFER;
        } else if (slot != t.null_slot) {
            u64 key_hash;
            Req r;
            parse_request<Row::COMPACT>(stage[buf] + (size_t)threadIdx.x * Row::REQ_BYTES, pol, npol, now_batch, key_hash, r);
            Decision d;
            Outputs o;
            if (dbg & 8) { d.allowed = (r.q & 1) != 0; d.live = true; d.new_tat = r.now; d.new_exp = r.now + r.dvt; d.tat = s.tat; d.allow_at = 0; o.remaining = r.q; o.reset_after = r.ei; o.retry_after = 0; }
            else { d = decide(s.tat, s.exp, r); if (!Row::R16) o = outputs_of(d, r); }
            if (!(dbg & 2)) {
                if (Row::R16) {
                    rstage[buf][threadIdx.x] = make_longlong2(d.allowed ? d.new_tat : d.tat, (i64)(u32)0 | ((i64)(d.allowed ? 1 : 0) << 32));
                } else {
                    rstage[buf][threadIdx.x * 2] = make_longlong2(o.remaining, o.reset_after);
                    rstage[buf][threadIdx.x * 2 + 1] = make_longlong2(o.retry_after, (i64)(u32)0 | ((i64)(d.allowed ? 1 : 0) << 32));
                }
                rwrite[buf][threadIdx.x] = 1;
            }
            const bool mut = d.allowed && ((d.new_tat != s.tat) | (d.new_exp != s.exp));
            // a write over an entry that exists but is expired (adaptive_cleanup.rs:233,267)
            const bool hit = d.allowed && !d.live && has_state(s.exp);
            if (!(bits & F_SHARED)) {
                // the only request of the batch on this key: final, and its write is the key's only write
                flags[row] = 0;
                if (mut && !(dbg & 1)) {
                    const bool created = !has_state(s.exp);
                    RunState ns = {d.new_tat, d.new_exp, r.ei};
                    store_state(t, slot, ns, created);
                    real_inc += created ? 1 : 0;
                }
                n_allowed += d.allowed ? 1 : 0;
                n_denied += d.allowed ? 0 : 1;
                exp_hits += hit ? 1 : 0;
            } else {
                flags[row] = (unsigned char)(F_SHARED | (d.allowed ? F_ALLOWED : 0) | (mut ? F_MUTATES : 0) | (hit ? F_EXP_HIT : 0));
                if (mut && !(dbg & 4)) {
                    // marks only ever decrease while this kernel runs, so a (possibly stale, L1) value at or below
                    // mine proves an earlier state change is already recorded: hot keys cost one L2 read per SM
                    // and a handful of atomics instead of one same-address atomic per request
                    const u64 mine = mark_value(epoch, row);
                    if (t.mark[slot] > mine) atomicMin(&t.mark[slot], mine);   // result unused: RED.MIN
                }
            }
        }
        __syncthreads();   // everybody is done with stage[buf]; the tile's results are staged
        {
            // rows that failed validation (pass A wrote their error) or were deferred (the tail will write them) keep
            // their place: only staged rows are stored
            longlong2 *dst = Row::R16 ? reinterpret_cast<longlong2 *>(b.res16_at(cur.row0)) : reinterpret_cast<longlong2 *>(b.res_at(cur.row0));
#pragma unroll
            for (int k = 0; k < (int)PIECES; k++) {
                const u32 c = threadIdx.x + k * TILE_THREADS;
                if (rwrite[buf][c / PIECES]) dst[c] = rstage[buf][c];
            }
        }
        if (!has_nxt) break;
        if (has_nn && threadIdx.x == 0) issue_tile(stage[buf], &bar[buf], nn, Row::REQ_BYTES);
        tile += G;
        cur = nxt; nxt = nn;
        slot_c = slot_n; s_c = s_n; bits_c = bits_n;
        slot_n = slot_nn;
        has_nxt = has_nn;
        buf ^= 1;
    }
    n_allowed = __reduce_add_sync(0xffffffffu, n_allowed);
    n_denied = __reduce_add_sync(0xffffffffu, n_denied);
    real_inc = __reduce_add_sync(0xffffffffu, real_inc);
    exp_hits = __reduce_add_sync(0xffffffffu, exp_hits);
    if ((threadIdx.x & 31) == 0) {
        if (n_allowed) atomicAdd(&t.counters[C_ALLOWED], (u64)n_allowed);
        if (n_denied) atomicAdd(&t.counters[C_DENIED], (u64)n_denied);
        if (real_inc) atomicAdd(&t.counters[C_REAL], (u64)real_inc);
        if (exp_hits) atomicAdd(&t.counters[C_EXPIRED_HITS], (u64)exp_hits);
    }
}

// ---------------------------------------------------------------------------------------------
// pass C: requests on shared slots -- final / first state change (commit) / residue (stable compaction)
// ---------------------------------------------------------------------------------------------
// control block of one batch: word 0 = {tile ticket, residue count}, then one status word per tile.
// Tiles are handed out in order to RUNNING CTAs (ticket), so the decoupled look-back only ever waits for a tile
// whose CTA already runs, whatever else shares the GPU.
constexpr u32 RC_TICKET = 0, RC_NRES = 1;
constexpr u64 TS_AGG = 1ULL << 62, TS_INC = 2ULL << 62, TS_MASK = 3ULL << 62;

// exclusive prefix of this tile's residue count over all earlier tiles (warp 0 calls it, result uniform)
__device__ __forceinline__ u32 lookback(volatile u64 *__restrict__ status, u32 tile, u32 total, u32 lane) {
    if (tile == 0) {
        if (lane == 0) status[0] = TS_INC | total;
        return 0;
    }
    if (lane == 0) status[tile] = TS_AGG | total;
    u32 base = 0;
    int j = (int)tile - 1;            // nearest predecessor not yet accounted for
    for (;;) {
        const int idx = j - (int)lane;
        u64 v = TS_INC;               // before tile 0: an inclusive prefix of 0
        if (idx >= 0) {
            do { v = status[idx]; } while ((v & TS_MASK) == 0);
        }
        const u32 inc = __ballot_sync(0xffffffffu, (v & TS_MASK) == TS_INC);
        const int stop = inc ? (__ffs(inc) - 1) : 31;           // lanes 0..stop contribute
        const u32 contrib = (int)lane <= stop ? (u32)v : 0;
        base += __reduce_add_sync(0xffffffffu, contrib);
        if (inc) break;
        j -= 32;
    }
    if (lane == 0) status[tile] = TS_INC | (u64)(base + total);
    return base;
}

template <int FMT>
__global__ void __launch_bounds__(TILE_THREADS)
resolve_kernel(Table t, BatchView b, const PolicyDerived *__restrict__ pol, u32 npol, i64 now_batch,
               const u32 *__restrict__ slot_arr, u32 bm_mask,
               const unsigned char *__restrict__ flags, u32 epoch, u32 *__restrict__ ctrl,
               volatile u64 *__restrict__ tile_status, u64 *__restrict__ res_keys,
               u32 *__restrict__ next_pend, volatile u32 *__restrict__ host_nres, u32 res_cap) {
    using Row = Rows<FMT>;
    __shared__ u32 part[TILE_THREADS / 32];
    __shared__ u32 sm_tile, sm_base;
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 n_allowed = 0, n_denied = 0, exp_hits = 0, real_inc = 0;
    for (;;) {
        if (threadIdx.x == 0) sm_tile = atomicAdd(&ctrl[RC_TICKET], 1u);
        __syncthreads();
        const u32 tile = sm_tile;
        u32 row0, cnt;
        if (!res_tile_lookup(b, tile, row0, cnt)) break;
        // thread i owns rows row0 + 4 i .. + 3 (batch order is preserved by ranking thread-major)
        const u32 first_row = row0 + threadIdx.x * RES_ROWS;
        u32 slot[RES_ROWS];
        bool residue[RES_ROWS];
#pragma unroll
        for (int k = 0; k < RES_ROWS; k++) {
            slot[k] = (threadIdx.x * RES_ROWS + k < cnt) ? slot_arr[first_row + k] : t.null_slot;
            residue[k] = false;
        }
        // what pass B found out about each row: F_SHARED / F_DEFER (+ its verdict)
        u32 bits[RES_ROWS];
        if (threadIdx.x * RES_ROWS + RES_ROWS <= cnt) {
            const u32 f4 = *reinterpret_cast<const u32 *>(flags + first_row);
#pragma unroll
            for (int k = 0; k < RES_ROWS; k++) bits[k] = slot[k] != t.null_slot ? ((f4 >> (8 * k)) & 0xFF) : 0;
        } else {
#pragma unroll
            for (int k = 0; k < RES_ROWS; k++) bits[k] = slot[k] != t.null_slot ? flags[first_row + k] : 0;
        }
        u64 mk[RES_ROWS];
#pragma unroll
        for (int k = 0; k < RES_ROWS; k++) {
            const bool look = (bits[k] & F_SHARED) && !(bits[k] & F_DEFER);
            mk[k] = look ? t.mark[slot[k]] : ~0ULL;
        }
        u32 mine = 0;
#pragma unroll
        for (int k = 0; k < RES_ROWS; k++) {
            if (slot[k] == t.null_slot) continue;
            const u32 row = first_row + k;
            if (bits[k] & F_DEFER) {
                residue[k] = true;                                   // deferred by pass B
            } else if (bits[k] & F_SHARED) {
                const bool has = (u32)(mk[k] >> 32) == ~epoch;
                const u32 first = (u32)mk[k];
                if (has && row > first) {
                    residue[k] = true;
                } else {
                    const u32 f = bits[k];
                    n_allowed += (f & F_ALLOWED) ? 1 : 0;
                    n_denied += (f & F_ALLOWED) ? 0 : 1;
                    exp_hits += (f & F_EXP_HIT) ? 1 : 0;
                    if (has && row == first) {
                        // the first state change of the key in this batch: redo its decision and commit
                        u64 key_hash;
                        Req r;
                        parse_request<Row::COMPACT>(b.req_at(row, Row::REQ_BYTES), pol, npol, now_batch, key_hash, r);
                        RunState s;
                        load_state(t, slot[k], s);
                        const Decision d = decide(s.tat, s.exp, r);
                        const bool created = !has_state(s.exp);
                        RunState ns = {d.new_tat, d.new_exp, r.ei};
                        store_state(t, slot[k], ns, created);
                        real_inc += created ? 1 : 0;
                    }
                }
            }
            mine += residue[k] ? 1 : 0;
        }
        // stable compaction of the residue rows: rank inside the tile + decoupled look-back for the tile base
        u32 total;
        u32 rank = block_exclusive_scan(mine, part, &total);
        if (warp == 0) {
            const u32 base = lookback(tile_status, tile, total, lane);
            if (lane == 0) {
                sm_base = base;
                u32 r0, c0;
                if (!res_tile_lookup(b, tile + 1, r0, c0)) {                // last tile: residue size
                    ctrl[RC_NRES] = min(base + total, res_cap);
                    *host_nres = min(base + total, res_cap);                // mapped pinned host memory: feedback for the host
                }
            }
        }
        __syncthreads();
        const u32 base = sm_base;
#pragma unroll
        for (int k = 0; k < RES_ROWS; k++) {
            if (!residue[k]) continue;
            const u32 row = first_row + k;
            const u32 p = base + rank++;
            if (p >= res_cap) {
                // more residue than the engine's batch capacity (a multi-GPU tick far beyond max_batch): the row
                // is answered with an internal error instead of overrunning the sort buffers
                if (Row::R16) write_result16(b.res16_at(row), 0, GCRA_INTERNAL, 0);
                else write_result(b.res_at(row), 0, 0, 0, GCRA_INTERNAL, 0);
                atomicAdd(&t.counters[C_ERRORS], 1ULL);
                continue;
            }
            res_keys[p] = ((u64)slot[k] << 32) | row;     // the tail parses the request of row `row` itself
            // the next batch must keep off this key until this batch's tail is through with it
            const u32 e = slot[k] & bm_mask;
            if (!((next_pend[e >> 5] >> (e & 31)) & 1)) atomicOr(next_pend + (e >> 5), 1u << (e & 31));   // (a stale L1 line shows a subset; result unused: RED)
        }
        __syncthreads();   // sm_tile / sm_base / part are reused by the next tile
    }
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

}  // namespace gcra
