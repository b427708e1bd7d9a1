// gcra_p2p.cuh -- multi-GPU routing over NVLink peer memory (one process per GPU, key space hash-sharded).
//
// The reference is single-process and recommends "client-side sharding by key" (README.md:247-249); inside a tick
// requests are applied in GLOBAL index order, rank r's slice before rank r+1's (actor.rs:217-236 applied to the
// union stream).  Every rank owns one WINDOW of device memory that all peers map (CUDA IPC):
//
//   header   req_tick[r]   newest tick whose rows from sender r are complete in my inbox          (written by r)
//            res_tick[p]   newest tick whose results from owner p are complete in my outbox        (written by p)
//            counts[d][r]  rows sender r put into inbox slot d                                     (written by r)
//   inbox    [DEPTH][world][cap] gcra_request   segment (d, r): the rows sender r routed to me, in r's order
//   outbox   [DEPTH][world][cap] gcra_result    segment (d, p): results of the rows I routed to owner p
//
// A tick on the sender: stable partition by owner (count -> scan -> scatter); the scatter kernel STORES every row
// straight into its owner's inbox over NVLink -- partition and transfer are one kernel, there is no pack buffer,
// no count exchange and no host synchronisation -- then one thread per peer publishes the count and, after a
// system-scope fence, the tick number.  On the owner a one-warp kernel waits for the tick number of every sender;
// the engine then runs its index-order pipeline over the inbox slot as ONE batch of `world` segments whose row
// counts it reads from the header, and its kernels store every result straight into the sender's outbox (a
// segment's result pointer is peer-mapped); a last kernel publishes res_tick.  Back on the sender a one-warp
// kernel waits for every owner's res_tick and the un-permutation kernel moves the results into the caller's
// buffer in input order.  Slot d of tick t is reused by tick t + DEPTH; a sender only routes tick t + DEPTH after
// it has un-permuted tick t, i.e. after every owner published res_tick >= t -- which the owner does after its last
// read of inbox slot d and its last write to my outbox slot d -- so one flag orders both reuses.
// A ring tick (gcra_resp_ring_submit_route) knows its row count only on the device: the *_dev_kernel variants read it
// there and size their grids from the host's bound of it.
#pragma once
#include "gcra_index_path.cuh"

namespace gcra {

constexpr int P2P_DEPTH = 4;
constexpr int P2P_MAX_WORLD = MAX_SEGS;

struct P2PHeader {
    u64 req_tick[P2P_MAX_WORLD];
    u64 res_tick[P2P_MAX_WORLD];
    u32 counts[P2P_DEPTH][P2P_MAX_WORLD];
    u32 error;                       // a wait gave up (a peer never arrived): results of that tick are garbage
    u32 pad0;
    u64 seed[2];                     // the rank's key-hash seed (gcra_p2p_prepare): gcra_ring_p2p checks every rank's
    u32 pad[26];
};

// what a rank knows about everybody's window (device memory; index = rank)
struct P2PPeers {
    P2PHeader *hdr[P2P_MAX_WORLD];
    unsigned char *inbox[P2P_MAX_WORLD];
    unsigned char *outbox[P2P_MAX_WORLD];
};

__device__ __forceinline__ void st_release_sys(u64 *p, u64 v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ u64 ld_acquire_sys(const u64 *p) {
    u64 v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// one CTA per owner: exclusive scan of that owner's per-tile counts; the total is the owner's row count
__global__ void __launch_bounds__(TILE_THREADS)
p2p_scan_kernel(u32 *__restrict__ tile_counts, u32 num_tiles, u32 *__restrict__ counts) {
    __shared__ u32 part[TILE_THREADS / 32];
    u32 *row = tile_counts + (size_t)blockIdx.x * num_tiles;
    const u32 per = (num_tiles + TILE_THREADS - 1) / TILE_THREADS;
    const u32 lo = min(threadIdx.x * per, num_tiles), hi = min(lo + per, num_tiles);
    u32 s = 0;
    for (u32 i = lo; i < hi; i++) s += row[i];
    u32 total;
    u32 acc = block_exclusive_scan(s, part, &total);
    for (u32 i = lo; i < hi; i++) { u32 v = row[i]; row[i] = acc; acc += v; }
    if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// stable partition + transfer: row i goes to position (offset of its tile for its owner + rank among the tile's
// earlier rows of that owner) of segment (slot, me) in the OWNER's inbox; res_loc[i] remembers where its result
// will arrive in my outbox.  The tile's rows are first grouped by owner in shared memory, then written out as
// contiguous 16-byte pieces -- a warp's store covers 512 consecutive bytes of one inbox, which is what NVLink wants
// (a lane storing the three pieces of its own row would send 16-byte packets).
__device__ __forceinline__ void p2p_scatter_tile(const gcra_request *__restrict__ req, u32 n, u32 world, u32 me,
                                                 u32 slot, u32 cap_shift, u32 num_tiles,
                                                 const u32 *__restrict__ tile_offsets,
                                                 const P2PPeers *__restrict__ peers, u32 *__restrict__ res_loc) {
    constexpr int NW = TILE_THREADS / 32;
    __shared__ u32 wc[NW][ROUTE_MAX_SHARDS];
    __shared__ u32 lbase[ROUTE_MAX_SHARDS + 1];              // first tile-local position of every owner's rows
    __shared__ unsigned long long dst_base[ROUTE_MAX_SHARDS]; // where the tile's rows of owner o start in o's inbox
    __shared__ __align__(16) ulonglong2 rows[TILE_THREADS * 3];
    __shared__ unsigned char own_of[TILE_THREADS];           // owner of the row at a tile-local position
    const u32 w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x < NW * ROUTE_MAX_SHARDS) (&wc[0][0])[threadIdx.x] = 0;
    __syncthreads();
    const u32 i = blockIdx.x * TILE_THREADS + threadIdx.x;
    const u32 cnt = min((u32)TILE_THREADS, n - blockIdx.x * TILE_THREADS);
    const bool valid = i < n;
    ulonglong2 r0 = make_ulonglong2(0, 0), r1 = r0, r2 = r0;
    u32 own = 0;
    if (valid) {
        const ulonglong2 *s = reinterpret_cast<const ulonglong2 *>(req + i);
        r0 = s[0]; r1 = s[1]; r2 = s[2];
        own = owner_of(r0.x, world);
    }
    const u32 peers_m = __match_any_sync(0xffffffffu, valid ? own : (0x80000000u | lane));
    const u32 rank = __popc(peers_m & ((1u << lane) - 1));
    if (valid && rank == 0) wc[w][own] = __popc(peers_m);
    __syncthreads();
    if (threadIdx.x < world) {
        u32 acc = 0;
        for (int x = 0; x < NW; x++) { u32 v = wc[x][threadIdx.x]; wc[x][threadIdx.x] = acc; acc += v; }
        lbase[threadIdx.x + 1] = acc;                        // the owner's count in this tile (scanned below)
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 acc = 0;
        lbase[0] = 0;
        for (u32 o = 0; o < world; o++) { const u32 c = lbase[o + 1]; lbase[o + 1] = acc + c; acc += c; }
    }
    if (threadIdx.x < world) {
        const u32 o = threadIdx.x;
        const size_t seg = ((size_t)slot * world + me) << cap_shift;
        const unsigned char *base = (const unsigned char *)__ldg((const u64 *)&peers->inbox[o]);
        dst_base[o] = (unsigned long long)(base + (seg + tile_offsets[o * num_tiles + blockIdx.x]) * sizeof(gcra_request));
    }
    __syncthreads();
    if (valid) {
        const u32 in_owner = wc[w][own] + rank;              // rank among the tile's rows of this owner
        const u32 lpos = lbase[own] + in_owner;
        rows[lpos * 3] = r0; rows[lpos * 3 + 1] = r1; rows[lpos * 3 + 2] = r2;
        own_of[lpos] = (unsigned char)own;
        res_loc[i] = (own << cap_shift) | (tile_offsets[own * num_tiles + blockIdx.x] + in_owner);
    }
    __syncthreads();
    for (u32 c = threadIdx.x; c < cnt * 3; c += TILE_THREADS) {
        const u32 lpos = c / 3, o = own_of[lpos];
        ulonglong2 *d = reinterpret_cast<ulonglong2 *>(dst_base[o]) + (c - lbase[o] * 3);
        *d = rows[c];                                        // NVLink store (local when o == me)
    }
}

__global__ void __launch_bounds__(TILE_THREADS)
p2p_scatter_kernel(const gcra_request *__restrict__ req, u32 n, u32 world, u32 me, u32 slot, u32 cap_shift,
                   u32 num_tiles, const u32 *__restrict__ tile_offsets, const P2PPeers *__restrict__ peers,
                   u32 *__restrict__ res_loc) {
    p2p_scatter_tile(req, n, world, me, slot, cap_shift, num_tiles, tile_offsets, peers, res_loc);
}

// the row count on the device (a ring slot's parsed rows, gcra_resp_ring_submit_route): min(*dev_n, n_bound) rows
// over a grid sized from n_bound; a tile past the count stores nothing (route_count_dev_kernel counted it as empty)
__global__ void __launch_bounds__(TILE_THREADS)
p2p_scatter_dev_kernel(const gcra_request *__restrict__ req, u32 n_bound, const u32 *__restrict__ dev_n, u32 world,
                       u32 me, u32 slot, u32 cap_shift, u32 num_tiles, const u32 *__restrict__ tile_offsets,
                       const P2PPeers *__restrict__ peers, u32 *__restrict__ res_loc) {
    const u32 n = min(*dev_n, n_bound);
    if (blockIdx.x * TILE_THREADS >= n) return;
    p2p_scatter_tile(req, n, world, me, slot, cap_shift, num_tiles, tile_offsets, peers, res_loc);
}

// after the scatter kernel: lane p tells owner p how many rows it got and that tick `tick` is complete
__global__ void p2p_signal_req_kernel(const P2PPeers *__restrict__ peers, const u32 *__restrict__ counts, u32 world,
                                      u32 me, u32 slot, u64 tick) {
    const u32 p = threadIdx.x;
    if (p >= world) return;
    P2PHeader *h = (P2PHeader *)__ldg((const u64 *)&peers->hdr[p]);
    *reinterpret_cast<volatile u32 *>(&h->counts[slot][me]) = counts[p];
    __threadfence_system();
    st_release_sys(&h->req_tick[me], tick);
}

// after the last kernel of the tick on the owner: every sender may read its results and reuse my inbox slot
__global__ void p2p_signal_res_kernel(const P2PPeers *__restrict__ peers, u32 world, u32 me, u64 tick) {
    const u32 r = threadIdx.x;
    if (r >= world) return;
    P2PHeader *h = (P2PHeader *)__ldg((const u64 *)&peers->hdr[r]);
    __threadfence_system();
    st_release_sys(&h->res_tick[me], tick);
}

// one warp: lane r waits until flags[r] >= tick (flags = req_tick or res_tick of MY header).  A peer that never
// arrives must not hang the GPU: after ~20 s the wait gives up and raises the header's error flag.
__global__ void p2p_wait_kernel(P2PHeader *__restrict__ hdr, int which, u32 world, u64 tick) {
    const u32 r = threadIdx.x;
    if (r >= world) return;
    const u64 *flag = which == 0 ? &hdr->req_tick[r] : &hdr->res_tick[r];
    const long long t0 = clock64();
    while (ld_acquire_sys(flag) < tick) {
        if (clock64() - t0 > 40000000000LL) { hdr->error = 1; break; }
        __nanosleep(200);
    }
}

// results back into input order: row i's result sits at outbox segment (slot, owner) position pos
__device__ __forceinline__ void p2p_unpermute_row(const unsigned char *__restrict__ outbox,
                                                  const u32 *__restrict__ res_loc, u32 n, u32 world, u32 slot,
                                                  u32 cap_shift, gcra_result *__restrict__ out) {
    const u32 i = blockIdx.x * TILE_THREADS + threadIdx.x;
    if (i >= n) return;
    const u32 loc = res_loc[i];
    const u32 own = loc >> cap_shift, pos = loc & ((1u << cap_shift) - 1);
    const size_t seg = ((size_t)slot * world + own) << cap_shift;
    const ulonglong2 *s = reinterpret_cast<const ulonglong2 *>(outbox + (seg + pos) * sizeof(gcra_result));
    ulonglong2 *d = reinterpret_cast<ulonglong2 *>(out + i);
    d[0] = s[0]; d[1] = s[1];
}

__global__ void __launch_bounds__(TILE_THREADS)
p2p_unpermute_kernel(const unsigned char *__restrict__ outbox, const u32 *__restrict__ res_loc, u32 n, u32 world,
                     u32 slot, u32 cap_shift, gcra_result *__restrict__ out) {
    p2p_unpermute_row(outbox, res_loc, n, world, slot, cap_shift, out);
}

// the row count on the device: rows past min(*dev_n, n_bound) are not un-permuted
__global__ void __launch_bounds__(TILE_THREADS)
p2p_unpermute_dev_kernel(const unsigned char *__restrict__ outbox, const u32 *__restrict__ res_loc, u32 n_bound,
                         const u32 *__restrict__ dev_n, u32 world, u32 slot, u32 cap_shift,
                         gcra_result *__restrict__ out) {
    p2p_unpermute_row(outbox, res_loc, min(*dev_n, n_bound), world, slot, cap_shift, out);
}

}  // namespace gcra
