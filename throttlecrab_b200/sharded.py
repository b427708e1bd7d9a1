"""Hash-sharded multi-GPU engine: one process per GPU, key space partitioned by owner shard.

The reference is single-process; its docs recommend "client-side sharding by key"
(README.md:247-249).  Here every rank ingests an arbitrary slice of a tick, a stable partition
kernel (gcra_route_partition) groups the slice by owner, one all-to-all moves each group to its
owning GPU, the owner decides locally (gcra_rate_limit_batch_device), a second all-to-all returns the
results and gcra_route_unpermute puts them back in input order.

Ordering rule: inside a tick, requests are applied in GLOBAL index order, where rank r's slice
precedes rank r+1's.  The stable partition keeps slice order inside every group and all-to-all
concatenates the groups in source-rank order, so the owner sees each key's requests in that order.
Ticks are decided strictly in submission order on one stream.

Pipelining: `submit()` only enqueues.  A tick has three stages on three streams, ordered by events:
route (partition, count exchange, request all-to-all), decide (the engine's kernels) and return
(result all-to-all, un-permutation).  Each stage's collectives use their own communicator so that
NCCL does not serialise the stages of neighbouring ticks; tick i+1 is routed while tick i is decided
and tick i-1's results travel back.  `DEPTH` buffer sets are cycled; `finish()` drains.
`step()` = submit + finish (blocking).

torch is plumbing only: device buffers, the NCCL process group and stream/event ordering.
"""
import os

import numpy as np
import torch

REQ_B, RES_B = 48, 32
DEPTH = 4


class _Snapshots:
    """Snapshots of a sharded key space.  Every rank submits every tick, so ranks that each save after joining the
    same tick together hold one consistent cut; any number of ranks can take it up again, whatever the world size
    that wrote it (gcra_snapshot_restore keeps the entries each rank owns)."""

    def save(self, directory):
        """Wait for every tick submitted so far, then write this rank's table to <directory>/rank<r>.gcra."""
        self.finish()
        path = os.path.join(directory, "rank%d.gcra" % self.rank)
        self.lim.store.save(path)          # gcra_snapshot_save waits for the device
        return path

    def save_begin(self, directory):
        """Begin a background save of this rank's table to <directory>/rank<r>.gcra without joining any tick: the cut
        is this call's place among the ticks submitted here.  Ranks that each call it after submitting the same tick
        take one consistent cut, and ticks continue meanwhile.  save_wait() waits for the file."""
        path = os.path.join(directory, "rank%d.gcra" % self.rank)
        self.lim.store.save_begin(path)
        return path

    def save_wait(self):
        """Wait for this rank's background save; returns the number of entries written."""
        return self.lim.store.save_wait()

    def restore(self, paths):
        """Insert this rank's share of every snapshot file in `paths` (all files of a save(), any world size), next to
        what the engine holds.  Call it between ticks, on every rank.  Returns (restored, conflicts) over the files."""
        self.finish()
        restored = conflicts = 0
        for p in paths:
            r, c = self.lim.store.restore(p, self.rank, self.world)
            restored, conflicts = restored + r, conflicts + c
        return restored, conflicts


def merge_top_denied(lists, k):
    """The global top k of the ranks' top-denied lists ([(key_hash, count)] each, as RateLimiter.store.top_denied
    returns them).  Every pipeline counts a denied request on the engine that owns its key, so the lists hold
    disjoint keys and the global top k is the top k of their concatenation; the order is gcra_top_denied's: count
    descending, then hash ascending.  A key in more than one list means the lists are not of one sharded key space."""
    merged = [(int(h), int(c)) for lst in lists for h, c in lst]
    if len({h for h, _ in merged}) != len(merged):
        raise ValueError("merge_top_denied: a key appears in more than one list")
    merged.sort(key=lambda hc: (-hc[1], hc[0]))
    return merged[:k]


class _DeniedKeys:
    """Top denied keys of a sharded key space (gcra_track_denied / gcra_top_denied on every rank's engine)."""

    def track_denied(self, max_keys):
        """Count denied requests per key on this rank's engine (0 = off); max_keys is per rank.  Call it between
        ticks: only later ticks are counted."""
        self.finish()
        self.lim.store.track_denied(max_keys)

    def top_denied(self, k):
        """Collective: every rank calls it between ticks, after the same tick.  Waits for every tick submitted here,
        all-gathers each rank's top k and its dropped count, and returns on every rank the global top k
        (merge_top_denied) and the sum of the ranks' dropped counts.  Each rank's own query prunes its table by the
        per-rank rule of gcra_top_denied."""
        self.finish()
        mine, dropped = self.lim.store.top_denied(k)
        buf = np.zeros((k + 1, 2), np.uint64)
        buf[0] = (len(mine), dropped)
        if mine:
            buf[1:len(mine) + 1] = np.array(mine, np.uint64)
        t = torch.from_numpy(buf.view(np.int64)).to(self.dev)
        every = [torch.empty_like(t) for _ in range(self.world)]
        self.dist.all_gather(every, t)
        lists, total = [], 0
        for e in every:
            a = e.cpu().numpy().view(np.uint64)
            n = int(a[0, 0])
            total += int(a[0, 1])
            lists.append([(int(h), int(c)) for h, c in a[1:n + 1]])
        return merge_top_denied(lists, k), total


class CudaOps:
    """The three device steps, all through the C ABI."""

    def __init__(self, limiter):
        self.lim = limiter
        self.L, self.h = limiter._L, limiter._h

    def _check(self, rc):
        self.lim.store._check(rc)

    def partition(self, n, req, world, routed, src_index, counts, stream):
        self._check(self.L.gcra_route_partition(self.h, n, req.data_ptr(), world, routed.data_ptr(),
                                                src_index.data_ptr(), counts.data_ptr(), stream))

    def decide(self, n, req, res, stream):
        self._check(self.L.gcra_rate_limit_batch_device(self.h, n, req.data_ptr(), res.data_ptr(), stream))

    def unpermute(self, n, routed_res, src_index, res, stream):
        self._check(self.L.gcra_route_unpermute(self.h, n, routed_res.data_ptr(), src_index.data_ptr(),
                                                res.data_ptr(), stream))


class _Slot:
    def __init__(self, max_rows, device, world=1):
        u8 = dict(dtype=torch.uint8, device=device)
        self.routed = torch.empty(max_rows * REQ_B, **u8)
        # a shard can receive every rank's whole tick: sized for that, no rank ever bails out of a tick alone
        self.recv_req = torch.empty(world * max_rows * REQ_B, **u8)
        self.recv_res = torch.empty(world * max_rows * RES_B, **u8)
        self.back_res = torch.empty(max_rows * RES_B, **u8)
        self.src_index = torch.empty(max_rows, dtype=torch.int32, device=device)
        self.counts = torch.zeros(16, dtype=torch.int32, device=device)
        self.recv_counts = torch.zeros(16, dtype=torch.int32, device=device)
        self.both_host = torch.empty(32, dtype=torch.int32, pin_memory=(device.type == "cuda"))
        self.routed_ev = None      # request all-to-all finished
        self.decided_ev = None     # engine kernels finished
        self.done_ev = None        # results un-permuted into the caller's buffer


class ShardedLimiter(_Snapshots, _DeniedKeys):
    def __init__(self, limiter, dist, device, ops=None, max_rows=None):
        self.lim, self.dist, self.dev = limiter, dist, device
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.ops = ops if ops is not None else CudaOps(limiter)
        self.max_rows = max_rows or limiter.store.max_batch
        self.cuda = device.type == "cuda"
        self.slots = [_Slot(self.max_rows, device, self.world) for _ in range(DEPTH if self.cuda else 1)]
        self.n_submitted = 0
        self.pending = None
        self.returned = []
        self.last_recv_rows = 0
        # one communicator per stage (NCCL executes the collectives of ONE communicator in issue order)
        self.pg_counts = dist.new_group()
        self.pg_req = dist.new_group()
        self.pg_res = dist.new_group()
        if self.cuda:
            self.s_route = torch.cuda.Stream(device)
            self.s_decide = torch.cuda.Stream(device)
            self.s_return = torch.cuda.Stream(device)

    # ------------------------------------------------------------------ the stages of a tick
    def _route_a(self, slot, d_req, n, stream):
        """partition + count exchange (asynchronous)"""
        W = self.world
        self.ops.partition(n, d_req, W, slot.routed, slot.src_index, slot.counts, stream)
        self.dist.all_to_all_single(slot.recv_counts[:W], slot.counts[:W], group=self.pg_counts)
        slot.both = torch.cat([slot.counts[:W], slot.recv_counts[:W]])
        if self.cuda:
            slot.both_host[:2 * W].copy_(slot.both, non_blocking=True)
            slot.counts_ev = torch.cuda.Event()
            slot.counts_ev.record()

    def _route_b(self, slot, n):
        """read the counts on the host (the only host sync of a tick), then the request all-to-all"""
        W = self.world
        if self.cuda:
            slot.counts_ev.synchronize()
            both = slot.both_host[:2 * W].tolist()
        else:
            both = slot.both.tolist()
        send_l, recv_l = both[:W], both[W:]
        n_recv = sum(recv_l)          # <= world * max_rows, which the buffers hold
        self.dist.all_to_all_single(slot.recv_req[:n_recv * REQ_B], slot.routed[:n * REQ_B],
                                    output_split_sizes=[c * REQ_B for c in recv_l],
                                    input_split_sizes=[c * REQ_B for c in send_l], group=self.pg_req)
        return send_l, recv_l, n_recv

    def _decide(self, slot, n_recv, stream):
        # more rows than one engine batch carries: several batches, cut anywhere (the order is kept)
        for a in range(0, max(n_recv, 1), self.max_rows):
            m = min(n_recv - a, self.max_rows)
            self.ops.decide(m, slot.recv_req[a * REQ_B:], slot.recv_res[a * RES_B:], stream)

    def _return(self, slot, d_res, n, send_l, recv_l, n_recv, stream):
        self.dist.all_to_all_single(slot.back_res[:n * RES_B], slot.recv_res[:n_recv * RES_B],
                                    output_split_sizes=[c * RES_B for c in send_l],
                                    input_split_sizes=[c * RES_B for c in recv_l], group=self.pg_res)
        self.ops.unpermute(n, slot.back_res, slot.src_index, d_res, stream)

    def _issue_decide_return(self):
        if self.pending is None:
            return
        slot, d_res, n, send_l, recv_l, n_recv = self.pending
        self.pending = None
        with torch.cuda.stream(self.s_decide):
            self.s_decide.wait_event(slot.routed_ev)
            self._decide(slot, n_recv, self.s_decide.cuda_stream)
            slot.decided_ev = torch.cuda.Event()
            slot.decided_ev.record(self.s_decide)
        with torch.cuda.stream(self.s_return):
            self.s_return.wait_event(slot.decided_ev)
            self._return(slot, d_res, n, send_l, recv_l, n_recv, self.s_return.cuda_stream)
            slot.done_ev = torch.cuda.Event()
            slot.done_ev.record(self.s_return)
        self.returned.append(slot.done_ev)

    def pop_returned(self):
        """Events of the ticks whose results are (or will be) in their d_res buffers, oldest first;
        lets a caller chain per-tick device->host copies without waiting for finish()."""
        out, self.returned = self.returned, []
        return out

    # ------------------------------------------------------------------ public
    def submit(self, d_req, d_res):
        """Enqueue one tick.  d_req: uint8 tensor of n*48 bytes (gcra_request rows), ready on the
        caller's current stream; d_res: uint8 tensor of n*32 bytes, valid after finish()."""
        n = d_req.numel() // REQ_B
        slot = self.slots[self.n_submitted % len(self.slots)]
        self.n_submitted += 1
        if not self.cuda:
            self._route_a(slot, d_req, n, None)
            send_l, recv_l, n_recv = self._route_b(slot, n)
            self._decide(slot, n_recv, None)
            self._return(slot, d_res, n, send_l, recv_l, n_recv, None)
            self.last_recv_rows = n_recv
            return n_recv
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(self.s_route):
            self.s_route.wait_event(ready)
            if slot.done_ev is not None:
                self.s_route.wait_event(slot.done_ev)            # the slot's buffers are free again
            self._route_a(slot, d_req, n, self.s_route.cuda_stream)
        # while the partition + count exchange of THIS tick run, enqueue the previous tick's engine
        # kernels and result return: the count read-back below then finds its data ready
        self._issue_decide_return()
        with torch.cuda.stream(self.s_route):
            send_l, recv_l, n_recv = self._route_b(slot, n)
            slot.routed_ev = torch.cuda.Event()
            slot.routed_ev.record(self.s_route)
        self.pending = (slot, d_res, n, send_l, recv_l, n_recv)
        self.last_recv_rows = n_recv
        return n_recv

    def finish(self):
        """Issue what is still pending and make the caller's current stream wait for every tick."""
        if self.cuda:
            self._issue_decide_return()
            cur = torch.cuda.current_stream(self.dev)
            for st in (self.s_route, self.s_decide, self.s_return):
                cur.wait_stream(st)

    def step(self, d_req, d_res):
        n_recv = self.submit(d_req, d_res)
        self.finish()
        return n_recv


class NativeShardedLimiter(_Snapshots, _DeniedKeys):
    """The same pipeline driven by ONE C call per tick (gcra_shard_submit): partition, NCCL count exchange and
    all-to-alls (libnccl resolved with dlopen inside the library), the engine's pipelined kernels and the way
    back all live in libgcra_b200.so.  torch.distributed is used once, to hand the three ncclUniqueIds that
    rank 0 creates to the other ranks."""

    def __init__(self, limiter, dist, device, max_rows=None):
        import ctypes as C
        self.lim, self.dist, self.dev = limiter, dist, device
        self.L, self.h = limiter._L, limiter._h
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.max_rows = max_rows or limiter.store.max_batch
        ids = torch.zeros(384, dtype=torch.uint8)
        if self.rank == 0:
            buf = (C.c_char * 384)()
            if self.L.gcra_shard_unique_ids(C.addressof(buf)) != 0:
                raise RuntimeError("ncclGetUniqueId failed (libnccl.so.2 not loadable)")
            ids = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
        ids = ids.to(device)
        dist.broadcast(ids, src=0)
        raw = bytes(ids.cpu().numpy().tobytes())
        limiter.store._check(self.L.gcra_shard_init(self.h, self.rank, self.world, raw, self.max_rows))
        self.n_submitted = 0

    def submit(self, d_req, d_res, ready_stream=None):
        n = d_req.numel() // REQ_B
        st = ready_stream if ready_stream is not None else torch.cuda.current_stream(self.dev).cuda_stream
        self.lim.store._check(self.L.gcra_shard_submit(self.h, n, d_req.data_ptr(), d_res.data_ptr(), st))
        self.n_submitted += 1

    def wait_tick(self, ticks_back, stream):
        """make `stream` (a torch stream) wait for the results of an earlier tick (0 = latest)"""
        self.lim.store._check(self.L.gcra_shard_wait_tick(self.h, ticks_back, stream.cuda_stream))

    def finish(self):
        self.lim.store._check(self.L.gcra_shard_join(self.h, torch.cuda.current_stream(self.dev).cuda_stream))

    def step(self, d_req, d_res):
        self.submit(d_req, d_res)
        self.finish()

    def describe(self):
        return "native NCCL pipeline (gcra_shard_submit: partition, count exchange, all-to-all, decide, all-to-all)"


class PeerShardedLimiter(_Snapshots, _DeniedKeys):
    """The sharded tick over NVLink peer memory (gcra_p2p_*, csrc/gcra_p2p.cuh): the partition kernel stores every
    request row straight into its owner's inbox, the owner's engine runs over the inbox as one batch of `world`
    segments and stores every result straight into the sender's outbox; ranks synchronise with tick numbers in peer
    memory.  No NCCL in the data path, no host synchronisation.  torch.distributed is used once, to all-gather the
    64-byte CUDA IPC handles of the ranks' windows."""

    def __init__(self, limiter, dist, device, max_rows=None):
        import ctypes as C
        self.lim, self.dist, self.dev = limiter, dist, device
        self.L, self.h = limiter._L, limiter._h
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.cap = max_rows or limiter.store.max_batch
        buf = (C.c_char * 64)()
        win = C.c_void_p()
        limiter.store._check(self.L.gcra_p2p_prepare(self.h, self.rank, self.world, self.cap, C.addressof(buf), C.byref(win)))
        mine = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone().to(device)
        allh = [torch.zeros(64, dtype=torch.uint8, device=device) for _ in range(self.world)]
        dist.all_gather(allh, mine)
        raw = b"".join(bytes(t.cpu().numpy().tobytes()) for t in allh)
        limiter.store._check(self.L.gcra_p2p_connect(self.h, raw, None))
        dist.barrier()                       # every window is mapped everywhere before the first row is stored
        self.n_submitted = 0

    def submit(self, d_req, d_res, ready_stream=None):
        n = d_req.numel() // REQ_B
        st = ready_stream if ready_stream is not None else torch.cuda.current_stream(self.dev).cuda_stream
        self.lim.store._check(self.L.gcra_p2p_submit(self.h, n, d_req.data_ptr(), d_res.data_ptr(), st))
        self.n_submitted += 1

    def wait_tick(self, ticks_back, stream):
        self.lim.store._check(self.L.gcra_p2p_wait_tick(self.h, ticks_back, stream.cuda_stream))

    def finish(self):
        self.lim.store._check(self.L.gcra_p2p_join(self.h, torch.cuda.current_stream(self.dev).cuda_stream))

    def step(self, d_req, d_res):
        self.submit(d_req, d_res)
        self.finish()

    def error(self):
        import ctypes as C
        e = C.c_uint32()
        self.lim.store._check(self.L.gcra_p2p_error(self.h, C.byref(e)))
        return int(e.value)

    def describe(self):
        return ("NVLink peer memory (gcra_p2p_submit: partition kernel stores rows into the owners' inboxes, owners store "
                "results into the senders' outboxes, flags in peer memory; no NCCL, no host sync)")


def connect_local(limiters, cap_rows):
    """Engines that live in ONE process (the single-GPU loop-back test): windows are exchanged as plain pointers."""
    import ctypes as C
    world = len(limiters)
    wins = (C.c_void_p * world)()
    for r, lim in enumerate(limiters):
        w = C.c_void_p()
        lim.store._check(lim._L.gcra_p2p_prepare(lim._h, r, world, cap_rows, None, C.byref(w)))
        wins[r] = w.value
    for lim in limiters:
        lim.store._check(lim._L.gcra_p2p_connect(lim._h, None, wins))


def make_sharded(limiter, dist, device, max_rows=None):
    """The sharded pipeline bench.py and the tests use: NVLink peer-memory routing (gcra_p2p_*) when the ranks can
    map each other's memory, else the NCCL pipeline.  GCRA_SHARD=nccl / p2p forces one."""
    import os
    want = os.environ.get("GCRA_SHARD", "auto")
    if want != "nccl" and "PeerShardedLimiter" in globals():
        try:
            return PeerShardedLimiter(limiter, dist, device, max_rows)
        except Exception:
            if want == "p2p":
                raise
    return NativeShardedLimiter(limiter, dist, device, max_rows)
