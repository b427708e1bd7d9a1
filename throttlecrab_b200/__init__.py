"""throttlecrab_b200 -- H100-native batched GCRA rate-limit engine (host-side mirror).

Mirrors the part of lazureykis/throttlecrab's library API that sits on the hot path:

    reference (Rust)                                         here
    RateLimiter::new(store)          rate_limiter.rs:56      RateLimiter(store)
    RateLimiter::rate_limit(..)      rate_limiter.rs:102     RateLimiter.rate_limit(..)
    RateLimitResult                  rate_limiter.rs:12-22   RateLimitResult
    CellError                        core/mod.rs:48-56       NegativeQuantity / InvalidRateLimit / Internal
    trait Store                      store/mod.rs:85-133     Store methods of the store classes
    AdaptiveStore / PeriodicStore / ProbabilisticStore (+builders)   same names

All state and all decisions live on the GPU behind the C ABI (include/gcra_b200.h); this
module only marshals arguments.  There is no CPU fallback.
"""
import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

from . import _native
from ._native import (REQ_DTYPE, RES_DTYPE, REQ16_DTYPE, RES16_DTYPE, POLICY_DTYPE, OK, NEGATIVE_QUANTITY,
                      INVALID_RATE_LIMIT, INTERNAL, RESP_CONN_DTYPE, RESP_OUTCOME_DTYPE, RESP_MAX_CONN_BYTES,
                      RESP_REPLY_MAX, HTTP_REPLY_MAX, GRPC_CONN_DTYPE, GRPC_OUTCOME_DTYPE, GRPC_REPLY_MAX,
                      GRPC_MAX_DYN, PROTO_RESP, PROTO_HTTP, PROTO_GRPC, MIXED_CONN_DTYPE, DENIED_NAME_MAX,
                      RING_METRICS_MAX_KEYS, NAME_UNKNOWN, NAME_TOO_LONG)

__all__ = ["RateLimiter", "RateLimitResult", "Rate", "CellError", "NegativeQuantity", "InvalidRateLimit",
           "Internal", "AdaptiveStore", "PeriodicStore", "ProbabilisticStore", "ManualStore",
           "hash_key", "key_ref", "pack_keys", "RespRing", "GrpcRing", "MixedRing", "derive_params", "expand_results16", "REQ_DTYPE", "RES_DTYPE",
           "REQ16_DTYPE", "RES16_DTYPE", "POLICY_DTYPE"]

NS = 1_000_000_000


class CellError(Exception):
    """core/mod.rs:48-56"""


class NegativeQuantity(CellError):
    def __init__(self, quantity):
        super().__init__("negative quantity: %d" % quantity)
        self.quantity = quantity


class InvalidRateLimit(CellError):
    def __init__(self):
        super().__init__("invalid rate limit parameters")


class Internal(CellError):
    pass


@dataclass
class RateLimitResult:
    """rate_limiter.rs:12-22; durations are integer nanoseconds."""
    limit: int
    remaining: int
    reset_after: int
    retry_after: int

    @property
    def reset_after_secs(self):      # throttlecrab-server/src/types.rs:93
        return self.reset_after // NS

    @property
    def retry_after_secs(self):      # types.rs:94
        return self.retry_after // NS


def _kb(key):
    return key.encode("utf-8") if isinstance(key, str) else bytes(key)


def _ns(t):
    """SystemTime -> ns since the epoch: int ns, or anything with .timestamp()."""
    if isinstance(t, (int, np.integer)):
        return int(t)
    if hasattr(t, "timestamp"):
        return int(round(t.timestamp() * 1e6)) * 1000
    raise TypeError("now must be int nanoseconds or a datetime")


def hash_key(key):
    k = _kb(key)
    return int(_native.lib().gcra_hash_key(k, len(k)))


def key_ref(off, length):
    """include/gcra_b200.h: the key reference of the bytes [off, off + length) of a key arena"""
    return (int(length) << 32) | int(off)


def pack_keys(keys):
    """(refs, arena) for a sequence of keys (str or bytes): arena = the keys' bytes back to back (uint8), refs[i] =
    GCRA_KEY_REF(off, len) of keys[i] in it (uint64) -- what the keyed calls take in a row's key_hash field."""
    kb = [_kb(k) for k in keys]
    lens = np.fromiter(map(len, kb), np.uint64, len(kb))
    offs = np.zeros(len(kb), np.uint64)
    if len(kb) > 1:
        np.cumsum(lens[:-1], out=offs[1:])
    if len(kb) and int(offs[-1]) > 0xFFFFFFFF:
        raise ValueError("key references hold 32-bit offsets: the keys exceed 4 GiB")
    return (lens << np.uint64(32)) | offs, np.frombuffer(b"".join(kb), np.uint8)


def hash_key_ids(ids, prefix="k:"):
    """hash_key("<prefix><id>") for an array of integer ids (trace generation)."""
    ids = np.ascontiguousarray(ids, np.uint64)
    out = np.empty(len(ids), np.uint64)
    pb = _kb(prefix)
    _native.lib().gcra_hash_key_ids(pb, len(pb), ids.ctypes.data, len(ids), out.ctypes.data)
    return out


def derive_params(max_burst, count_per_period, period):
    """(status, emission_interval_ns, tolerance_ns) -- rate/mod.rs:164-176, rate_limiter.rs:120-122"""
    ei, dvt = C.c_int64(), C.c_int64()
    st = _native.lib().gcra_derive_params(max_burst, count_per_period, period, C.byref(ei), C.byref(dvt))
    return st, ei.value, dvt.value


def expand_results16(req16, now, policies, res16, out=None):
    """RES_DTYPE results of a compact batch from its RES16_DTYPE results (gcra_expand_results16: host only, no GPU).
    Bit-exact with the 32-byte path when `policies` is the table that was registered when the batch ran; raises
    Internal when an OK row names a policy that table does not have (or an invalid one)."""
    req = np.ascontiguousarray(req16, REQ16_DTYPE)
    res = np.ascontiguousarray(res16, RES16_DTYPE)
    pol = np.ascontiguousarray(policies, POLICY_DTYPE)
    if len(req) != len(res):
        raise ValueError("req16 and res16 differ in length")
    out = np.empty(len(req), RES_DTYPE) if out is None else out
    rc = _native.lib().gcra_expand_results16(len(req), req.ctypes.data, _ns(now), pol.ctypes.data, len(pol),
                                            res.ctypes.data, out.ctypes.data)
    if rc != OK:
        raise Internal("gcra_expand_results16: a row names a policy outside the given table, or an invalid one")
    return out


class Rate:
    """core/rate/mod.rs:35-38: an emission interval (integer nanoseconds here instead of a Duration)."""

    def __init__(self, period_ns):
        self._period = int(period_ns)

    @classmethod
    def new(cls, period_ns):                       # rate/mod.rs:56-58
        return cls(period_ns)

    @classmethod
    def per_second(cls, n):                        # :74-78  Duration::from_secs(1) / n as u32
        return cls(NS // _u32(n))

    @classmethod
    def per_minute(cls, n):                        # :94-98
        return cls(60 * NS // _u32(n))

    @classmethod
    def per_hour(cls, n):                          # :114-118
        return cls(3600 * NS // _u32(n))

    @classmethod
    def per_day(cls, n):                           # :134-138
        return cls(86400 * NS // _u32(n))

    @classmethod
    def from_count_and_period(cls, count, period_seconds):   # :164-176
        if count <= 0 or period_seconds <= 0:
            return cls((2**64 - 1) * NS)           # Duration::from_secs(u64::MAX): "a very slow rate"
        st, ei, _ = derive_params(1, count, period_seconds)
        return cls(ei & (2**64 - 1))

    def period(self):                              # :191-193
        return self._period


def _u32(n):
    n = int(n) & 0xFFFFFFFF                        # `n as u32`; Duration / 0 panics in the reference
    if n == 0:
        raise ZeroDivisionError("divide by zero error when dividing duration by scalar")
    return n


class _GpuStore:
    """A GPU-resident key -> (tat, expiry) table standing in for one reference store."""
    KIND = _native.STORE_ADAPTIVE

    def __init__(self, capacity=1000, device=0, created_ns=None, p0=0, p1=0, p2=0, max_batch=0, flags=0, hash_seed=(0, 0)):
        import time
        L = _native.lib()
        cfg = _native.Config(capacity=capacity, device=device, store_kind=self.KIND, p0=p0, p1=p1,
                             p2=p2, created_ns=time.time_ns() if created_ns is None else created_ns,
                             max_batch=max_batch, flags=flags, hash_seed=(C.c_uint64 * 2)(*hash_seed))
        h = C.c_void_p()
        if L.gcra_create(C.byref(cfg), C.byref(h)) != OK or not h:
            raise RuntimeError("gcra_create failed: the CUDA engine is unavailable "
                               "(no device, or libgcra_b200.so not built) -- there is no CPU path")
        self._h = h
        self._L = L
        self.max_batch = max_batch or (1 << 20)

    # -- constructors named like the reference's
    @classmethod
    def new(cls, **kw):
        return cls(**kw)

    @classmethod
    def with_capacity(cls, capacity, **kw):
        return cls(capacity=capacity, **kw)

    def close(self):
        if getattr(self, "_h", None):
            self._L.gcra_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != OK:
            raise Internal(self._L.gcra_last_error(self._h).decode())

    # -- trait Store (core/store/mod.rs:85-133)
    def get(self, key, now):
        k = _kb(key)
        v, f = C.c_int64(), C.c_uint8()
        self._check(self._L.gcra_store_get(self._h, k, len(k), _ns(now), C.byref(v), C.byref(f)))
        return v.value if f.value else None

    def compare_and_swap_with_ttl(self, key, old, new, ttl_ns, now):
        k = _kb(key)
        f = C.c_uint8()
        self._check(self._L.gcra_store_cas(self._h, k, len(k), old, new, ttl_ns, _ns(now), C.byref(f)))
        return bool(f.value)

    def set_if_not_exists_with_ttl(self, key, value, ttl_ns, now):
        k = _kb(key)
        f = C.c_uint8()
        self._check(self._L.gcra_store_set_nx(self._h, k, len(k), value, ttl_ns, _ns(now), C.byref(f)))
        return bool(f.value)

    # -- test helpers of the reference (periodic.rs:113-126) and engine introspection
    def len(self):
        return int(self._L.gcra_len(self._h))

    def is_empty(self):
        return self.len() == 0

    def stats(self):
        s = _native.Stats()
        self._check(self._L.gcra_get_stats(self._h, C.byref(s)))
        return {n: int(getattr(s, n)) for n, _ in s._fields_}

    def sweep(self, now):
        r = C.c_uint64()
        self._check(self._L.gcra_sweep(self._h, _ns(now), C.byref(r)))
        return r.value

    def track_denied(self, max_keys):
        """metrics.rs:162-173: count denied requests per key hash from every finished batch (0 = off)"""
        self._check(self._L.gcra_track_denied(self._h, max_keys))

    def top_denied(self, k):
        """[(key_hash, denied_count)] most denied first, and the number of denials dropped by a full table"""
        keys, cnts = np.zeros(k, np.uint64), np.zeros(k, np.uint64)
        n, dropped = C.c_uint32(), C.c_uint64()
        self._check(self._L.gcra_top_denied(self._h, k, keys.ctypes.data, cnts.ctypes.data, C.byref(n), C.byref(dropped)))
        return [(int(keys[i]), int(cnts[i])) for i in range(n.value)], int(dropped.value)

    def ring_metrics(self, on):
        """gcra_ring_metrics: every later ring submit counts its rows per transport and names its denied keys (on
        zeroes both); off launches nothing more.  Refused while denied tracking runs with more than 10,000 keys."""
        self._check(self._L.gcra_ring_metrics(self._h, 1 if on else 0))

    def ring_transport_counts(self):
        """the ring rows counted so far: uint64 [3, 3], rows RESP, HTTP, gRPC and columns allowed, denied, errors"""
        out = np.zeros((3, 3), np.uint64)
        self._check(self._L.gcra_ring_transport_counts(self._h, out.ctypes.data))
        return out

    def denied_names(self, key_hashes):
        """gcra_denied_names: per hash (from top_denied) its key's bytes as a ring named them, or the marker
        NAME_UNKNOWN or NAME_TOO_LONG (an int)"""
        hs = np.ascontiguousarray(key_hashes, np.uint64)
        names = np.zeros((max(len(hs), 1), DENIED_NAME_MAX), np.uint8)
        lens = np.zeros(max(len(hs), 1), np.uint32)
        self._check(self._L.gcra_denied_names(self._h, len(hs), hs.ctypes.data, names.ctypes.data, lens.ctypes.data))
        return [names[i, :int(lens[i])].tobytes() if lens[i] <= DENIED_NAME_MAX else int(lens[i])
                for i in range(len(hs))]

    def ring_metrics_sharded(self, on, max_keys):
        """gcra_ring_metrics_sharded: ring metrics for rings whose ticks may be peer-memory ticks: every later ring
        submit counts its rows per transport on this engine and names the keys its connections saw denied in a name
        table of this engine (max_keys as track_denied's; 0: no names); the denied counts stay on the keys' owners.
        Switching on zeroes the counts and empties the table.  Refused while ring_metrics is on."""
        self._check(self._L.gcra_ring_metrics_sharded(self._h, 1 if on else 0, max_keys))

    def ring_names_keep(self, key_hashes):
        """gcra_ring_names_keep: keep the name table's names of these hashes and forget the others -> the denied rows
        whose key found the table full since the last keep"""
        hs = np.ascontiguousarray(key_hashes, np.uint64)
        full = C.c_uint64()
        self._check(self._L.gcra_ring_names_keep(self._h, len(hs), hs.ctypes.data, C.byref(full)))
        return int(full.value)

    def policy_tick(self, now):
        """The store kind's sweep policy against the caller's clock (for device-resident / pipelined / sharded
        submissions, which never sweep by themselves); returns the number of entries removed."""
        r = C.c_uint64()
        self._check(self._L.gcra_policy_tick(self._h, _ns(now), C.byref(r)))
        return r.value

    def hash_key(self, key):
        """The identity THIS engine gives a key (SipHash-2-4 under the engine's seed when it has one)."""
        k = _kb(key)
        return int(self._L.gcra_engine_hash_key(self._h, k, len(k)))

    def hash_seed(self):
        out = (C.c_uint64 * 2)()
        self._L.gcra_get_hash_seed(self._h, C.byref(out))
        return int(out[0]), int(out[1])

    def peek(self, key_hash):
        t, e, f = C.c_int64(), C.c_int64(), C.c_uint8()
        self._check(self._L.gcra_peek(self._h, key_hash, C.byref(t), C.byref(e), C.byref(f)))
        return (t.value, e.value) if f.value else None

    def save(self, path):
        self._check(self._L.gcra_snapshot_save(self._h, os.fsencode(path)))

    def load(self, path):
        self._check(self._L.gcra_snapshot_load(self._h, os.fsencode(path)))

    def save_begin(self, path):
        """Begin a background save (gcra_snapshot_begin): the file will hold the table as every batch submitted before
        this call left it.  Returns at once; traffic continues while the file is written."""
        self._check(self._L.gcra_snapshot_begin(self._h, os.fsencode(path)))

    def save_poll(self):
        """True when no background save is in flight (the last one's file is complete); raises if it failed."""
        d = C.c_int32()
        self._check(self._L.gcra_snapshot_poll(self._h, C.byref(d)))
        return bool(d.value)

    def save_wait(self):
        """Wait for the background save; returns the number of entries written."""
        n = C.c_uint64()
        self._check(self._L.gcra_snapshot_wait(self._h, C.byref(n)))
        return n.value

    def restore(self, path, rank=0, world=1):
        """Insert the entries of a snapshot file that shard `rank` of `world` owns next to what this store holds
        (gcra_snapshot_restore); returns (restored, conflicts)."""
        r, c = C.c_uint64(), C.c_uint64()
        self._check(self._L.gcra_snapshot_restore(self._h, os.fsencode(path), rank, world, C.byref(r), C.byref(c)))
        return r.value, c.value

    def sync(self):
        self._check(self._L.gcra_sync(self._h))

    def last_kernel_ms(self):
        out = (C.c_float * 4)()
        self._check(self._L.gcra_last_kernel_ms(self._h, C.byref(out)))
        return [float(x) for x in out]

    def last_kernel_ms_detail(self):
        out = (C.c_float * 7)()
        self._check(self._L.gcra_last_kernel_ms_detail(self._h, C.byref(out)))
        return dict(zip(("probe", "unused", "decide_index", "resolve", "clear", "residue_sort", "residue_decide"),
                        [float(x) for x in out]))

    def last_sweep_ms(self):
        ms = C.c_float()
        self._check(self._L.gcra_last_sweep_ms(self._h, C.byref(ms)))
        return float(ms.value)

    def launch_count(self):
        return int(self._L.gcra_launch_count(self._h))


class _Builder:
    def __init__(self, cls):
        self._cls, self._kw = cls, {}

    def capacity(self, n):
        self._kw["capacity"] = n
        return self

    def device(self, d):
        self._kw["device"] = d
        return self

    def build(self):
        return self._cls(**self._kw)


class AdaptiveStore(_GpuStore):
    """adaptive_cleanup.rs: self-tuning sweep interval."""
    KIND = _native.STORE_ADAPTIVE

    class Builder(_Builder):             # adaptive_cleanup.rs:292-339
        def min_interval(self, secs):
            self._kw["p0"] = int(secs)
            return self

        def max_interval(self, secs):
            self._kw["p1"] = int(secs)
            return self

        def max_operations(self, n):
            self._kw["p2"] = int(n)
            return self

    @classmethod
    def builder(cls):
        return cls.Builder(cls)


class PeriodicStore(_GpuStore):
    """periodic.rs: sweep every cleanup_interval."""
    KIND = _native.STORE_PERIODIC

    class Builder(_Builder):             # periodic.rs:223-259
        def cleanup_interval(self, secs):
            self._kw["p0"] = int(secs)
            return self

    @classmethod
    def builder(cls):
        return cls.Builder(cls)


class ProbabilisticStore(_GpuStore):
    """probabilistic.rs: sweep when ops * 2654435761 % modulo == 0."""
    KIND = _native.STORE_PROBABILISTIC

    class Builder(_Builder):             # probabilistic.rs:197-233
        def cleanup_probability(self, modulo):
            self._kw["p0"] = int(modulo)
            return self

    @classmethod
    def builder(cls):
        return cls.Builder(cls)


class ManualStore(_GpuStore):
    """Never sweeps on its own (bench / tests drive gcra_sweep)."""
    KIND = _native.STORE_MANUAL


class RateLimiter:
    """rate_limiter.rs:42-58: owns its store."""

    def __init__(self, store):
        self.store = store
        self._L = store._L
        self._h = store._h

    @classmethod
    def new(cls, store):
        return cls(store)

    def rate_limit(self, key, max_burst, count_per_period, period, quantity, now):
        """rate_limiter.rs:102-110 -> (allowed, RateLimitResult); raises CellError."""
        k = _kb(key)
        out = np.zeros(1, RES_DTYPE)
        st = self._L.gcra_rate_limit(self._h, k, len(k), max_burst, count_per_period, period,
                                     quantity, _ns(now), out.ctypes.data)
        if st == NEGATIVE_QUANTITY:
            raise NegativeQuantity(quantity)
        if st == INVALID_RATE_LIMIT:
            raise InvalidRateLimit()
        if st != OK:
            raise Internal(self._L.gcra_last_error(self._h).decode())
        r = out[0]
        return bool(r["allowed"]), RateLimitResult(max_burst, int(r["remaining"]),
                                                   int(r["reset_after_ns"]), int(r["retry_after_ns"]))

    def rate_limit_batch(self, requests, out=None):
        """Apply REQ_DTYPE requests as if one after another in index order; RES_DTYPE results."""
        req = np.ascontiguousarray(requests, REQ_DTYPE)
        res = np.empty(len(req), RES_DTYPE) if out is None else out
        self.store._check(self._L.gcra_rate_limit_batch(self._h, len(req), req.ctypes.data, res.ctypes.data))
        return res

    def rate_limit_batch_keys(self, keys, rows, out=None):
        """rate_limit_batch with string keys: rows[i] (REQ_DTYPE, key_hash ignored) is decided for keys[i] (str or
        bytes), which the GPU hashes as store.hash_key would (gcra_rate_limit_batch_keys)."""
        refs, arena = pack_keys(keys)
        req = np.array(rows, REQ_DTYPE, copy=True)
        if len(req) != len(refs):
            raise ValueError("keys and rows differ in length")
        req["key_hash"] = refs
        res = np.empty(len(req), RES_DTYPE) if out is None else out
        self.store._check(self._L.gcra_rate_limit_batch_keys(self._h, len(req), req.ctypes.data, arena.ctypes.data,
                                                             len(arena), res.ctypes.data))
        return res

    def hash_keys_device(self, n, d_rows_ptr, row_bytes, d_keys_ptr, keys_len, stream=None):
        """The hash pass (gcra_hash_keys_device): n device rows of row_bytes (48 or 16) whose key_hash holds a key
        reference into the device arena d_keys_ptr (keys_len bytes) get the engine's hash of those bytes, in place,
        asynchronously on `stream`.  Enqueue it before a device batch call on the same stream."""
        self.store._check(self._L.gcra_hash_keys_device(self._h, n, d_rows_ptr, row_bytes, d_keys_ptr, keys_len,
                                                        stream))

    def set_policies(self, policies):
        pol = np.ascontiguousarray(policies, POLICY_DTYPE)
        self.store._check(self._L.gcra_set_policies(self._h, len(pol), pol.ctypes.data))

    def rate_limit_batch16(self, requests, now, out=None, compact_results=False):
        """REQ16_DTYPE requests against the registered policy table; RES_DTYPE results, or with compact_results
        RES16_DTYPE results (16 bytes: cur_tat_ns, status, allowed -- expand_results16 derives the rest)."""
        req = np.ascontiguousarray(requests, REQ16_DTYPE)
        if compact_results:
            res = np.empty(len(req), RES16_DTYPE) if out is None else out
            self.store._check(self._L.gcra_rate_limit_batch16_r16(self._h, len(req), req.ctypes.data, _ns(now),
                                                                  res.ctypes.data))
            return res
        res = np.empty(len(req), RES_DTYPE) if out is None else out
        self.store._check(self._L.gcra_rate_limit_batch16(self._h, len(req), req.ctypes.data, _ns(now),
                                                          res.ctypes.data))
        return res

    # device-resident batches (torch tensors or raw device pointers)
    def rate_limit_batch_device(self, n, d_req_ptr, d_res_ptr, stream=None):
        self.store._check(self._L.gcra_rate_limit_batch_device(self._h, n, d_req_ptr, d_res_ptr, stream))

    def submit_device(self, n, d_req_ptr, d_res_ptr, ready_stream=None):
        """Pipelined: ingest+order of this batch overlap the decide kernels of the previous one."""
        self.store._check(self._L.gcra_rate_limit_batch_device_pipelined(self._h, n, d_req_ptr, d_res_ptr, ready_stream))

    def join(self, stream=None):
        self.store._check(self._L.gcra_pipeline_join(self._h, stream))

    def rate_limit_batch16_device(self, n, d_req_ptr, now, d_res_ptr, stream=None, compact_results=False):
        """compact_results: d_res_ptr receives n RES16_DTYPE rows instead of RES_DTYPE rows."""
        fn = self._L.gcra_rate_limit_batch16_r16_device if compact_results else self._L.gcra_rate_limit_batch16_device
        self.store._check(fn(self._h, n, d_req_ptr, _ns(now), d_res_ptr, stream))


class Ring:
    """Pinned host ring (gcra_ring_*): fill a slot in place, submit, wait, read results in place.
    compact: False = REQ_DTYPE / RES_DTYPE slots, True = REQ16_DTYPE / RES_DTYPE, 2 = REQ16_DTYPE / RES16_DTYPE.
    key_capacity > 0: every slot also has a pinned key arena `keys[slot]` (uint8, key_capacity bytes); rows then
    hold key references (pack_keys) and submit(..., keys_len=...) hashes them on the GPU before the batch."""

    def __init__(self, limiter, slots, slot_capacity, compact=False, key_capacity=0):
        self.lim, self.store = limiter, limiter.store
        self._L, self._h = limiter._L, limiter._h
        self.slots, self.cap, self.compact, self.key_capacity = slots, slot_capacity, compact, key_capacity
        mode = 2 if (compact == 2 and compact is not True) else (1 if compact else 0)
        if key_capacity:
            self.store._check(self._L.gcra_ring_create_keyed(self._h, slots, slot_capacity, mode, key_capacity))
        else:
            self.store._check(self._L.gcra_ring_create(self._h, slots, slot_capacity, mode))
        dt = REQ16_DTYPE if mode else REQ_DTYPE
        rdt = RES16_DTYPE if mode == 2 else RES_DTYPE
        results = self._L.gcra_ring_results16 if mode == 2 else self._L.gcra_ring_results
        self.req, self.res = [], []
        for s in range(slots):
            rp = self._L.gcra_ring_requests(self._h, s)
            sp = results(self._h, s)
            rb = (C.c_char * (slot_capacity * dt.itemsize)).from_address(rp)
            sb = (C.c_char * (slot_capacity * rdt.itemsize)).from_address(sp)
            self.req.append(np.frombuffer(rb, dtype=dt))
            self.res.append(np.frombuffer(sb, dtype=rdt))
        self.keys = [np.frombuffer((C.c_char * key_capacity).from_address(self._L.gcra_ring_keys(self._h, s)),
                                   dtype=np.uint8) for s in range(slots)] if key_capacity else None

    def submit(self, slot, n, now=0, keys_len=None):
        """keys_len (keyed ring): the rows hold key references into the first keys_len bytes of keys[slot]."""
        if keys_len is None:
            self.store._check(self._L.gcra_ring_submit(self._h, slot, n, _ns(now)))
        else:
            self.store._check(self._L.gcra_ring_submit_keyed(self._h, slot, n, keys_len, _ns(now)))

    def wait(self, slot):
        self.store._check(self._L.gcra_ring_wait(self._h, slot))


class RespRing:
    """The engine's ring as a RESP ring (gcra_resp_ring_*): connections' read buffers in, reply bytes out.
    Fill input[slot] (uint8, in_capacity bytes) and conns[slot][:n] (RESP_CONN_DTYPE: off, len <= 65536), submit,
    wait; outcome[slot][:n] (RESP_OUTCOME_DTYPE) then says what each connection consumed, how many frames it had
    decided, where it stopped, and where its replies lie in replies[slot].  Contract and stop codes: gcra_b200.h.
    An engine has one ring: this takes the place of Ring.
    protocol="http" makes it an HTTP ring (gcra_http_ring_create): POST /throttle requests in, HTTP responses out,
    with the same calls and outcome table (HttpRing).  protocol="grpc" makes it a gRPC ring (GrpcRing), and
    protocol="mixed" a ring that takes all three in one slot (MixedRing)."""

    # protocol -> (create call, connection table and its dtype, outcome table and its dtype, reply bytes per row)
    _PROTOCOLS = {
        "resp": ("gcra_resp_ring_create", "gcra_resp_ring_conns", RESP_CONN_DTYPE, "gcra_resp_ring_outcome",
                 RESP_OUTCOME_DTYPE, RESP_REPLY_MAX),
        "http": ("gcra_http_ring_create", "gcra_resp_ring_conns", RESP_CONN_DTYPE, "gcra_resp_ring_outcome",
                 RESP_OUTCOME_DTYPE, HTTP_REPLY_MAX),
        "grpc": ("gcra_grpc_ring_create", "gcra_grpc_ring_conns", GRPC_CONN_DTYPE, "gcra_grpc_ring_outcome",
                 GRPC_OUTCOME_DTYPE, GRPC_REPLY_MAX),
        "mixed": ("gcra_mixed_ring_create", "gcra_mixed_ring_conns", MIXED_CONN_DTYPE, "gcra_resp_ring_outcome",
                  RESP_OUTCOME_DTYPE, HTTP_REPLY_MAX),
    }

    def __init__(self, limiter, slots, max_conns, in_capacity, row_capacity, protocol="resp"):
        if protocol not in self._PROTOCOLS:
            raise ValueError("protocol must be 'resp', 'http', 'grpc' or 'mixed'")
        create, conns, conn_dt, outcome, outcome_dt, reply_max = self._PROTOCOLS[protocol]
        self.lim, self.store = limiter, limiter.store
        self._L, self._h = limiter._L, limiter._h
        self.slots, self.max_conns, self.in_capacity, self.row_capacity = slots, max_conns, in_capacity, row_capacity
        self.protocol = protocol
        self.store._check(getattr(self._L, create)(self._h, slots, max_conns, in_capacity, row_capacity))

        def view(ptr, n, dt):
            return np.frombuffer((C.c_char * (n * np.dtype(dt).itemsize)).from_address(ptr), dtype=dt)
        L, h = self._L, self._h
        self.input = [view(L.gcra_resp_ring_input(h, s), in_capacity, np.uint8) for s in range(slots)]
        self.conns = [view(getattr(L, conns)(h, s), max_conns, conn_dt) for s in range(slots)]
        self.replies = [view(L.gcra_resp_ring_replies(h, s), row_capacity * reply_max, np.uint8)
                        for s in range(slots)]
        self.outcome = [view(getattr(L, outcome)(h, s), max_conns, outcome_dt) for s in range(slots)]
        if protocol == "mixed":                            # the gRPC connections' state and outcome rows
            self.grpc_conns = [view(L.gcra_grpc_ring_conns(h, s), max_conns, GRPC_CONN_DTYPE) for s in range(slots)]
            self.grpc_outcome = [view(L.gcra_grpc_ring_outcome(h, s), max_conns, GRPC_OUTCOME_DTYPE)
                                 for s in range(slots)]

    def submit(self, slot, n_conns, now=0):
        self.store._check(self._L.gcra_resp_ring_submit(self._h, slot, n_conns, _ns(now)))

    def peer_memory(self, on=True):
        """on: every later submit is a peer-memory tick of the engine's gcra_p2p_* ranks (gcra_ring_p2p): the rows
        are decided on their keys' owners, against the ranks' one sharded table.  Contract: gcra_b200.h."""
        self.store._check(self._L.gcra_ring_p2p(self._h, 1 if on else 0))

    def submit_route(self, slot, n_conns, now=0):
        """First half of a peer-memory submit: parse the slot and route its rows to their owners.  Engines of one
        process route every engine's tick before the first submit_finish."""
        self.store._check(self._L.gcra_resp_ring_submit_route(self._h, slot, n_conns, _ns(now)))

    def submit_finish(self, slot):
        """Second half: decide this rank's inbox, bring the slot's results back, write its replies and outcomes."""
        self.store._check(self._L.gcra_resp_ring_submit_finish(self._h, slot))

    def wait(self, slot):
        self.store._check(self._L.gcra_ring_wait(self._h, slot))

    def rows(self, slot):
        """after wait: the slot's parsed rows and their results (REQ_DTYPE, RES_DTYPE), in batch order"""
        req = np.empty(self.row_capacity, REQ_DTYPE)
        res = np.empty(self.row_capacity, RES_DTYPE)
        n = C.c_uint32()
        self.store._check(self._L.gcra_resp_ring_rows(self._h, slot, req.ctypes.data, res.ctypes.data,
                                                      self.row_capacity, C.byref(n)))
        return req[:n.value], res[:n.value]


def HttpRing(limiter, slots, max_conns, in_capacity, row_capacity):
    """The engine's ring as an HTTP ring: RespRing(..., protocol="http")."""
    return RespRing(limiter, slots, max_conns, in_capacity, row_capacity, protocol="http")


def GrpcRing(limiter, slots, max_conns, in_capacity, row_capacity):
    """The engine's ring as a gRPC ring (gcra_grpc_ring_create): HTTP/2 connections' bytes in, Throttle responses
    out.  RespRing(..., protocol="grpc"): conns[slot] is GRPC_CONN_DTYPE (off, len and the connection's HTTP/2 state:
    last_stream, send_window, init_window and the class bytes of its HPACK dynamic table) and outcome[slot] is
    GRPC_OUTCOME_DTYPE (RespRing's fields, the DATA octets taken and sent, a PING to acknowledge and the state after
    the walk).  Contract and stop codes: gcra_b200.h.  throttlecrab_b200.grpc_transport drives one."""
    return RespRing(limiter, slots, max_conns, in_capacity, row_capacity, protocol="grpc")


def MixedRing(limiter, slots, max_conns, in_capacity, row_capacity):
    """The engine's ring as a mixed ring (gcra_mixed_ring_create): RESP, HTTP and gRPC connections in one slot, all
    their rows decided as one batch on the engine's one table.  RespRing(..., protocol="mixed"): conns[slot] is
    MIXED_CONN_DTYPE (off, len, protocol PROTO_RESP / PROTO_HTTP / PROTO_GRPC and, for gRPC, grpc_state: 0, 1, 2, ...
    in table order among the gRPC connections); grpc_conns[slot][grpc_state] (GRPC_CONN_DTYPE, off and len unused)
    holds a gRPC connection's HTTP/2 state and grpc_outcome[slot][grpc_state] (GRPC_OUTCOME_DTYPE) receives its
    outcome; outcome[slot] (RESP_OUTCOME_DTYPE) has every connection's.  replies[slot] has HTTP_REPLY_MAX bytes per
    row.  Contract: gcra_b200.h.  throttlecrab_b200.mixed drives one."""
    return RespRing(limiter, slots, max_conns, in_capacity, row_capacity, protocol="mixed")
