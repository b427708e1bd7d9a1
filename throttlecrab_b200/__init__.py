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
from ._native import (REQ_DTYPE, RES_DTYPE, REQ16_DTYPE, POLICY_DTYPE, OK, NEGATIVE_QUANTITY,
                      INVALID_RATE_LIMIT, INTERNAL)

__all__ = ["RateLimiter", "RateLimitResult", "Rate", "CellError", "NegativeQuantity", "InvalidRateLimit",
           "Internal", "AdaptiveStore", "PeriodicStore", "ProbabilisticStore", "ManualStore",
           "hash_key", "derive_params", "REQ_DTYPE", "RES_DTYPE", "REQ16_DTYPE", "POLICY_DTYPE"]

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

    def set_policies(self, policies):
        pol = np.ascontiguousarray(policies, POLICY_DTYPE)
        self.store._check(self._L.gcra_set_policies(self._h, len(pol), pol.ctypes.data))

    def rate_limit_batch16(self, requests, now, out=None):
        req = np.ascontiguousarray(requests, REQ16_DTYPE)
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

    def rate_limit_batch16_device(self, n, d_req_ptr, now, d_res_ptr, stream=None):
        self.store._check(self._L.gcra_rate_limit_batch16_device(self._h, n, d_req_ptr, _ns(now), d_res_ptr, stream))


class Ring:
    """Pinned host ring (gcra_ring_*): fill a slot in place, submit, wait, read results in place."""

    def __init__(self, limiter, slots, slot_capacity, compact=False):
        self.lim, self.store = limiter, limiter.store
        self._L, self._h = limiter._L, limiter._h
        self.slots, self.cap, self.compact = slots, slot_capacity, compact
        self.store._check(self._L.gcra_ring_create(self._h, slots, slot_capacity, 1 if compact else 0))
        dt = REQ16_DTYPE if compact else REQ_DTYPE
        self.req, self.res = [], []
        for s in range(slots):
            rp = self._L.gcra_ring_requests(self._h, s)
            sp = self._L.gcra_ring_results(self._h, s)
            rb = (C.c_char * (slot_capacity * dt.itemsize)).from_address(rp)
            sb = (C.c_char * (slot_capacity * RES_DTYPE.itemsize)).from_address(sp)
            self.req.append(np.frombuffer(rb, dtype=dt))
            self.res.append(np.frombuffer(sb, dtype=RES_DTYPE))

    def submit(self, slot, n, now=0):
        self.store._check(self._L.gcra_ring_submit(self._h, slot, n, _ns(now)))

    def wait(self, slot):
        self.store._check(self._L.gcra_ring_wait(self._h, slot))
