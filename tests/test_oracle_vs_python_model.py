"""An independent arbitrary-precision restatement of the decision (SURVEY Appendix A, written from the
pseudocode with Python integers and explicit clamps) against the C++ oracle on random and adversarial
sequences -- saturation, the u32 burst truncation, the wrapping `now + dvt`, TTL wrap, expiry boundaries.
Two independently written restatements agreeing does not replace the reference's known-answer tests (those
pin the oracle in test_oracle_known_answers.py); it guards the corners those tests do not reach."""
import math

from hypothesis import given, settings, strategies as st

import oracle

I64_MAX, I64_MIN, U64 = 2**63 - 1, -2**63, 2**64


def clamp(x):
    return I64_MAX if x > I64_MAX else I64_MIN if x < I64_MIN else x


def wrap64(x):
    x &= U64 - 1
    return x - U64 if x >= 2**63 else x


def derive(max_burst, count, period):
    v = float(period) * 1e9 / float(count)                     # rate/mod.rs:172, IEEE double
    ei_u = 0 if (math.isnan(v) or v <= 0) else (U64 - 1 if v >= 18446744073709551616.0 else int(v))
    factor = (max_burst - 1) & 0xFFFFFFFF                      # (max_burst - 1) as u32
    dvt_u = ei_u * factor
    panics = dvt_u // 10**9 > U64 - 1                          # Duration * u32 overflow
    return panics, wrap64(ei_u), wrap64(dvt_u)


class Model:
    def __init__(self):
        self.t = {}                                            # key -> (tat, expiry as unbounded int)
        self.expired_writes = 0                                # allowed writes over an existing, expired entry

    def rate_limit(self, key, max_burst, count, period, q, now):
        if q < 0:
            return (1, False, 0, 0, 0)
        if max_burst <= 0 or count <= 0 or period <= 0:
            return (2, False, 0, 0, 0)
        panics, ei, dvt = derive(max_burst, count, period)
        if panics or now < 0:
            return (3, False, 0, 0, 0)
        e = self.t.get(key)
        live = e is not None and e[1] > now
        tat = max(e[0], clamp(now - dvt)) if live else clamp(now - ei)
        new_tat = clamp(tat + clamp(ei * q))
        allow_at = clamp(new_tat - dvt)
        allowed = now >= allow_at
        if allowed:
            self.expired_writes += e is not None and not live
            ttl = clamp(clamp(new_tat - now) + dvt) % U64     # `as u64`
            self.t[key] = (new_tat, now + ttl)
        cur = new_tat if allowed else tat
        room = clamp(wrap64(now + dvt) - cur)
        remaining = max(_tdiv(room, ei), 0) if ei > 0 else 0
        reset = max(clamp(clamp(cur - now) + dvt), 0)
        retry = 0 if allowed else max(clamp(allow_at - now), 0)
        return (0, allowed, remaining, reset, retry)


def _tdiv(a, b):                                              # truncating division
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


T0 = 1_700_000_000 * 10**9
small = st.integers(1, 200)
edge = st.sampled_from([1, 2, 3, 2**31, 2**32, 2**32 + 1, 2**33 + 7, I64_MAX // 1000, I64_MAX - 1, I64_MAX])
posint = st.one_of(small, edge, st.integers(1, I64_MAX))
qty = st.one_of(st.integers(-2, 6), st.sampled_from([0, 1, I64_MAX // 2, I64_MAX]), st.integers(0, 10**12))
dt = st.one_of(st.sampled_from([0, 0, 1, 999_999_999, 10**9, 6 * 10**9, 3600 * 10**9]), st.integers(-10**10, 10**13))
step = st.tuples(st.integers(0, 2), posint, posint, posint, qty, dt)


@settings(max_examples=400, deadline=None)
@given(st.lists(step, min_size=1, max_size=40))
def test_oracle_matches_python_model(steps):
    orc = oracle.OracleStore(oracle.PERIODIC, capacity=100, created_ns=T0, p0=10**9)
    mod = Model()
    now = T0
    for key, b, c, p, q, d in steps:
        now = max(now + d, 0)
        got = orc.rate_limit("k%d" % key, b, c, p, q, now)
        want = mod.rate_limit(key, b, c, p, q, now)
        assert got == want, ((key, b, c, p, q, now), got, want)
        ent = orc.entry("k%d" % key)
        me = mod.t.get(key)
        assert (ent is None) == (me is None)
        if me is not None:
            assert ent == (me[0], min(me[1], I64_MAX))
        assert orc.expired_writes() == mod.expired_writes


def test_expired_writes_count_every_write_over_an_expired_entry():
    """The oracle's expired-write total (the engine's expired_hits) on hand-picked boundaries: a write exactly at
    expiry counts, one a nanosecond before does not, denied requests and a swept entry never count, and it is
    counted for every store kind."""
    b, c, p = 2, 120, 60                                         # P5: ei = dvt = 0.5 s
    _, ei, dvt = derive(b, c, p)
    # (all clocks stay below the adaptive store's first cleanup at created + 5 s, so no store sweeps on its own)
    steps = [("a", 1, T0), ("a", 1, T0 + dvt - 1), ("a", 1, T0 + 4 * 10**9),   # written, live, expired: counts
             ("b", 0, T0), ("b", 0, T0),                                       # a zero TTL: expiry == now counts
             ("c", b + 1, T0), ("c", 1, T0 + 4 * 10**9)]                       # denied: no entry, then a fresh one
    for kind in (oracle.PERIODIC, oracle.PROBABILISTIC, oracle.ADAPTIVE):
        orc = oracle.OracleStore(kind, capacity=100, created_ns=T0, p0=10**9, p1=10**9, p2=10**9)
        mod = Model()
        for key, q, now in steps:
            assert orc.rate_limit(key, b, c, p, q, now) == mod.rate_limit(key, b, c, p, q, now)
        assert orc.sweeps() == 0
        assert orc.expired_writes() == mod.expired_writes == 2, (kind, orc.expired_writes(), mod.expired_writes)
        orc.force_sweep(T0 + 10**13)                             # a swept entry is gone: the next write is fresh
        orc.rate_limit("a", b, c, p, 1, T0 + 10**13)
        assert orc.expired_writes() == 2


@settings(max_examples=300, deadline=None)
@given(posint, posint, posint)
def test_derive_matches_python_model(b, c, p):
    panics, ei, dvt = derive(b, c, p)
    assert oracle.derive(b, c, p) == (3 if panics else 0, ei, dvt)
