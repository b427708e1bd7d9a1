"""16-byte results of compact requests, on the host alone: gcra_expand_results16 turns the oracle's `cur` (read off
its store by oracle_cur.py), status and allowed into exactly the oracle's 32-byte result -- over the adversarial
corners of test_oracle_vs_python_model.py expressed as compact requests (a policy table and an i32 quantity):
saturation, the u32 burst truncation, TTL wrap, ei = 0, max_burst = 1 with q = 0, invalid and overflowing policies.
No device work."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import oracle
import oracle_cur
import throttlecrab_b200 as tc
from throttlecrab_b200 import _native

I64_MAX, I32_MAX = 2**63 - 1, 2**31 - 1
T0 = 1_700_000_000 * 10**9


def test_result16_layout():
    assert tc.RES16_DTYPE.itemsize == 16
    assert tc.RES16_DTYPE.fields["cur_tat_ns"][1] == 0
    assert tc.RES16_DTYPE.fields["status"][1] == 8 and tc.RES16_DTYPE.fields["allowed"][1] == 12


def policy_table(policies):
    pol = np.zeros(len(policies), tc.POLICY_DTYPE)
    if len(policies):
        pol["max_burst"], pol["count_per_period"], pol["period"] = np.array(policies, dtype=object).T
    return pol


def replay_compact(policies, steps):
    """Every step (key, policy index, quantity, now) through the oracle one call at a time, then the oracle's
    (cur, status, allowed) through gcra_expand_results16 row by row (one `now` per row); returns (oracle rows,
    expanded rows)."""
    orc = oracle.OracleStore(oracle.PERIODIC, capacity=100, created_ns=T0, p0=10**9)
    table = policy_table(policies)
    want = np.zeros(len(steps), tc.RES_DTYPE)
    got = np.zeros(len(steps), tc.RES_DTYPE)
    for i, (key, p, q, now) in enumerate(steps):
        req16 = np.zeros(1, tc.REQ16_DTYPE)
        req16["key_hash"], req16["quantity"], req16["policy"] = key, q, p
        res16 = np.zeros(1, tc.RES16_DTYPE)
        if p < len(policies):
            row, cur = oracle_cur.rate_limit_cur(orc, "k%d" % key, *[int(x) for x in policies[p]], q, now)
            want[i]["status"], want[i]["allowed"] = row[0], row[1]
            want[i]["remaining"], want[i]["reset_after_ns"], want[i]["retry_after_ns"] = row[2:]
            res16["cur_tat_ns"], res16["status"], res16["allowed"] = cur, row[0], row[1]
        else:
            want[i]["status"] = tc.INTERNAL           # the engine refuses a policy index beyond the table
            res16["status"] = tc.INTERNAL
        got[i] = tc.expand_results16(req16, now, table, res16)[0]
    return want, got


def assert_rows_equal(want, got, steps):
    a = want.view(np.uint8).reshape(len(want), -1)
    b = got.view(np.uint8).reshape(len(got), -1)
    bad = np.nonzero((a != b).any(axis=1))[0]
    assert len(bad) == 0, "row %d: oracle=%s expanded=%s step=%s" % (bad[0], want[bad[0]], got[bad[0]], steps[bad[0]])


# (max_burst, count, period) with the corner each reaches
CORNERS = [
    (100, 1000, 60),                 # ordinary
    (3, 7, 60),                      # inexact emission interval
    (1, 3, 3600),                    # max_burst = 1: dvt = 0, zero quantities toggle the entry
    (2**32 + 1, 1, 60),              # (max_burst - 1) as u32 == 0: no burst at all
    (2**32, 1, 60),                  # as u32 == 2^32 - 1: a huge dvt
    (5, 10**18, 1),                  # ei = 0 (period * 1e9 / count < 1): remaining is 0
    (2, 1, I64_MAX),                 # ei beyond i64: saturation everywhere, expiry clamps
    (I64_MAX, 1, 10**9),             # Duration * u32 overflows: GCRA_INTERNAL
    (2**32, 1, 2**63 - 1),           # the same through a wrapped factor
    (0, 10, 60), (5, -5, 60), (5, 10, 0),   # invalid: GCRA_INVALID_RATE_LIMIT
    (10, 3, 2**40),                  # ei * q saturates for large quantities
]

policy_st = st.one_of(st.sampled_from(CORNERS),
                      st.tuples(st.integers(-1, 2**33), st.integers(-1, 2**62), st.integers(-1, 2**62)))
qty_st = st.one_of(st.integers(-2, 6), st.sampled_from([0, 1, I32_MAX, -2**31]), st.integers(0, I32_MAX))
dt_st = st.one_of(st.sampled_from([0, 0, 1, 999_999_999, 10**9, 6 * 10**9, 3600 * 10**9]),
                  st.integers(-10**10, 10**13), st.sampled_from([2**62, -2**62]))


@settings(max_examples=400, deadline=None)
@given(st.lists(policy_st, min_size=1, max_size=6),
       st.lists(st.tuples(st.integers(0, 3), st.integers(0, 7), qty_st, dt_st), min_size=1, max_size=40))
def test_expanded_oracle_cur_equals_oracle_results(policies, raw):
    """Random sequences over random tables (indices past the table included): the expansion of (cur, status,
    allowed) is the oracle's 32-byte row, byte for byte.  Clocks wander far from T0, including below 0 and towards
    2^63, so the wrapping `now + dvt` and the TTL / expiry clamps are reached."""
    steps, now = [], T0
    for key, p, q, d in raw:
        now = min(max(now + d, -10**9), I64_MAX)
        steps.append((key, p, q, now))
    want, got = replay_compact(policies, steps)
    assert_rows_equal(want, got, steps)


def test_expanded_oracle_cur_on_hand_picked_corners():
    """Each corner policy driven through allowed, denied, exhausted, expired and saturated states."""
    steps = []
    now = T0
    for p in range(len(CORNERS)):
        for q in (0, 1, 0, 1, 5, I32_MAX, 0, 1, -1, 0):
            steps.append((p % 4, p, q, now))
            now += 1_000_000
        for q, d in ((1, 10**13), (0, 0), (0, 0), (1, 2**61), (I32_MAX, 0), (0, 0)):
            now += d
            steps.append((p % 4, p, q, now))
        now = T0 + (p + 1) * 10**12
    steps.append((0, len(CORNERS), 1, now))          # a policy index beyond the table
    steps.append((0, 2**32 - 1, 1, now))
    steps.append((0, 0, 1, -1))                      # a pre-epoch clock: GCRA_INTERNAL
    want, got = replay_compact(CORNERS, steps)
    assert_rows_equal(want, got, steps)
    statuses = set(int(x) for x in want["status"])
    assert statuses == {0, 1, 2, 3}, statuses
    ok = want["status"] == 0
    assert want["allowed"][ok].any() and not want["allowed"][ok].all()


def test_expand_batch_and_wrong_table():
    """A whole batch in one call (one clock); an OK row whose policy is missing from the table given is reported
    (Internal), and error rows are expanded without reading the table at all."""
    pol = policy_table(CORNERS[:3])
    req = np.zeros(4, tc.REQ16_DTYPE)
    req["key_hash"] = [1, 2, 3, 4]
    req["quantity"] = [1, 1, -1, 1]
    req["policy"] = [0, 2, 0, 99]
    res = np.zeros(4, tc.RES16_DTYPE)
    res["cur_tat_ns"] = [T0, T0 - 5, 0, 0]
    res["status"] = [0, 0, tc.NEGATIVE_QUANTITY, tc.INTERNAL]
    res["allowed"] = [1, 0, 0, 0]
    out = tc.expand_results16(req, T0, pol, res)
    assert out["status"].tolist() == [0, 0, 1, 3]
    assert (out[2:].view(np.uint8).reshape(2, -1)[:, :24] == 0).all() and (out["allowed"][2:] == 0).all()
    orc = oracle.OracleStore(oracle.PERIODIC, capacity=10, created_ns=T0, p0=10**9)
    row, cur = oracle_cur.rate_limit_cur(orc, "x", 100, 1000, 60, 1, T0)
    assert cur == T0 and row[1]          # a fresh key spends one emission interval: new_tat = now
    # the same batch against a table that lacks policy 2: reported, not silently wrong
    with pytest.raises(tc.Internal):
        tc.expand_results16(req, T0, pol[:2], res)
    # the C entry point itself: no handle, a row written with status GCRA_INTERNAL
    L = _native.lib()
    out2 = np.zeros(4, tc.RES_DTYPE)
    rc = L.gcra_expand_results16(4, req.ctypes.data, T0, pol.ctypes.data, 2, res.ctypes.data, out2.ctypes.data)
    assert rc == tc.INTERNAL and out2["status"].tolist() == [0, 3, 1, 3]
