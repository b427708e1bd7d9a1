"""Decisions off the fast path, in every K1 kernel, against the oracle.

`decide()` (gcra_device.cuh) runs plain 64-bit arithmetic only when `ordinary_request()` holds (0 <= now < 2^61,
ei, dvt and q below 2^60, ei * q < 2^60 and, for a live entry, |tat| < 2^61); everything else goes through the
saturating forms.  `outputs_from()` has the same split (`plain`: now < 2^61, dvt < 2^60, |cur| < 2^62).  2^61 ns after
the epoch is 2043-01-25 23:56:49 UTC: from then on every decision takes the saturating forms.  Each kernel also decides
on its own whether an allowed request changed the state, which picks the final rows, the retrying lanes, the marks
and the residue.  Here the traces that reach every kernel (warp chunks, one-CTA runs of 256-4095 rows, cluster runs of
4096 and more with their finite-state rounds, index-order passes B and C with marks, PEND deferral and the residue
tail) run with clocks past 2^61 and 2^62 and up to I64_MAX, with request magnitudes straddling the bounds and with
stored TATs beyond +-2^61.

Every scenario compares every row bit-exact with ONE oracle store replaying the same rows in order, then the final
entries of its corner keys and the counters.  A numpy restatement of the two predicates (`ordinary` and `plain` below)
proves that each scenario really has rows on both sides of the bounds it names, so that a later trace edit cannot
move it back onto the fast path unnoticed."""
import functools

import numpy as np
import pytest

import oracle
import oracle_cur
import throttlecrab_b200 as tc
import traces
from gpu_util import engine_requests, first_mismatch
from test_compact_results_cpu import CORNERS
from test_gpu_compact_results import STAT_DECISIONS, assert_pair
from test_gpu_pipelined_runs import assert_counters, check_universe, ring_run

pytestmark = pytest.mark.gpu

T0 = traces.T0
MS, S = 1_000_000, 1_000_000_000
I64_MAX, I32_MAX = 2**63 - 1, 2**31 - 1
B60, B61, B62 = 1 << 60, 1 << 61, 1 << 62
NEVER = 10**10          # oracle cleanup interval (s): its first periodic sweep would fall past I64_MAX
TOGGLER = 90_000_000    # max_burst = 1, q = 0: the entry toggles between live and expired on every row


# ---------------------------------------------------------------------------------------------------------------
# the two predicates, restated
# ---------------------------------------------------------------------------------------------------------------
def _u(x):
    return np.asarray(x, np.int64).view(np.uint64)


def mul_u64(a, b):
    """(hi, lo) words of the exact 128-bit products of two u64 arrays (__umul64hi and the wrapping product)"""
    m32, s32 = np.uint64(0xFFFFFFFF), np.uint64(32)
    a_lo, a_hi, b_lo, b_hi = a & m32, a >> s32, b & m32, b >> s32
    p0, p1, p2, p3 = a_lo * b_lo, a_lo * b_hi, a_hi * b_lo, a_hi * b_hi
    mid = (p0 >> s32) + (p1 & m32) + (p2 & m32)
    return p3 + (p1 >> s32) + (p2 >> s32) + (mid >> s32), a * b


def derived(max_burst, count, period):
    """(ei, dvt) of every row from tc.derive_params, which must equal oracle.derive for every policy."""
    cols = np.stack([max_burst, count, period], 1).astype(np.int64)
    u, inv = np.unique(cols, axis=0, return_inverse=True)
    ei, dvt = np.zeros(len(u), np.int64), np.zeros(len(u), np.int64)
    for i, p in enumerate(u.tolist()):
        d = tc.derive_params(*p)
        assert d == oracle.derive(*p), (p, d, oracle.derive(*p))
        ei[i], dvt[i] = d[1], d[2]
    inv = inv.reshape(-1)
    return ei[inv], dvt[inv]


class Sides:
    """The fast-path predicates of every row, from the request fields (and `cur` where it is known)."""

    def __init__(self, max_burst, count, period, q, now, cur=None):
        self.ei, self.dvt = derived(max_burst, count, period)
        now, q = np.asarray(now, np.int64), np.asarray(q, np.int64)
        s60, s61 = np.uint64(60), np.uint64(61)
        hi, lo = mul_u64(_u(self.ei), _u(q))
        self.inc_big = (hi != 0) | ((lo >> s60) != 0)          # ei * q >= 2^60, exactly
        self.hi_only = (hi != 0) & ((lo >> s60) == 0)           # ... seen by the hi word alone
        self.dvt_big = (_u(self.dvt) >> s60) != 0
        self.now_big = (_u(now) >> s61) != 0
        small = ((_u(self.ei) >> s60) | (_u(q) >> s60)) == 0
        # ordinary_request(): the request alone (the stored tat's bound is checked where a scenario claims it)
        self.ordinary = ~self.now_big & small & ~self.dvt_big & ~self.inc_big
        self.plain = ~self.now_big & ~self.dvt_big
        if cur is not None:
            cur = np.asarray(cur, np.int64)
            self.plain &= (cur > -B62) & (cur < B62)
        # now + dvt past I64_MAX: the wrapping sum of outputs_from
        self.wraps = (self.dvt >= 0) & (now > I64_MAX - np.maximum(self.dvt, 0))


def sides(mask, decided, what):
    """rows of `decided` on both sides of one bound"""
    n_in, n_out = int((mask & decided).sum()), int((~mask & decided).sum())
    assert n_in > 0 and n_out > 0, "%s: %d rows inside, %d outside" % (what, n_in, n_out)


def req_sides(req, cur=None):
    return Sides(req["max_burst"], req["count_per_period"], req["period"], req["quantity"], req["now_ns"], cur)


def test_restated_predicates_on_hand_picked_rows():
    """The restatement against hand-derived verdicts, which the other tests' side checks rest on.  It needs no GPU,
    but runs with the rest of this file under the `gpu` mark."""
    k = 40
    rows = [  # (max_burst, count, period, q, now, ordinary, plain)
        (100, 1000, 60, 1, T0, True, True),
        (100, 1000, 60, 1, B61 - 1, True, True),
        (100, 1000, 60, 1, B61, False, False),
        (100, 1000, 60, 1, -1, False, False),
        ((1 << 20), 10**9, 1 << k, 1, T0, True, True),              # dvt = 2^60 - 2^40
        ((1 << 20) + 1, 10**9, 1 << k, 1, T0, False, False),        # dvt = 2^60
        (2, 10**9, 1 << k, (1 << 20) - 1, T0, True, True),         # ei * q = 2^60 - 2^40
        (2, 10**9, 1 << k, 1 << 20, T0, False, True),               # ei * q = 2^60
        (2, 10**9, 1 << k, 1 << 24, T0, False, True),               # ei * q = 2^64: only the hi term
        (2**32 + 1, 10**9, 1 << 30, 1, T0, True, True),             # factor truncated to 0
        (2**32, 10**9, 1 << 30, 1, T0, False, False),               # factor 2^32 - 1: dvt ~ 2^62
        (2, 1, I64_MAX, 1, T0, False, False),                       # ei = dvt = -1
    ]
    a = np.array(rows, dtype=object)
    s = Sides(*[a[:, i].astype(np.int64) for i in range(5)])
    assert s.ordinary.tolist() == [bool(x) for x in a[:, 5]]
    assert s.plain.tolist() == [bool(x) for x in a[:, 6]]
    assert s.hi_only.tolist() == [i == 8 for i in range(len(rows))]


# ---------------------------------------------------------------------------------------------------------------
# engine and oracle runs
# ---------------------------------------------------------------------------------------------------------------
def new_oracle(created_ns, kind=oracle.PERIODIC, p0=NEVER):
    return oracle.OracleStore(kind, capacity=1000, created_ns=created_ns, p0=p0)


def run_engine(req, bounds, capacity, store_cls=tc.ManualStore, created_ns=0):
    st = store_cls(capacity=capacity, created_ns=created_ns, max_batch=int(np.diff(bounds).max()))
    lim = tc.RateLimiter(st)
    ereq = engine_requests(req)
    got = np.empty(len(req), tc.RES_DTYPE)
    for a, b in zip(bounds, bounds[1:]):
        lim.rate_limit_batch(ereq[a:b], out=got[a:b])
    return st, got


def assert_entries(st, ora, keys):
    hashes = tc.hash_key_ids(np.asarray(keys, np.uint64))
    for k, h in zip(keys, hashes):
        assert st.peek(int(h)) == ora.entry("k:%d" % k), k


def assert_engine(req, bounds, want, ora, capacity, corner_keys):
    """engine rows, corner entries and counters against the oracle that produced `want`"""
    st, got = run_engine(req, bounds, capacity)
    bad = first_mismatch(want, got, req)
    assert bad is None, bad
    assert_entries(st, ora, corner_keys)
    assert_counters(st, want, ora, require_expired=len(corner_keys) > 1)    # one key alone never expires here
    return st


# ---------------------------------------------------------------------------------------------------------------
# scenario 1: realistic traces with every clock shifted
# ---------------------------------------------------------------------------------------------------------------
TICK = 1 << 17


def hot_trace():
    """config4 hot keys in 2^17-row ticks: 24 hot keys (~2700 rows a tick: one-CTA runs), two of them merged into one
    (~5500 rows: a cluster run), cold keys in warp chunks, and a toggling key with 4500 rows a tick."""
    n_keys, n_ticks = 50_000, 4
    req = traces.config4(n_keys=n_keys, n_ticks=n_ticks, tick_size=TICK, hot=24)
    hot = traces.rank_to_key(np.arange(24, dtype=np.uint64), n_keys)
    req["key"][req["key"] == hot[1]] = hot[0]
    rng = np.random.default_rng(31)
    for t in range(n_ticks):
        tog = t * TICK + rng.choice(TICK, 4500, replace=False)
        req["key"][tog] = TOGGLER
        req["quantity"][tog] = 0
    traces.fill_policy(req, (req["key"] % np.uint64(8)).astype(np.int64))
    req["max_burst"][req["key"] == TOGGLER], req["count_per_period"][req["key"] == TOGGLER] = 1, 3
    req["period"][req["key"] == TOGGLER] = 3600
    aligned = [t * TICK for t in range(n_ticks + 1)]
    straddle = [0] + [t * TICK + TICK // 2 for t in range(n_ticks)] + [n_ticks * TICK]
    corner = hot.tolist() + [TOGGLER] + list(range(0, n_keys, 997))
    return req, aligned, straddle, corner, n_keys + 10


def single_key_trace():
    """The one-key 2^20-row mixed run of test_gpu_full_size: cluster plain and finite-state rounds."""
    n = 1 << 20
    rng = np.random.default_rng(5)
    req = np.zeros(n, traces.REQ_DTYPE)
    req["key"] = 7
    pol = np.repeat(rng.integers(0, 8, n // 4096 + 1), 4096)[:n]
    mixed = rng.random(n) < 0.02
    pol[mixed] = rng.integers(0, 8, int(mixed.sum()))
    traces.fill_policy(req, pol)
    req["quantity"] = rng.choice([0, 1, 1, 1, 1, 2, 5], n)
    req["now_ns"] = T0 + np.cumsum(rng.choice([0, 0, 0, 1000, 1_000_000, 50_000_000], n))
    now = req["now_ns"]
    mid = n // 2 + int(np.argmax(now[n // 2:] > now[n // 2 - 1]))
    return req, [0, mid, n], [0, n], [7], 100


def zipf_trace():
    """A warm pass over 200 K keys, then two Zipf ticks of 2^17 rows: index-order residue, marks and PEND deferral."""
    n_keys = 200_000
    req = np.concatenate([traces.warm_pass(n_keys), traces.config2(n_keys=n_keys, n_ticks=2, tick_size=TICK)])
    w = n_keys
    u, c = np.unique(req["key"][w:w + TICK], return_counts=True)
    corner = u[np.argsort(-c)[:40]].tolist() + list(range(0, n_keys, 4999))
    return (req, [0, w, w + TICK, w + 2 * TICK], [0, w, w + TICK // 2, w + 3 * TICK // 2, w + 2 * TICK], corner,
            n_keys)


TRACES = {"hot": hot_trace, "single_key": single_key_trace, "zipf": zipf_trace}
PLACEMENTS = {"a": "from 2^61", "b": "from 2^62", "c": "2^61 inside a batch", "d": "entries written below 2^61"}


@functools.lru_cache(maxsize=None)
def base_trace(name):
    req, aligned, straddle, corner, capacity = TRACES[name]()
    want = new_oracle(int(req["now_ns"][0])).replay(req)
    return req, aligned, straddle, corner, capacity, want


def placement(now, aligned, straddle, where):
    """(shift, batch bounds, row index where the shifted trace reaches 2^61 or 2^62)"""
    if where in ("a", "b"):
        return (B61 if where == "a" else B62) - int(now[0]), aligned, 0
    if where == "c":                                   # the first batch holding two clocks: 2^61 in its middle
        for a, b in zip(straddle, straddle[1:]):
            if now[a] != now[b - 1]:
                m = (a + b) // 2
                i = m + int(np.argmax(now[m:b] > now[m - 1]))
                assert now[i] > now[i - 1]
                return B61 - int(now[i]), straddle, i
    b = aligned[len(aligned) // 2]                     # "d": batches before b below 2^61, b and later above
    assert now[b] > now[b - 1]
    return B61 - int(now[b]), aligned, b


@functools.lru_cache(maxsize=None)
def shifted(name, where):
    req0, aligned, straddle, corner, capacity, want0 = base_trace(name)
    delta, bounds, cut = placement(req0["now_ns"], aligned, straddle, where)
    req = req0.copy()
    req["now_ns"] += delta
    ora = new_oracle(int(req["now_ns"][0]))
    want = ora.replay(req)
    return req, bounds, cut, corner, capacity, want, ora


@pytest.mark.parametrize("where", list(PLACEMENTS))
@pytest.mark.parametrize("name", list(TRACES))
def test_shifted_clocks(name, where):
    """config4 hot keys (warp chunks, 256-4095-row runs, a run of ~5500 rows and a 4500-row toggling key in each
    2^17-row batch), the one-key 2^20-row run, and Zipf ticks after a warm pass (batches of 2^17 rows and more), with
    every clock moved by one constant: (a) the whole trace from 2^61, (b) from 2^62, (c) 2^61 reached between two
    rows of one batch, (d) entries written below 2^61 read by later batches above it.  GCRA results depend on time
    differences alone away from saturation, so the oracle's rows must equal its rows for the unshifted trace; the
    engine's must equal both."""
    req0, _, _, _, _, want0 = base_trace(name)
    req, bounds, cut, corner, capacity, want, ora = shifted(name, where)
    check_universe(req["key"])
    assert want.tobytes() == want0.tobytes()
    decided = want["status"] == 0
    fast, slow = req_sides(req0), req_sides(req)
    assert fast.ordinary[decided].all() and fast.plain[decided].all()
    now = req["now_ns"]
    if where in ("a", "b"):
        assert now.min() >= (B61 if where == "a" else B62)
        assert not slow.ordinary[decided].any() and not slow.plain[decided].any()
    else:
        assert (now[:cut] < B61).all() and (now[cut:] >= B61).all()
        sides(slow.ordinary, decided, "ordinary_request")
        sides(slow.plain, decided, "plain outputs")
        if where == "c":
            assert cut not in bounds
        else:
            assert cut in bounds
    assert max(np.diff(bounds)) > 255
    assert_engine(req, bounds, want, ora, capacity, corner)


# ---------------------------------------------------------------------------------------------------------------
# the policy table of scenarios 2, 3 and 5, and batches of every run shape
# ---------------------------------------------------------------------------------------------------------------
def families():
    """count = 10^9, period = 2^k s: ei = 2^k ns exactly.  max_burst - 1 in {2^(60-k) - 1, 2^(60-k), 2^(60-k) + 1}
    puts dvt on 2^60 - 2^k, 2^60 and 2^60 + 2^k; the quantities put ei * q on the same three values, on 2^64 (only
    the hi term of the product) and just past it.  Then the u32 burst truncation: max_burst = 2^32 (factor 2^32 - 1)
    and 2^32 + 1 (factor 0).  All quantities fit an i32."""
    pols, qs = [], []
    for k in (34, 40, 46, 52):
        m = 1 << (60 - k)
        for mb1 in (m - 1, m, m + 1):
            pols.append((mb1 + 1, 10**9, 1 << k))
            qs.append([0, 1, m - 1, m, m + 1, 1 << (64 - k), (1 << (64 - k)) + 1])
    for mb in (2**32, 2**32 + 1):
        pols.append((mb, 10**9, 1 << 30))
        qs.append([0, 1, 2, 1 << 30])
    return pols, qs


FAM, FAM_Q = families()
C0 = len(FAM)                                  # CORNERS of test_compact_results_cpu
O0 = C0 + len(CORNERS)                         # traces.POLICIES
HUGE = O0 + len(traces.POLICIES)               # ei = 2^32, dvt = 2^63 - 2^32: q = 2^31 - 1 stores tat = I64_MAX
NEG = C0 + CORNERS.index((2, 1, I64_MAX))      # ei = dvt = -1: a large q stores a hugely negative tat
TABLE = np.array(FAM + CORNERS + [tuple(p) for p in traces.POLICIES.tolist()] + [(2**31, 10**9, 2**32)], np.int64)
P6_INDEX = O0 + 6                              # (1, 3, 3600)
SINGLES = 400
RUNS = [(2, 31)] * 40 + [(33, 255)] * 20 + [(256, 4095)] * 3 + [(4096, 6000)]
SINGLE_BASE, RUN_BASE, BG_KEYS = 1_000_000, 2_000_000, 5000
SHAPE_KEYS = list(range(SINGLE_BASE, SINGLE_BASE + SINGLES)) + list(range(RUN_BASE, RUN_BASE + len(RUNS)))


def family_rows(rng, n, group):
    """n rows of the scenario-2 families: (policy index, quantity)"""
    p = rng.integers(0, len(FAM), n)
    q = np.array([FAM_Q[i][rng.integers(len(FAM_Q[i]))] for i in p], np.int64)
    return p, q


def shaped_batch(rng, draw, n_background=20_000, n_toggle=300):
    """One batch: 400 singleton keys (pass B's commit-at-once), runs of 2-31 and 33-255 rows (warp chunks and
    chunk-crossing walks), three runs of 256-4095 (one CTA) and one of 4096-6000 (a cluster), each on its own key with
    rows from `draw(rng, n, group)`, mixed with ordinary keys (policy = key % 8) and a toggling max_burst = 1 key.
    The rows of one key keep the order `draw` gave them.  Returns (key, policy index, quantity)."""
    keys, pols, qs, pos = [], [], [], []

    def add(key, p, q, ordered=True):
        keys.append(np.full(len(p), key, np.uint64) if np.isscalar(key) else np.asarray(key, np.uint64))
        pols.append(np.asarray(p, np.int64))
        qs.append(np.asarray(q, np.int64))
        r = rng.random(len(p))
        pos.append(np.sort(r) if ordered else r)

    for i in range(SINGLES):
        add(SINGLE_BASE + i, *draw(rng, 1, i))
    for j, (lo, hi) in enumerate(RUNS):
        add(RUN_BASE + j, *draw(rng, int(rng.integers(lo, hi + 1)), SINGLES + j))
    bg = rng.integers(0, BG_KEYS, n_background).astype(np.uint64)
    add(bg, O0 + (bg % np.uint64(8)).astype(np.int64), traces.quantities(rng.integers(0, 2**63, n_background,
                                                                                        dtype=np.uint64)), False)
    add(TOGGLER, np.full(n_toggle, P6_INDEX), np.zeros(n_toggle))
    order = np.argsort(np.concatenate(pos), kind="stable")
    return np.concatenate(keys)[order], np.concatenate(pols)[order], np.concatenate(qs)[order]


def rows48(key, pol, q, now):
    req = np.zeros(len(key), traces.REQ_DTYPE)
    req["key"] = key
    p = TABLE[pol]
    req["max_burst"], req["count_per_period"], req["period"] = p[:, 0], p[:, 1], p[:, 2]
    req["quantity"] = q
    req["now_ns"] = now
    return req


def shaped_trace(seed, draw, clocks, small_at=None):
    """Batches of `shaped_batch` at the given clocks, plus (before batch `small_at`) one 200-row batch drawn from the
    same keys and rows: the one-CTA small-batch kernel."""
    rng = np.random.default_rng(seed)
    parts = []
    for t, now in enumerate(clocks):
        key, pol, q = shaped_batch(rng, draw)
        if t == small_at:
            pick = np.sort(rng.choice(len(key), 200, replace=False))
            parts.append(rows48(key[pick], pol[pick], q[pick], now))
        parts.append(rows48(key, pol, q, now))
    bounds = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).tolist()
    return np.concatenate(parts), bounds


def shape_corner_keys():
    return SHAPE_KEYS + [TOGGLER] + list(range(0, BG_KEYS, 97))


def assert_shapes(bounds):
    sizes = np.diff(bounds)
    assert (sizes <= 255).any() and (sizes > 255).any()


# ---------------------------------------------------------------------------------------------------------------
# scenario 2: request magnitudes straddling the bounds, at an ordinary clock
# ---------------------------------------------------------------------------------------------------------------
def test_request_magnitudes_straddling_the_bounds():
    """dvt and ei * q on 2^60 - 2^k, 2^60 and 2^60 + 2^k, ei * q on and past 2^64 and the u32 burst truncation, as
    singletons, warp-chunk runs, one-CTA runs and a cluster run of 4096 or more rows in batches of ~35 K rows at
    clocks near T0, mixed with ordinary keys; one 200-row batch of the same rows.  Allowed huge quantities leave
    TATs past 2^61 behind, which later rows read."""
    req, bounds = shaped_trace(32, family_rows, [T0 + t * S for t in range(3)], small_at=1)
    check_universe(req["key"])
    assert_shapes(bounds)
    ora = new_oracle(T0)
    want = ora.replay(req)
    s = req_sides(req)
    ok = want["status"] == 0
    sides(s.ordinary, ok, "ordinary_request")
    sides(s.dvt_big, ok, "dvt < 2^60")
    sides(s.inc_big, ok, "ei * q < 2^60")
    sides(s.hi_only, ok, "ei * q >= 2^64 with its low word below 2^60")
    sides(s.plain, ok, "plain outputs")
    assert (s.dvt == B60).any() and (s.dvt == B60 - (1 << 34)).any() and (s.dvt == B60 + (1 << 52)).any()
    assert want["allowed"][ok & s.inc_big].any() and not want["allowed"][ok & s.inc_big].all()
    tats = [ora.entry("k:%d" % k) for k in SHAPE_KEYS]
    assert any(e is not None and e[0] >= B61 for e in tats)
    assert_engine(req, bounds, want, ora, 10_000, shape_corner_keys())


# ---------------------------------------------------------------------------------------------------------------
# scenario 3: stored TATs beyond +-2^61 at an ordinary clock
# ---------------------------------------------------------------------------------------------------------------
def extreme_tat_rows(rng, n, group):
    """Even groups: a first row with the huge-dvt policy and q = 2^31 - 1 stores tat = I64_MAX (allowed: dvt = 2^63 -
    2^32), then ordinary rows.  Odd groups: ei = -1 with q in {2^62, I64_MAX} stores a tat below -2^61 with expiry
    I64_MAX, every 8th row and the last; ordinary rows in between.  Ordinary rows: policies 0-7, q in {0, 1, 2, 5}."""
    p = O0 + rng.integers(0, 8, n)
    q = rng.choice([0, 1, 1, 2, 5], n)
    if group % 2 == 0:
        p[0], q[0] = HUGE, I32_MAX
    else:
        d = np.unique(np.append(np.arange(0, n, 8), n - 1))
        p[d], q[d] = NEG, rng.choice([B62, I64_MAX], len(d))
    return p, q


def test_stored_tats_beyond_2_61():
    """Keys whose entries hold tat = I64_MAX or a tat below -2^61 (expiry clamped to I64_MAX: live for good), read by
    ordinary requests in the same batch and in the next ones, so that the |s_tat| < 2^61 term alone sends them to
    the saturating forms; singletons, warp-chunk, one-CTA and cluster (4096+ rows) runs in batches of ~35 K rows and
    one of 200."""
    clocks = [T0 + t * S for t in range(3)]
    req, bounds = shaped_trace(33, extreme_tat_rows, clocks, small_at=2)
    check_universe(req["key"])
    assert_shapes(bounds)
    ora = new_oracle(T0)
    want = np.empty(len(req), tc.RES_DTYPE)
    n_big = n_neg = n_read = 0
    for i, (a, b) in enumerate(zip(bounds, bounds[1:])):
        if i > 0:                       # entries left by the batches before, read by this batch's ordinary rows
            ent = {k: ora.entry("k:%d" % k) for k in SHAPE_KEYS}
            big = {k for k, e in ent.items() if e is not None and e[0] >= B61}
            neg = {k for k, e in ent.items() if e is not None and e[0] <= -B61 and e[1] == I64_MAX}
            n_big, n_neg = n_big + len(big), n_neg + len(neg)
            sl = req[a:b]
            s = req_sides(sl)
            on = np.isin(sl["key"], np.array(sorted(big | neg), np.uint64))
            n_read += int((on & s.ordinary).sum())
        want[a:b] = ora.replay(req[a:b])
    assert n_big > 0 and n_neg > 0 and n_read > 0, (n_big, n_neg, n_read)
    s = req_sides(req)
    ok = want["status"] == 0
    sides(s.ordinary, ok, "ordinary_request")
    assert_engine(req, bounds, want, ora, 10_000, shape_corner_keys())


# ---------------------------------------------------------------------------------------------------------------
# scenario 4: the top of the clock
# ---------------------------------------------------------------------------------------------------------------
def top_rows(rng, n, group):
    """q in {0, 1} with an ordinary policy per key (policy = group % 8)"""
    return np.full(n, O0 + group % 8), rng.choice([0, 1], n)


def top_trace():
    """Three shaped batches with per-row clocks rising through [I64_MAX - 10^12, I64_MAX] (the last quarter of the
    last batch, the tail of its cluster run included, exactly at I64_MAX), a 4500-row toggling key, and 1 % of the
    rows at clock 0 and 1 % at negative clocks scattered among them."""
    rng = np.random.default_rng(34)
    parts, lo, span = [], I64_MAX - 10**12, 10**12 // 3
    for t in range(3):
        key, pol, q = shaped_batch(rng, top_rows, n_background=10_000, n_toggle=4500)
        n = len(key)
        now = lo + t * span + np.sort(rng.integers(0, span, n))
        if t == 2:
            now[3 * n // 4:] = I64_MAX
        r = rng.random(n)
        now[r < 0.01] = 0
        now[(r >= 0.01) & (r < 0.02)] = rng.choice([-1, -5 * MS, -2**63], int(((r >= 0.01) & (r < 0.02)).sum()))
        parts.append(rows48(key, pol, q, now))
    return np.concatenate(parts), np.concatenate([[0], np.cumsum([len(p) for p in parts])]).tolist()


def replay_tracking(ora, req):
    """ora.replay row by row, also returning which allowed rows left their key's stored entry bit-for-bit unchanged"""
    out = np.zeros(len(req), tc.RES_DTYPE)
    same = np.zeros(len(req), bool)
    cols = [req[f].tolist() for f in ("key", "max_burst", "count_per_period", "period", "quantity", "now_ns")]
    for i, (k, b, c, p, q, now) in enumerate(zip(*cols)):
        key = "k:%d" % k
        before = ora.entry(key)
        r = ora.rate_limit(key, b, c, p, q, now)
        out[i]["status"], out[i]["allowed"] = r[0], r[1]
        out[i]["remaining"], out[i]["reset_after_ns"], out[i]["retry_after_ns"] = r[2:]
        same[i] = r[0] == 0 and r[1] and before is not None and before == ora.entry(key)
    return out, same


def test_top_of_the_clock():
    """Clocks up to exactly I64_MAX: `now + dvt` wraps, expiries clamp to I64_MAX and allowed requests that leave a
    clamped entry unchanged (q = 0) are common, which is what each kernel's "changed the state" choice must get
    right -- in cluster runs of 4096+ rows with q in {0, 1}, one-CTA runs, warp chunks, singletons and a toggling key
    in batches of ~25 K rows.  Clock-0 rows read TATs near I64_MAX; negative clocks come back INTERNAL without
    disturbing their neighbours.  Then sweeps at I64_MAX - 1 and at I64_MAX, as in the oracle."""
    req, bounds = top_trace()
    check_universe(req["key"])
    ora = new_oracle(I64_MAX - 10**12)
    want, same = replay_tracking(ora, req)
    assert (want["status"][req["now_ns"] < 0] == tc.INTERNAL).all()
    ok = want["status"] == 0
    s = req_sides(req)
    sides(s.ordinary, ok, "ordinary_request")
    sides(s.plain, ok, "plain outputs")
    sides(s.wraps, ok, "now + dvt past I64_MAX")
    top = ok & (req["now_ns"] == I64_MAX)
    assert top.sum() > 1000 and (ok & (req["now_ns"] == 0)).sum() > 100
    assert (top & (req["key"] == RUN_BASE + len(RUNS) - 1)).sum() > 100       # inside the cluster run
    run_rows = np.isin(req["key"], np.arange(RUN_BASE, RUN_BASE + len(RUNS), dtype=np.uint64))
    assert (same & run_rows).sum() > 1000, int((same & run_rows).sum())
    assert sum(1 for k in SHAPE_KEYS if (ora.entry("k:%d" % k) or (0, 0))[1] == I64_MAX) > 10
    st = assert_engine(req, bounds, want, ora, 10_000, shape_corner_keys())
    removed = []
    for now in (I64_MAX - 1, I64_MAX):
        removed.append(ora.force_sweep(now))
        assert st.sweep(now) == removed[-1]
        assert st.len() == ora.len()
        assert_entries(st, ora, shape_corner_keys())
    assert removed[0] > 0 and removed[1] > 0 and st.len() > 0, removed    # expiries past I64_MAX outlive both


def test_expiries_at_and_past_i64_max():
    """Regression case: an expiry past I64_MAX (the entry never expires) and one of exactly I64_MAX (live up to
    I64_MAX - 1) were both stored as I64_MAX, so at clock I64_MAX the first read as expired and a sweep removed it.
    Key 7: the huge-dvt policy with q = 2^31 - 1 stores tat = I64_MAX with an expiry past I64_MAX.  Keys 8 and 9: P0
    with q = 1 at I64_MAX - dvt stores an expiry of exactly I64_MAX.  Then q = 0 rows at I64_MAX - 1 and I64_MAX and
    sweeps at both clocks; one row per batch (the one-CTA small batch) and all rows in one batch with 300 others."""
    p0 = 5_940_000_000                                   # dvt of P0 = (100, 1000, 60)
    rows = rows48(np.array([7, 8, 9, 8, 7, 8], np.uint64), np.array([HUGE, O0, O0, O0, O0, O0]),
                  np.array([I32_MAX, 1, 1, 0, 0, 0]),
                  np.array([T0, I64_MAX - p0, I64_MAX - p0, I64_MAX - 1, I64_MAX, I64_MAX]))
    bg = rows48(np.arange(10, 310, dtype=np.uint64), np.full(300, O0), np.ones(300), I64_MAX - 10**9)
    for batch, bounds in ((rows, list(range(7))), (np.concatenate([rows[:3], bg, rows[3:]]), [0, 306])):
        ora = new_oracle(T0)
        want = ora.replay(batch)
        st, got = run_engine(batch, bounds, 1000)
        bad = first_mismatch(want, got, batch)
        assert bad is None, bad
        assert_counters(st, want, ora)
        assert ora.entry("k:7") == (I64_MAX, I64_MAX) and ora.entry("k:9") == (I64_MAX - p0, I64_MAX)
        for now in (I64_MAX - 1, I64_MAX):
            removed = ora.force_sweep(now)
            assert st.sweep(now) == removed and st.len() == ora.len()
            assert_entries(st, ora, [7, 8, 9] + list(range(10, 310)))
        assert ora.entry("k:7") is not None and ora.entry("k:9") is None    # past I64_MAX stays, I64_MAX goes


# ---------------------------------------------------------------------------------------------------------------
# scenario 5: compact requests, 32- and 16-byte results
# ---------------------------------------------------------------------------------------------------------------
class Compact:
    """one compact batch (the fields assert_pair reads)"""

    def __init__(self, key, pol, q, now):
        self.key, self.now = key, int(now)
        self.req16 = np.zeros(len(key), tc.REQ16_DTYPE)
        self.req16["key_hash"] = tc.hash_key_ids(key)
        self.req16["quantity"] = q
        self.req16["policy"] = pol


def compact_rows(rng, n, group):
    """scenario 2's family rows, and one row in four from the CORNERS policies with q in {0, 1, 5, 2^31 - 1, -1}"""
    p, q = family_rows(rng, n, group)
    c = rng.random(n) < 0.25
    p[c] = C0 + rng.integers(0, len(CORNERS), int(c.sum()))
    q[c] = rng.choice([0, 1, 5, I32_MAX, -1], int(c.sum()))
    return p, q


@functools.lru_cache(maxsize=None)
def compact_trace():
    rng = np.random.default_rng(35)
    batches = []
    for now in (B61 - 1, B61, B62, I64_MAX):
        key, pol, q = shaped_batch(rng, compact_rows, n_background=8000)
        if now == B62:
            pick = np.sort(rng.choice(len(key), 200, replace=False))
            batches.append(Compact(key[pick], pol[pick], q[pick], now))
        batches.append(Compact(key, pol, q, now))
    ora = new_oracle(B61 - 1)
    want, cur = [], []
    for b in batches:
        w, c = oracle_cur.replay_cur(ora, rows48(b.key, b.req16["policy"].astype(np.int64),
                                                b.req16["quantity"].astype(np.int64), b.now))
        want.append(w.view(tc.RES_DTYPE))
        cur.append(c)
    return batches, np.concatenate(want), np.concatenate(cur), ora


def test_compact_requests_both_result_widths():
    """The scenario-2 families and the CORNERS of test_compact_results_cpu as a policy table, i32 quantities and
    per-call clocks 2^61 - 1, 2^61, 2^62 and I64_MAX, on the batch shapes of scenario 2 (batches of ~20 K rows with a
    cluster run of 4096+ rows, and one of 200): the 16-byte rows carry the oracle's cur, status and allowed, and
    their expansion equals the 32-byte engine's rows and the oracle's."""
    batches, want, cur, ora = compact_trace()
    keys = np.concatenate([b.key for b in batches])
    check_universe(keys)
    assert_shapes(np.concatenate([[0], np.cumsum([len(b.key) for b in batches])]))
    pol = np.concatenate([b.req16["policy"] for b in batches]).astype(np.int64)
    now = np.concatenate([np.full(len(b.key), b.now) for b in batches])
    p = TABLE[pol]
    s = Sides(p[:, 0], p[:, 1], p[:, 2], np.concatenate([b.req16["quantity"] for b in batches]), now, cur)
    ok = want["status"] == 0
    sides(s.ordinary, ok, "ordinary_request")
    sides(s.plain, ok, "plain outputs")
    sides(s.hi_only, ok, "ei * q >= 2^64 with its low word below 2^60")
    sides(s.wraps, ok, "now + dvt past I64_MAX")
    table = np.zeros(len(TABLE), tc.POLICY_DTYPE)
    table["max_burst"], table["count_per_period"], table["period"] = TABLE.T
    out = {}
    for r16 in (False, True):
        st = tc.ManualStore(capacity=10_000, created_ns=0, max_batch=max(len(b.key) for b in batches))
        lim = tc.RateLimiter(st)
        lim.set_policies(table)
        st.track_denied(4096)
        out[r16] = (st, np.concatenate([lim.rate_limit_batch16(b.req16, b.now, compact_results=r16) for b in batches]))
    (st32, res32), (st16, res16) = out[False], out[True]
    assert_pair(batches, want, cur, res32, res16, st32, st16, ora, shape_corner_keys(), STAT_DECISIONS, table)
    assert_counters(st32, want, ora)


# ---------------------------------------------------------------------------------------------------------------
# scenario 6: pipelined submission and sweeping stores far past 2^62
# ---------------------------------------------------------------------------------------------------------------
def test_pipelined_submission_past_2_62():
    """The hot trace of scenario 1 from 2^62 (2^17-row batches with a ~5500-row cluster run and a 4500-row toggling
    key) through a paced 3-slot ring and back to back through submit_device / join, where the index-order overlap
    and the PEND bits apply."""
    import torch
    req, bounds, _, corner, capacity, want, ora = shifted("hot", "b")
    sizes = np.diff(bounds).tolist()
    ereq = engine_requests(req)

    st = tc.ManualStore(capacity=capacity, created_ns=0, max_batch=max(sizes))
    ring = tc.Ring(tc.RateLimiter(st), slots=3, slot_capacity=max(sizes))

    def fill(t, dst):
        dst[:] = ereq[bounds[t]:bounds[t + 1]]

    got = ring_run(ring, sizes, fill, lambda t: int(req["now_ns"][bounds[t]]))
    bad = first_mismatch(want, got, req)
    assert bad is None, "ring: " + bad
    assert_entries(st, ora, corner)
    assert_counters(st, want, ora)
    st.close()

    st = tc.ManualStore(capacity=capacity, created_ns=0, max_batch=max(sizes))
    lim = tc.RateLimiter(st)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    with torch.cuda.stream(stream):
        d_req = torch.from_numpy(ereq.view(np.uint8)).to(dev)
        d_res = torch.zeros(len(req) * 32, dtype=torch.uint8, device=dev)
        stream.synchronize()
        for a, b in zip(bounds, bounds[1:]):
            lim.submit_device(b - a, d_req[a * 48:].data_ptr(), d_res[a * 32:].data_ptr(), stream.cuda_stream)
        lim.join(stream.cuda_stream)
        stream.synchronize()
    got = d_res.cpu().numpy().view(tc.RES_DTYPE)
    bad = first_mismatch(want, got, req)
    assert bad is None, "submit_device: " + bad
    assert_entries(st, ora, corner)
    assert_counters(st, want, ora)


STORES = [(tc.PeriodicStore, oracle.PERIODIC), (tc.ProbabilisticStore, oracle.PROBABILISTIC),
          (tc.AdaptiveStore, oracle.ADAPTIVE)]


def sweeping_trace(where):
    """config1 (per-request clocks over ~60 days, 1 % foreign policies, invalid rows) with every clock moved past
    2^62, or so that it ends 0.1 s before I64_MAX; 4096-row batches, the last one starting within 30 s of the end
    (and over 60 s after the one before), so that a periodic store's last sweep schedules the next past I64_MAX."""
    req = traces.config1(n=100_000)
    now = req["now_ns"]
    created = T0
    delta = (B62 + 10**15 - T0) if where == "past_2_62" else (I64_MAX - 10**8 - int(now[-1]))
    req["now_ns"] += delta
    now = req["now_ns"]
    last = int(np.searchsorted(now, now[-1] - 30 * S))
    bounds = list(range(0, last, 4096)) + [last, len(req)]
    if where == "top":
        assert now[bounds[-3]] < now[last] - 60 * S
    return req, bounds, created + delta


@pytest.mark.parametrize("where", ["past_2_62", "top"])
@pytest.mark.parametrize("store_cls,okind", STORES, ids=["periodic", "probabilistic", "adaptive"])
def test_sweeping_stores_at_the_end_of_the_clock(store_cls, okind, where):
    """PeriodicStore, ProbabilisticStore and AdaptiveStore sweeping on their own policies (the host schedules
    `next_cleanup` in 128-bit arithmetic) with every clock and the creation time moved past 2^62, or to end within an
    hour of I64_MAX: the results equal the oracle store of the same kind, both sweep, and the decision counters
    agree.  Batches of 4096 rows (and a last one of a few rows).  The engine sweeps at batch boundaries, the oracle
    before any request, so `len` and `expired_hits` depend on when each swept; after one sweep of both at the last
    clock, `len` and every key's entry must agree."""
    req, bounds, created = sweeping_trace(where)
    check_universe(req["key"])
    ora = oracle.OracleStore(okind, capacity=1000, created_ns=created)
    want = ora.replay(req)
    ok = want["status"] == 0
    s = req_sides(req)
    assert not s.ordinary[ok].any()
    st, got = run_engine(req, bounds, 1000, store_cls, created)
    bad = first_mismatch(want, got, req)
    assert bad is None, bad
    e = st.stats()
    assert e["sweeps"] > 0 and ora.sweeps() > 0, (e["sweeps"], ora.sweeps())
    assert {f: e[f] for f in ("allowed", "denied", "errors")} == {
        "allowed": int(want["allowed"].sum()), "denied": int((ok & (want["allowed"] == 0)).sum()),
        "errors": int((~ok).sum())}
    last = int(req["now_ns"][-1])
    st.sweep(last)
    ora.force_sweep(last)
    assert st.len() == ora.len() > 0
    assert_entries(st, ora, list(range(1000)))
    if where == "top" and store_cls is tc.PeriodicStore:
        # the sweep at the last batch scheduled the next one past I64_MAX: none is due even at the end of the clock,
        # as in the oracle, whose next mutating operation at I64_MAX (a probe key's insert) does not sweep either
        n = st.stats()["sweeps"]
        assert st.policy_tick(I64_MAX) == 0 and st.stats()["sweeps"] == n
        n = ora.sweeps()
        ora.set_if_not_exists_with_ttl("probe", 0, 0, I64_MAX)
        assert ora.sweeps() == n
