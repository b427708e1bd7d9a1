"""Hot keys whose entries cycle through 2 to 6 states, against the oracle.

A run of LONG_RUN_MIN (256) to GIANT_RUN_MIN - 1 (4095) rows on one key gets one CTA of `decide_runs_kernel`, which
steps through it CTA_STRIDE (256) rows at a time; a longer run gets an 8-CTA cluster, CLUSTER_STRIDE (2048) rows at a
time (csrc/gcra_kernels.cuh, read by kernel_geometry.py).  After FSM_AFTER (4) state changes in a run the group switches to finite-state rounds: up to
FSM_K (4) candidate states, one nibble map per request, maps composed over warps, CTAs and the cluster's distributed
shared memory, a state outside the set published through `sm_pub` into a free candidate or over the round-robin
`victim`.  Before the switch, plain rounds go back to a known candidate with `Cands::find`.

The keys here rotate through K policies of one rate and different bursts at one clock (`cycle_steps` in
test_algorithm_model.py): exactly K states, with q = 1 rows that start a new family of states and denied rows that
change nothing.  Each scenario runs its key sequences through the kernel-faithful model (`fsm_rounds_kernel`) first,
both as the sort pipeline sees a run (all its rows, from the batch-start entry) and as the index-order pipeline's
residue tail sees it (the rows behind the first change, from the state that change committed), and asserts that the
events it is about happen in both: the set filled exactly, evictions of s0 and of states that come back, plain-round
returns, the switch in the middle of a stride, new states at the last and the first position of a stride.  Then every
row is compared bit-exact with ONE oracle store replaying the same rows in order, followed by the final entry of every
cycling key and the counters."""
import functools

import numpy as np
import pytest

import oracle
import oracle_cur
import throttlecrab_b200 as tc
import traces
from gpu_util import engine_requests, first_mismatch
from kernel_geometry import CLUSTER_STRIDE as CLUSTER, CTA_STRIDE as CTA, GIANT_RUN_MIN, LONG_RUN_MIN
from test_algorithm_model import CYCLE_POLICIES, cycle_state, cycle_steps, fsm_rounds_kernel, model_run, residue_view, \
    run_stride, sequential
from test_gpu_compact_results import assert_pair
from test_gpu_pipelined_runs import assert_counters, check_universe

pytestmark = pytest.mark.gpu

T0 = traces.T0
MS, S = 1_000_000, 1_000_000_000
NCYC = len(CYCLE_POLICIES)                       # policy indices 0..5: the cycle policies (max_burst 8 .. 3)
P_TOGGLE = NCYC                                  # max_burst = 1, q = 0: writes over an expired entry every other row
P_BG = NCYC + 1                                  # + key % 8: traces.POLICIES for the background keys
P_INVALID = P_BG + len(traces.POLICIES)          # max_burst = 0 (compact requests only)
POLICIES = np.array(CYCLE_POLICIES + [(1, 3, 3600)] + [tuple(p) for p in traces.POLICIES.tolist()] + [(0, 10, 60)],
                    np.int64)
TOGGLER, BG_KEYS = 999, 500


def interleave(rng, runs):
    """The rows of `runs` [(key, policy, quantity)] in one random order that keeps each key's rows in order."""
    lab = np.concatenate([np.full(len(p), i) for i, (_, p, _) in enumerate(runs)])
    rng.shuffle(lab)
    order = np.argsort(lab, kind="stable")
    key, pol, q = np.empty(len(lab), np.uint64), np.empty(len(lab), np.int64), np.empty(len(lab), np.int64)
    a = 0
    for k, p, x in runs:
        at = order[a:a + len(p)]
        key[at], pol[at], q[at] = k, p, x
        a += len(p)
    return key, pol, q


class Trace:
    """The batches of one scenario (key ids, policy indices, quantities, one clock each), the model of its cycling keys
    and the events of their hot runs in both views."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.batches, self.state, self.cycling = [], {}, set()
        self.events = {"sort": [], "residue": []}

    def add(self, runs, now, background=0, toggler=0):
        key, pol, q = interleave(self.rng, list(runs) + ([(TOGGLER, np.full(toggler, P_TOGGLE), np.zeros(toggler))]
                                                         if toggler else []))
        if background:
            bg = self.rng.integers(0, BG_KEYS, background).astype(np.uint64)
            at = self.rng.integers(0, len(key) + 1, background)
            key = np.insert(key, at, bg)
            pol = np.insert(pol, at, P_BG + (bg % np.uint64(8)).astype(np.int64))
            q = np.insert(q, at, self.rng.choice([0, 1, 1, 2, 5], background))
        for k, p, x in runs:
            self.cycling.add(int(k))
            run, s0 = model_run(p, x, now, CYCLE_POLICIES), self.state.get(int(k))
            for view, (r, rs0) in (("sort", (run, s0)), ("residue", residue_view(run, s0))):
                if len(key) >= LONG_RUN_MIN and r is not None and run_stride(len(r)):
                    self.events[view].append((int(k), len(r), rs0, fsm_rounds_kernel(r, rs0, run_stride(len(r)))[2]))
            self.state[int(k)] = sequential(run, s0)[1]
        self.batches.append((key, pol, q, int(now)))

    def rows(self, t=None):
        sel = self.batches if t is None else [self.batches[t]]
        parts = []
        for key, pol, q, now in sel:
            req = np.zeros(len(key), traces.REQ_DTYPE)
            req["key"] = key
            p = POLICIES[pol]
            req["max_burst"], req["count_per_period"], req["period"] = p[:, 0], p[:, 1], p[:, 2]
            req["quantity"], req["now_ns"] = q, now
            parts.append(req)
        return np.concatenate(parts)

    def hot(self, view, stride=None):
        return [e for e in self.events[view] if stride is None or run_stride(e[1]) == stride]

    def each_view(self, check):
        for view in ("sort", "residue"):
            check(view, self.hot(view))

    def oracle(self):
        req = self.rows()
        check_universe(np.concatenate([req["key"], np.arange(BG_KEYS), [TOGGLER]]))
        ora = oracle.OracleStore(oracle.PERIODIC, capacity=10_000, created_ns=T0, p0=10**9)
        return req, ora.replay(req), ora


def assert_entries(st, ora, keys):
    keys = sorted(keys)
    for k, h in zip(keys, tc.hash_key_ids(np.asarray(keys, np.uint64))):
        assert st.peek(int(h)) == ora.entry("k:%d" % k), k


def run_blocking(trace, want, ora):
    """Every batch of `trace` as one rate_limit_batch call (48-byte rows), then rows, entries and counters."""
    req = trace.rows()
    st = tc.ManualStore(capacity=10_000, created_ns=T0, max_batch=max(len(b[0]) for b in trace.batches))
    lim = tc.RateLimiter(st)
    ereq = engine_requests(req)
    got = np.empty(len(req), tc.RES_DTYPE)
    a = 0
    for b in trace.batches:
        lim.rate_limit_batch(ereq[a:a + len(b[0])], out=got[a:a + len(b[0])])
        a += len(b[0])
    bad = first_mismatch(want, got, req)
    assert bad is None, bad
    assert_entries(st, ora, trace.cycling | {TOGGLER})
    assert_counters(st, want, ora)
    return st


def stride_edges(events, stride):
    """stride positions (stride - 1, or 0 past the first stride) at which a finite-state round added a new state"""
    out = set()
    for _, n, _, ev in events:
        if run_stride(n) != stride:
            continue
        for p, fsm, kind in ev.changes:
            if fsm and kind == "new" and (p % stride == stride - 1 or (p % stride == 0 and p > 0)):
                out.add(p % stride)
    return out


# ---------------------------------------------------------------------------------------------------------------
# cycle length x run shape
# ---------------------------------------------------------------------------------------------------------------
# around 1, 2 and 3 strides of a CTA (LONG_RUN_MIN - 1 .. + 1: warp chunks, the first CTA run, its first stride edge)
# and of a cluster (one CTA run of 8 CTA strides; GIANT_RUN_MIN - 1 .. + 1: the CTA / cluster boundary and the second
# cluster stride edge; GIANT_RUN_MIN + CLUSTER_STRIDE - 1 .. + 1: the third)
LENGTHS = sorted(n for n in {m * s + d for s in (CTA, CLUSTER) for m in (1, 2, 3) for d in (-1, 0, 1)}
                 | {LONG_RUN_MIN + d for d in (-1, 0, 1)} | {GIANT_RUN_MIN + d for d in (-1, 0, 1)}
                 | {GIANT_RUN_MIN + CLUSTER + d for d in (-1, 0, 1)} if n >= LONG_RUN_MIN - 1)
LEAD = 5                  # cycle policy of the first row of a K <= 3 key: a state outside its cycle


@functools.lru_cache(maxsize=None)
def shape_trace(k):
    """For every length L, a key with L rows and one with L + 1 (the index-order residue is one row shorter: both
    views have a run of exactly L rows).  K <= 3: fresh keys whose first row (policy LEAD) creates a state outside the
    cycle, so s0 differs from every cycle state in both views.  K >= 4: keys whose entry a first batch at the same clock
    put on the state of cycle policy 0, then a rotation from policy 1.  K >= 5 adds keys in random order.  2 % of the
    rows (never the first) are denied."""
    tr = Trace(100 + k)
    now = T0 + S
    base = 1_000_000 * k
    runs = []
    for j, n in enumerate([L + e for L in LENGTHS for e in (0, 1)]):
        pol, q = cycle_steps(n, k, start=1 if k >= 4 else 0, deny_at=1 + tr.rng.choice(n - 1, n // 50, replace=False))
        if k <= 3:
            pol[0] = LEAD
        runs.append((base + j, pol, q))
    if k >= 5:
        for j, n in enumerate([700, 2500, GIANT_RUN_MIN - 1, GIANT_RUN_MIN + 4, 3 * CLUSTER + 1]):
            runs.append((base + 100 + j, *cycle_steps(n, k, rng=tr.rng)))
    if k >= 4:
        pre = [(key, np.zeros(1, np.int64), np.zeros(1, np.int64)) for key, _, _ in runs]
        tr.add(pre, now, toggler=4)
    tr.add(runs, now, background=3000, toggler=64)

    cycle = {cycle_state(c, 0, now) for c in range(k)}

    def check(view, hot):
        assert {n for _, n, _, _ in hot} >= set(LENGTHS[1:]), view
        assert all(ev.fsm_rounds > 0 for _, _, _, ev in hot), view
        rot = [ev for key, _, _, ev in hot if key < base + 100]
        if k <= 3:
            assert all(s0 not in cycle for _, _, s0, _ in hot), view
            # sort view: no entry, the LEAD state, K cycle states; residue view: from the LEAD state
            n_states = k + 2 if view == "sort" else k + 1
        else:
            n_states = k
        assert {ev.max_nc for ev in rot} == {min(n_states, 4)}, view
        assert all((ev.evictions > 0) == (n_states > 4) for ev in rot), view
        if k == 4:
            assert all(ev.s0_returns > 0 for ev in rot), view
        if n_states > 4:
            assert all(ev.s0_evicted for ev in rot), view
        if k >= 5:
            assert all(ev.evicted_returns > 0 for ev in rot), view
            assert any(ev.cur_evicted > 0 for _, _, _, ev in hot), view
            assert stride_edges(hot, CTA) == {CTA - 1, 0} and stride_edges(hot, CLUSTER) == {CLUSTER - 1, 0}, view
    tr.each_view(check)
    return tr


@pytest.mark.parametrize("k", [2, 3, 4, 5, 6])
def test_cycle_length_by_run_shape(k):
    """K-cycles at run lengths 255 (warp chunks), 256-257 and 511-513, 767-769 (one CTA, around one to three strides),
    2047-2049 (one CTA, eight strides), 4095-4097 (the CTA / cluster boundary, two cluster strides) and 6143-6145 (three
    cluster strides), among 3000 background rows and a toggling key.  K = 4 fills the candidate set exactly and keeps coming back to s0; K = 5 and 6 evict s0, then evict
    every state they come back to, evict the candidate `cur` points at (random order) and create new states at both
    edges of a stride."""
    tr = shape_trace(k)
    req, want, ora = tr.oracle()
    run_blocking(tr, want, ora)


# ---------------------------------------------------------------------------------------------------------------
# the switch at the 4th change, and new states at the edges of a stride
# ---------------------------------------------------------------------------------------------------------------
def schedule(n, k, changes, seq, q1_at=()):
    """Rows holding one cycle policy at a time: seq[i] from row changes[i] on, then (from the last change) a plain
    rotation through the first k policies; q = 1 rows (new states) at q1_at."""
    pol, q = cycle_steps(n, k, start=seq[-1], q1_at=q1_at)
    rot = pol[changes[-1]:].copy()
    for a, b, c in zip(changes, list(changes[1:]) + [n], seq):
        pol[a:b] = c
    pol[changes[-1]:] = rot[:n - changes[-1]]
    return pol, q


@functools.lru_cache(maxsize=None)
def switch_trace():
    """Keys whose first changes go back and forth between two states (plain rounds back to a known candidate, s0 among
    them for the keys with an entry), whose 4th change falls inside a stride or on either side of its edge, and whose
    q = 1 rows create new states at the two rows either side of the first stride edge (254-257 in a CTA, 2046-2049 in
    a cluster), then again a stride later.  The first row
    of every key changes its state, so the residue tail sees the same positions one row earlier."""
    tr = Trace(7)
    now = T0 + 2 * S
    runs = []
    for j, (n, chg, k) in enumerate([
            (1500, [0, 37, 90, 200, 230], 4),            # the 4th change in the middle of the first stride
            (1500, [0, 1, 2, CTA - 1, CTA + 88], 3),       # ... on its last row
            (1500, [0, 1, 2, CTA, CTA + 88], 4),           # ... on the first row of the second stride
            (1200, [0, 5, 9, 14, 20], 2),
            (9000, [0, 500, 1000, 1500, 1750], 4),       # cluster: the 4th change in the middle of the first stride
            (9000, [0, 1, 2, CLUSTER - 1, CLUSTER + 104], 3),
            (9000, [0, 1, 2, CLUSTER, CLUSTER + 104], 2)]):
        stride = run_stride(n)
        edges = [e + d for e in (stride, 2 * stride) for d in (-2, -1, 0, 1)]
        for entry in (False, True):
            seq = [1, 0, 1, 0, 1] if entry else [0, 1, 0, 1, 0]
            runs.append((2_000_000 + 2 * j + entry, *schedule(n, k, chg, seq, q1_at=edges)))
    tr.add([(key, np.zeros(1, np.int64), np.zeros(1, np.int64)) for key, _, _ in runs if key & 1], now, toggler=4)
    tr.add(runs, now, background=2000, toggler=64)

    def check(view, hot):
        assert any(ev.switch_mid_stride for _, n, _, ev in hot if run_stride(n) == CTA), view
        assert any(ev.switch_mid_stride for _, n, _, ev in hot if run_stride(n) == CLUSTER), view
        assert any(ev.s0_returns > 0 and ev.plain_returns >= 2 for _, _, _, ev in hot), view
        assert stride_edges(hot, CTA) == {CTA - 1, 0} and stride_edges(hot, CLUSTER) == {CLUSTER - 1, 0}, view
    tr.each_view(check)
    return tr


def test_switch_at_the_fourth_change_and_stride_edges():
    """Plain rounds back to known states (s0 included) up to the 4th change; the switch to finite-state rounds in the
    middle of a stride, on its last row and on the first row of the next; new states created by the last thread of a
    stride and by the first thread of the next, in one CTA (255 / 256) and in a cluster (2047 / 2048)."""
    tr = switch_trace()
    req, want, ora = tr.oracle()
    run_blocking(tr, want, ora)


# ---------------------------------------------------------------------------------------------------------------
# more runs than one launch has groups
# ---------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def many_runs_trace():
    """150 one-CTA runs (258-700 rows; the one-CTA kernel has one CTA per SM, 132) and 20 cluster runs (4098-4400
    rows; the cluster kernel has 16 clusters), each key with its own K (2-6), start, order and entry, twice: the groups
    loop over their items and carry `par` from one run to the next."""
    tr = Trace(9)
    now = T0 + 3 * S
    spec = []
    for j in range(170):
        n = int(tr.rng.integers(258, 701) if j < 150 else tr.rng.integers(4098, 4401))
        spec.append((3_000_000 + j, n, int(tr.rng.integers(2, 7)), bool(tr.rng.random() < 0.3)))
    tr.add([(key, np.zeros(1, np.int64), np.zeros(1, np.int64)) for key, _, _, _ in spec[::2]], now, toggler=4)
    for rep in range(2):
        runs = []
        for key, n, k, rnd in spec:
            runs.append((key, *cycle_steps(n, k, start=int(tr.rng.integers(k)), rng=tr.rng if rnd else None,
                                           q1_at=tr.rng.choice(n, 2, replace=False),
                                           deny_at=tr.rng.choice(n, n // 40, replace=False))))
        tr.add(runs, now + rep * MS, background=1000, toggler=64)

    def check(view, hot):
        assert len(tr.hot(view, CTA)) >= 2 * 133 and len(tr.hot(view, CLUSTER)) >= 2 * 17, view
        assert sum(ev.fsm_rounds > 0 for _, _, _, ev in hot) > 0.9 * len(hot), view
        assert sum(ev.evictions > 0 for _, _, _, ev in hot) > 0.3 * len(hot), view
    tr.each_view(check)
    return tr


def test_many_runs_in_one_launch():
    """More one-CTA and cluster runs than their launches have groups, in two batches of the same keys."""
    tr = many_runs_trace()
    req, want, ora = tr.oracle()
    run_blocking(tr, want, ora)


# ---------------------------------------------------------------------------------------------------------------
# request and result formats, back-to-back pipelined batches, small batches and warp chunks
# ---------------------------------------------------------------------------------------------------------------
def mixed_runs(tr, base, lengths, q1=2):
    """one key per (length, K) pair, random K-cycle order for odd K"""
    runs = []
    for j, n in enumerate(lengths):
        k = 2 + j % 5
        runs.append((base + j, *cycle_steps(n, k, start=int(tr.rng.integers(k)), rng=tr.rng if k % 2 else None,
                                            q1_at=tr.rng.choice(n, min(q1, n), replace=False),
                                            deny_at=tr.rng.choice(n, n // 30, replace=False))))
    return runs


@functools.lru_cache(maxsize=None)
def compact_trace():
    """Three batches at 1 ms steps: 10 one-CTA runs and 5 cluster runs of cycling keys (the same keys in each batch),
    background keys, a toggling key, and rows with a negative quantity, the invalid policy and a policy index beyond
    the table."""
    tr = Trace(11)
    lengths = [300, 511, 513, 1000, 2000, 257, 600, 900, 3000, 4095, 4096, 4097, 5000, 6000, 8193]
    for t in range(3):
        tr.add(mixed_runs(tr, 4_000_000, lengths), T0 + 4 * S + t * MS, background=3000, toggler=64)
    tr.each_view(lambda view, hot: (len(hot) >= 40 and sum(ev.fsm_rounds > 0 for *_, ev in hot) >= 30
                                    and sum(ev.evictions > 0 for *_, ev in hot) >= 10) or pytest.fail(view))
    return tr


class Batch16:
    def __init__(self, key, pol, q, now):
        self.key, self.now = key, now
        self.req16 = np.zeros(len(key), tc.REQ16_DTYPE)
        self.req16["key_hash"] = tc.hash_key_ids(key)
        self.req16["quantity"], self.req16["policy"] = q, pol


def test_compact_requests_both_result_widths():
    """16-byte requests (policy index, one clock per call) with 32-byte results and with 16-byte results (`cur`): the
    hot-run kernels' R16 writes.  Every 16-byte row carries the oracle's cur; expanded, it equals the 32-byte row."""
    tr = compact_trace()
    rng = np.random.default_rng(12)
    batches, want, cur = [], [], []
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=10_000, created_ns=T0, p0=10**9)
    for key, pol, q, now in tr.batches:
        pol, q = pol.copy(), q.copy()
        edge = rng.choice(len(key), 60, replace=False)
        q[edge[:20]] = -1                                    # GCRA_NEGATIVE_QUANTITY
        pol[edge[20:40]] = P_INVALID                          # GCRA_INVALID_RATE_LIMIT
        pol[edge[40:]] = 2**32 - 1                            # beyond the table: GCRA_INTERNAL
        far = pol >= len(POLICIES)
        batches.append(Batch16(key, pol, q, now))
        req = np.zeros(int((~far).sum()), traces.REQ_DTYPE)
        req["key"] = key[~far]
        p = POLICIES[pol[~far]]
        req["max_burst"], req["count_per_period"], req["period"] = p[:, 0], p[:, 1], p[:, 2]
        req["quantity"], req["now_ns"] = q[~far], now
        w, c = np.zeros(len(key), tc.RES_DTYPE), np.zeros(len(key), np.int64)
        w["status"][far] = tc.INTERNAL
        o, c[~far] = oracle_cur.replay_cur(ora, req)
        w[~far] = o.view(tc.RES_DTYPE)
        want.append(w)
        cur.append(c)
    want, cur = np.concatenate(want), np.concatenate(cur)
    check_universe(np.concatenate([tr.rows()["key"], np.arange(BG_KEYS), [TOGGLER]]))
    table = np.zeros(len(POLICIES), tc.POLICY_DTYPE)
    table["max_burst"], table["count_per_period"], table["period"] = POLICIES.T
    out = {}
    for r16 in (False, True):
        st = tc.ManualStore(capacity=10_000, created_ns=T0, max_batch=max(len(b.key) for b in batches))
        lim = tc.RateLimiter(st)
        lim.set_policies(table)
        st.track_denied(4096)
        out[r16] = (st, np.concatenate([lim.rate_limit_batch16(b.req16, b.now, compact_results=r16) for b in batches]))
    (st32, res32), (st16, res16) = out[False], out[True]
    assert_pair(batches, want, cur, res32, res16, st32, st16, ora, sorted(tr.cycling | {TOGGLER}), table=table)


@functools.lru_cache(maxsize=None)
def pipelined_trace():
    """24 batches at 1 ms steps, each with the same cycling keys (runs of 257-3000 and 4097-6000 rows, no q = 1 rows:
    the states stay those of one family) among background keys and a toggling key: each batch starts the keys from the
    cycle state the previous one left."""
    tr = Trace(13)
    for t in range(24):
        lengths = [int(x) for x in tr.rng.integers(257, 3001, 8)] + [int(x) for x in tr.rng.integers(4097, 6001, 2)]
        tr.add(mixed_runs(tr, 5_000_000, lengths, q1=0), T0 + 5 * S + t * MS, background=2000, toggler=64)
    tr.each_view(lambda view, hot: (len(hot) >= 200 and sum(ev.fsm_rounds > 0 for *_, ev in hot) >= 200
                                    and sum(ev.evictions > 0 for *_, ev in hot) >= 50) or pytest.fail(view))
    return tr


def test_back_to_back_submit_device():
    """The batches submitted back to back with `submit_device` and joined at the end: in the index-order pipeline the
    cycling keys are the residue of every batch, and PEND deferral carries them from one tail to the next."""
    import torch
    tr = pipelined_trace()
    req, want, ora = tr.oracle()
    ereq = engine_requests(req)
    sizes = [len(b[0]) for b in tr.batches]
    off = np.concatenate([[0], np.cumsum(sizes)])
    st = tc.ManualStore(capacity=10_000, created_ns=T0, max_batch=max(sizes))
    lim = tc.RateLimiter(st)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    with torch.cuda.stream(stream):
        d_req = torch.from_numpy(ereq.view(np.uint8)).to(dev)
        d_res = torch.zeros(len(req) * 32, dtype=torch.uint8, device=dev)
        stream.synchronize()
        for a, b in zip(off[:-1], off[1:]):
            lim.submit_device(int(b - a), d_req[int(a) * 48:].data_ptr(), d_res[int(a) * 32:].data_ptr(),
                              stream.cuda_stream)
        lim.join(stream.cuda_stream)
        stream.synchronize()
    got = d_res.cpu().numpy().view(tc.RES_DTYPE)
    bad = first_mismatch(want, got, req)
    assert bad is None, bad
    assert_entries(st, ora, tr.cycling | {TOGGLER})
    assert_counters(st, want, ora)


@functools.lru_cache(maxsize=None)
def small_trace():
    """A 200-row batch (the one-CTA small-batch kernel) with three cycling keys, then two batches of warp-chunk runs
    of 2-255 rows, across and along the 32-row chunks, with every K."""
    tr = Trace(15)
    tr.add(mixed_runs(tr, 6_000_000, [60, 70, 50], q1=1), T0 + 6 * S, background=16, toggler=4)
    lengths = [2, 3, 31, 32, 33, 63, 64, 65, 95, 100, 127, 128, 129, 200, 254, 255]
    for t in range(2):
        tr.add(mixed_runs(tr, 6_000_100, lengths, q1=1), T0 + 6 * S + (t + 1) * MS, background=3000, toggler=64)
    assert not tr.events["sort"] and not tr.events["residue"]
    return tr


def test_small_batch_and_warp_chunks():
    """Cycling keys in the small-batch kernel and in warp chunks, where no run reaches the hot-run kernels."""
    tr = small_trace()
    req, want, ora = tr.oracle()
    run_blocking(tr, want, ora)
