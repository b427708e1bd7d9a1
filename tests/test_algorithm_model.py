"""CPU model of the two exactness arguments the decide kernels rest on (DESIGN.md section 4), checked against
plain sequential application on random runs of requests on ONE key:

  speculate-and-commit   every pending request is evaluated against the run's current state; everything up to
                         and including the first state-changing request is final; the rest re-evaluates.
  finite-state rounds    the last K distinct states are candidates; each request is a map candidate -> candidate
                         (or NEW); an inclusive scan of the composed maps gives every request its true input
                         state; a round is repeated only when a request creates a state outside the candidates.

This is a model of the ALGORITHM (the CUDA kernels are tested against the oracle on the GPU); it documents why
the parallel evaluation reproduces the sequential semantics bit for bit, including keys that toggle between
states (max_burst = 1 with zero-quantity requests).

`fsm_rounds_kernel` follows the hot-run kernel itself (plain rounds first, its candidate bookkeeping, its strides) and
reports which of its events a run reaches; tests/test_gpu_fsm_cycles.py uses it to prove that its key sequences
reach the events they are meant to, then runs them on the GPU against the oracle."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import kernel_geometry as kg
from test_oracle_vs_python_model import I64_MAX, U64, clamp, derive, wrap64, _tdiv

NEW = "new"


def decide(state, req):
    """state = (tat, expiry) or None; req = (now, ei, dvt, q) -> (allowed, new_state, outputs)"""
    now, ei, dvt, q = req
    live = state is not None and state[1] > now
    tat = max(state[0], clamp(now - dvt)) if live else clamp(now - ei)
    new_tat = clamp(tat + clamp(ei * q))
    allow_at = clamp(new_tat - dvt)
    allowed = now >= allow_at
    new_state = state
    if allowed:
        ttl = clamp(clamp(new_tat - now) + dvt) % U64
        new_state = (new_tat, min(now + ttl, I64_MAX))
    cur = new_tat if allowed else tat
    room = clamp(wrap64(now + dvt) - cur)
    out = (allowed, max(_tdiv(room, ei), 0) if ei > 0 else 0, max(clamp(clamp(cur - now) + dvt), 0),
           0 if allowed else max(clamp(allow_at - now), 0))
    return allowed, new_state, out


def sequential(run, s0):
    s, outs = s0, []
    for r in run:
        _, s, o = decide(s, r)
        outs.append(o)
    return outs, s


def speculate_commit(run, s0, width=32):
    outs, s = [None] * len(run), s0
    for base in range(0, len(run), width):
        pending = list(range(base, min(base + width, len(run))))
        while pending:
            ev = {i: decide(s, run[i]) for i in pending}
            first = next((i for i in pending if ev[i][1] != s), None)      # first state-changing request
            final = [i for i in pending if first is None or i <= first]
            for i in final:
                outs[i] = ev[i][2]
            if first is not None:
                s = ev[first][1]
            pending = [i for i in pending if i not in final]
    return outs, s


def fsm_rounds(run, s0, k=4, stride=16):
    outs = [None] * len(run)
    cands, cur, victim = [s0], 0, 0
    for base in range(0, len(run), stride):
        pending = list(range(base, min(base + stride, len(run))))
        while pending:
            maps = {}
            for i in pending:                                    # request -> map over the candidate indices
                m = []
                for c, cs in enumerate(cands):
                    ns = decide(cs, run[i])[1]
                    m.append(c if ns == cs else (cands.index(ns) if ns in cands else NEW))
                maps[i] = m
            idx, true_in = cur, {}
            for i in pending:                                    # what the inclusive prefix scan computes
                true_in[i] = idx
                if idx != NEW:
                    idx = maps[i][idx]
            done = [i for i in pending if true_in[i] != NEW]
            creator = None
            for i in done:
                _, ns, o = decide(cands[true_in[i]], run[i])
                outs[i] = o
                if maps[i][true_in[i]] == NEW:
                    creator = (i, ns)
            if creator is None:
                cur = idx
            else:                                                # a state outside the candidate set was created
                if len(cands) < k:
                    cands.append(creator[1])
                    cur = len(cands) - 1
                else:
                    cands[victim] = creator[1]
                    cur, victim = victim, (victim + 1) % k
            pending = [i for i in pending if i not in done]
    return outs, cands[cur]


# ---------------------------------------------------------------------------------------------------------
# decide_runs_kernel (csrc/gcra_kernels.cuh) step by step: plain rounds until FSM_AFTER state changes, then
# finite-state rounds over nibble maps; Cands::find (last match among the first nc), the round-robin victim,
# one stride of the group (kernel_geometry: CTA_STRIDE rows for a CTA, CLUSTER_STRIDE for a cluster) after another
# ---------------------------------------------------------------------------------------------------------
FSM_NEW = 0xF


def fsm_ident(k):
    return sum(c << (4 * c) for c in range(k))


def fsm_compose(f, g, k):
    """fsm_compose: first f, then g (nibble maps over k candidates; FSM_NEW stays FSM_NEW)"""
    gg = g | (0xF << 60)
    return sum(((gg >> (4 * ((f >> (4 * c)) & 0xF))) & 0xF) << (4 * c) for c in range(k))


class Events:
    """What a run made the kernel do: the largest nc, the evictions (of s0, of the candidate `cur` pointed at),
    insertions of a state evicted earlier in the run, plain-round returns to a known candidate, changes back to the
    candidate holding s0, the run position of every state change with its round kind and outcome, the run position of
    the change that switches to finite-state rounds, and the number of finite-state rounds."""

    def __init__(self):
        self.max_nc, self.evictions, self.s0_evicted, self.cur_evicted = 1, 0, False, 0
        self.evicted_returns, self.plain_returns, self.s0_returns, self.fsm_rounds = 0, 0, 0, 0
        self.changes = []           # (run position, finite-state round?, "new" | "known")
        self.switch_pos = None      # run position of the FSM_AFTER-th change
        self.switch_mid_stride = False   # ... with rows of its stride still pending: a finite-state round follows

    def new_at(self, stride):
        """stride positions of the requests whose state joined the candidate set"""
        return {p % stride for p, _, kind in self.changes if kind == "new"}


def fsm_rounds_kernel(run, s0, stride, k=4, fsm_after=4):
    """The hot-run kernel on one run: (outputs, final state, Events).  Each round evaluates the pending requests
    of the stride in order until the first one that leaves the candidate set (plain rounds: the first one that
    changes the state); the requests before it and itself are final, exactly what the kernel's min-reduction or
    prefix scan of composed maps decides.  The requests behind it wait for the next round, whose maps the kernel
    computes afresh, so evaluating them now would change nothing."""
    cache = {}

    def dec(s, r):
        v = cache.get((s, r))
        if v is None:
            v = cache[(s, r)] = decide(s, r)
        return v

    outs = [None] * len(run)
    cands = [s0] * k
    nc, cur, victim, n_changes = 1, 0, 0, 0
    ev, evicted = Events(), set()

    def find(s):                                             # Cands::find: the LAST match among the first nc
        j = FSM_NEW
        for c in range(k):
            if c < nc and cands[c] == s:
                j = c
        return j

    ident = fsm_ident(k)
    for base in range(0, len(run), stride):
        pending = list(range(base, min(base + stride, len(run))))
        while True:
            fsm = n_changes >= fsm_after
            ev.fsm_rounds += fsm
            creator, done = None, 0
            if not fsm:                                      # plain round: up to the first state change
                s = cands[cur]
                for i in pending:
                    done += 1
                    outs[i] = dec(s, run[i])[2]
                    if dec(s, run[i])[1] != s:
                        creator, cin = i, cur
                        break
            else:                                            # finite-state round: maps and their prefix
                excl = ident
                for i in pending:
                    m = 0
                    for c in range(k):
                        o = FSM_NEW
                        if c < nc:
                            ns = dec(cands[c], run[i])[1]
                            o = c if ns == cands[c] else find(ns)
                        m |= o << (4 * c)
                    cin = (excl >> (4 * cur)) & 0xF          # this request's true input candidate
                    done += 1
                    outs[i] = dec(cands[cin], run[i])[2]
                    to = (m >> (4 * cin)) & 0xF
                    ev.s0_returns += to not in (FSM_NEW, cin) and cands[to] == s0
                    excl = fsm_compose(excl, m, k)
                    if (excl >> (4 * cur)) & 0xF == FSM_NEW:
                        creator = i
                        break
            pending = pending[done:]
            if creator is None:
                if fsm:
                    cur = (excl >> (4 * cur)) & 0xF
                break
            ps = dec(cands[cin], run[creator])[1]
            v = find(ps)
            if v == FSM_NEW:
                if nc < k:
                    v, nc = nc, nc + 1
                else:
                    v, victim = victim, (victim + 1) % k
                    ev.evictions += 1
                    ev.s0_evicted |= cands[v] == s0
                    ev.cur_evicted += v == cur
                    evicted.add(cands[v])
                ev.evicted_returns += ps in evicted
                cands[v] = ps
                ev.changes.append((creator, fsm, "new"))
            else:
                ev.plain_returns += 1
                ev.s0_returns += cands[v] == s0
                ev.changes.append((creator, fsm, "known"))
            ev.max_nc = max(ev.max_nc, nc)
            cur = v
            n_changes += 1
            if n_changes == fsm_after:
                ev.switch_pos, ev.switch_mid_stride = creator, len(pending) > 0
    return outs, cands[cur], ev


def residue_view(run, s0):
    """The run as the index-order pipeline's residue tail decides it: the rows behind the first state change, from
    the state that change committed (pass C).  (None, None) when nothing changes: no residue."""
    s = s0
    for i, r in enumerate(run):
        ns = decide(s, r)[1]
        if ns != s:
            return run[i + 1:], ns
    return None, None


# K-cycles (DESIGN.md section 5): policies with one rate (10 per 60 s) and max_burst 8, 7, ..., 3.  With a live entry
# whose tat is at or above now, a q = 0 request with dvt = ei * (max_burst - 1) is allowed when tat <= now + dvt, leaves
# tat and sets the expiry to tat + dvt: rotating through K of these policies at one clock walks the entry through
# exactly K states.  A q = 1 request moves tat up by ei (a new family of states); q = DENY is never allowed.
CYCLE_POLICIES = [(8 - c, 10, 60) for c in range(6)]
DENY = 40


def cycle_steps(n, k, start=0, rng=None, q1_at=(), deny_at=()):
    """(policy index into CYCLE_POLICIES, quantity) of n rows rotating through the first k policies from `start`
    (or, with `rng`, drawing each row's policy at random among them), with q = 1 rows and denied rows at the given
    positions."""
    pol = (start + np.arange(n)) % k if rng is None else rng.integers(0, k, n)
    q = np.zeros(n, np.int64)
    q[list(q1_at)] = 1
    q[list(deny_at)] = DENY
    return pol.astype(np.int64), q


def model_run(pol, q, now, policies=CYCLE_POLICIES):
    der = [derive(*p) for p in policies]
    return [(int(t), der[p][1], der[p][2], int(x)) for p, x, t in zip(pol.tolist(), q.tolist(), np.broadcast_to(now, len(pol)).tolist())]


def run_stride(n):
    """the stride of the group a run of n rows gets: None (warp chunks), CTA_STRIDE (one CTA) or CLUSTER_STRIDE (one
    cluster)"""
    return None if n < kg.LONG_RUN_MIN else kg.CTA_STRIDE if n < kg.GIANT_RUN_MIN else kg.CLUSTER_STRIDE


# The hot-run geometry this model, its event proofs and the GPU scenarios built on them (test_gpu_fsm_cycles.py,
# test_gpu_hot_run_listing.py) were written for.  A change of the kernels' geometry fails the test below: the
# positions those scenarios call stride edges, and the events they are proved to reach, have to be looked at again.
MODEL_GEOMETRY = {"LONG_THREADS": 256, "CLUSTER_CTAS": 8, "LONG_RUN_MIN": 256, "GIANT_RUN_MIN": 4096, "SMALL_MAX": 255}


def test_model_geometry_is_the_kernels():
    """The model's strides and thresholds are the ones gcra_kernels.cuh compiles with, and the hot-run kernel and its
    launches step through a run by those strides."""
    assert kg.GEOMETRY == MODEL_GEOMETRY
    assert (kg.CTA_STRIDE, kg.CLUSTER_STRIDE) == (256, 2048)
    lo, hi = kg.LONG_RUN_MIN, kg.GIANT_RUN_MIN
    assert [run_stride(n) for n in (kg.SMALL_MAX, lo - 1, lo, hi - 1, hi, 1 << 20)] == \
        [None, None, kg.CTA_STRIDE, kg.CTA_STRIDE, kg.CLUSTER_STRIDE, kg.CLUSTER_STRIDE]
    assert kg.SMALL_MAX < lo < hi and kg.CLUSTER_STRIDE == kg.CLUSTER_CTAS * kg.LONG_THREADS
    with open(kg.HEADER) as f:
        src = f.read()
    for line in ("constexpr u32 STRIDE = CTAS * LONG_THREADS;", "const u32 gpos = rank * LONG_THREADS + tid;",
                 "const u32 hot_at = run_start + LONG_RUN_MIN - 1;",
                 "const bool giant = end - run_start >= GIANT_RUN_MIN;"):
        assert line in src, line
    # the model's rounds at the parsed strides: a run one row past two strides ends in a one-row stride
    for stride in (kg.CTA_STRIDE, kg.CLUSTER_STRIDE):
        pol, q = cycle_steps(2 * stride + 1, 5)
        run = model_run(pol, q, T0)
        outs, fin, ev = fsm_rounds_kernel(run, None, stride)
        assert (outs, fin) == sequential(run, None)
        assert ev.new_at(stride) >= {stride - 1, 0}


T0 = 1_700_000_000 * 10**9
policies = st.sampled_from([(1, 1, 1), (1, 3, 3600), (2, 120, 60), (5, 10, 60), (100, 1000, 60), (3, 7, 60)])
req = st.tuples(policies, st.sampled_from([0, 0, 1, 1, 1, 1, 2, 5]), st.sampled_from([0, 0, 0, 1000, 10**9, 7 * 10**9]))


@settings(max_examples=300, deadline=None)
@given(st.lists(req, min_size=1, max_size=120), st.booleans())
def test_parallel_schemes_equal_sequential(reqs, start_with_entry):
    now, run = T0, []
    for (b, c, p), q, d in reqs:
        now += d
        _, ei, dvt = derive(b, c, p)
        run.append((now, ei, dvt, q))
    s0 = (T0 - 10**9, T0 + 5 * 10**9) if start_with_entry else None
    want = sequential(run, s0)
    assert speculate_commit(run, s0) == want
    assert fsm_rounds(run, s0) == want
    for stride in (16, kg.CTA_STRIDE):
        assert fsm_rounds_kernel(run, s0, stride)[:2] == want


CYCLE_DER = [derive(*p) for p in CYCLE_POLICIES]


def cycle_state(c, j, now=T0):
    """the state of a live entry in family j (tat = now - ei + j * ei) after a q = 0 row of cycle policy c"""
    _, ei, dvt = CYCLE_DER[c]
    return (now - ei + j * ei, now - ei + j * ei + dvt)


@settings(max_examples=60, deadline=None)
@given(st.integers(1, 6), st.integers(1, 9000), st.sampled_from([kg.CTA_STRIDE, kg.CLUSTER_STRIDE]),
       st.integers(0, 2**32 - 1), st.booleans(), st.sampled_from(["fresh", "cycle", "family"]), st.integers(0, 4), st.sampled_from([0.0, 0.02, 0.3]),
       st.sampled_from([0, 10**6, 6 * 10**9]))
def test_kernel_rounds_on_k_cycles(k, n, stride, seed, periodic, start, n_q1, deny, step):
    """K-cycle runs (K = 1..6, periodic or random order, with q = 1 and denied rows, clocks that stand still or move)
    through the kernel-faithful model at both group strides, and their index-order residues."""
    rng = np.random.default_rng(seed)
    pol, q = cycle_steps(n, k, start=int(rng.integers(k)), rng=None if periodic else rng,
                         q1_at=rng.choice(n, min(n_q1, n), replace=False), deny_at=np.nonzero(rng.random(n) < deny)[0])
    now = T0 + np.cumsum(np.where(rng.random(n) < 0.01, step, 0))
    run = model_run(pol, q, now)
    s0 = {"fresh": None, "cycle": cycle_state(0, 0), "family": cycle_state(2, 2)}[start]
    want = sequential(run, s0)
    outs, fin, ev = fsm_rounds_kernel(run, s0, stride)
    assert (outs, fin) == want
    assert ev.max_nc <= 4 and ev.evictions <= len(ev.changes)
    res, rs0 = residue_view(run, s0)
    if res is not None:
        outs, fin, _ = fsm_rounds_kernel(res, rs0, stride)
        assert (outs, fin) == (want[0][len(run) - len(res):], want[1])


@pytest.mark.parametrize("stride", [kg.CTA_STRIDE, kg.CLUSTER_STRIDE])
@pytest.mark.parametrize("k", range(1, 7))
def test_k_cycle_events(k, stride):
    """The events a plain rotation through K policies makes the kernel reach over 3 strides and one row.  K <= 3 from
    no entry (s0 differs from every cycle state): K + 1 candidates, K = 3 fills the set; K >= 4 from the state of the
    first cycle policy (s0 is a cycle state): K = 4 fills the set exactly and returns to s0, K = 5 and 6 evict s0
    and then every state they come back to."""
    n = 3 * stride + 1
    pol, q = cycle_steps(n, k, start=1 if k >= 4 else 0)
    run = model_run(pol, q, T0)
    s0 = cycle_state(0, 0) if k >= 4 else None
    want = sequential(run, s0)
    outs, fin, ev = fsm_rounds_kernel(run, s0, stride)
    assert (outs, fin) == want
    assert ev.max_nc == min(k + (k <= 3), 4)
    assert (ev.evictions > 0) == (k >= 5)
    assert ev.fsm_rounds > 0 if k >= 2 else ev.fsm_rounds == 0
    assert ev.switch_pos == (3 if k >= 2 else None) and ev.switch_mid_stride == (k >= 2)
    if k >= 2:
        assert [p for p, fsm, _ in ev.changes[:4]] == [0, 1, 2, 3] and not any(f for _, f, _ in ev.changes[:4])
    if k == 4:
        assert ev.s0_returns > 0
    if k >= 5:
        assert ev.s0_evicted and ev.evicted_returns == ev.evictions - (k - 4) > 0
        assert ev.new_at(stride) >= {stride - 1, 0}         # new states at both edges of a stride



@pytest.mark.parametrize("scenario", ["shape_trace-2", "shape_trace-3", "shape_trace-4", "shape_trace-5", "shape_trace-6",
                                      "switch_trace", "many_runs_trace", "compact_trace", "pipelined_trace",
                                      "small_trace"])
def test_gpu_cycle_scenarios_reach_their_events(scenario):
    """The key sequences of tests/test_gpu_fsm_cycles.py reach the kernel events each scenario names, in the sort
    pipeline's view and in the index-order residue's view (each builder asserts its events)."""
    import test_gpu_fsm_cycles as g
    name, _, k = scenario.partition("-")
    tr = getattr(g, name)(*([int(k)] if k else []))
    assert tr.batches

def test_toggling_key_needs_few_finite_state_rounds():
    """max_burst = 1 with zero-quantity requests: the entry flips between two states (SURVEY V8)."""
    _, ei, dvt = derive(1, 3, 3600)
    run = [(T0, ei, dvt, q) for q in [1, 0, 1, 1, 0, 0, 1, 2, 0, 1] * 30]
    want = sequential(run, None)
    assert fsm_rounds(run, None, stride=64) == want
    assert speculate_commit(run, None) == want
    assert len({o for o in want[0]}) > 2          # allowed and denied outcomes really alternate


# ---------------------------------------------------------------------------------------------------------
# the index-order pipeline (csrc/gcra_index_path.cuh): probe -> decide against the batch-start state -> resolve
# -> sequential residue, over a batch that mixes several keys; `entries` models the hashed batch bitmap (two
# keys may share an entry: both are then treated as shared, which must not change any result)
# ---------------------------------------------------------------------------------------------------------
def index_order_pipeline(batch, table, entries=4):
    """batch = [(key, req)], table = {key: state}.  Returns (outputs per row, table after the batch)."""
    table = dict(table)
    seen, shared = set(), set()
    for key, _ in batch:                                         # pass A: the batch bitmap
        e = key % entries
        (shared if e in seen else seen).add(e)
    outs, first_change, verdict = [None] * len(batch), {}, {}
    for i, (key, r) in enumerate(batch):                         # pass B (any order: reads batch-start states only)
        s0 = table.get(key)
        _, ns, o = decide(s0, r)
        outs[i] = o
        if key % entries not in shared:
            table[key] = ns                                      # alone on its key: commit
        else:
            verdict[i] = ns != s0
    for i in sorted(verdict, reverse=True):                      # atomicMin(mark[slot]), any order
        if verdict[i]:
            first_change[batch[i][0]] = i
    residue = []
    commits = {}
    for i in verdict:                                            # pass C
        key = batch[i][0]
        fm = first_change.get(key)
        if fm is not None and i > fm:
            residue.append(i)
        elif fm == i:
            commits[key] = decide(table.get(key), batch[i][1])[1]
    table.update(commits)
    for i in sorted(residue):                                    # residue: one after another, in batch order
        key, r = batch[i]
        _, table[key], outs[i] = decide(table.get(key), r)
    return outs, table


@settings(max_examples=300, deadline=None)
@given(st.lists(st.tuples(st.integers(0, 9), req), min_size=1, max_size=150), st.integers(1, 7))
def test_index_order_pipeline_equals_sequential(rows, entries):
    now, batch = T0, []
    for key, ((b, c, p), q, d) in rows:
        now += d
        _, ei, dvt = derive(b, c, p)
        batch.append((key, (now, ei, dvt, q)))
    table0 = {k: (T0 - 10**9, T0 + 5 * 10**9) for k in range(0, 10, 3)}
    want_outs, want_table = [], dict(table0)
    for key, r in batch:
        _, want_table[key], o = decide(want_table.get(key), r)
        want_outs.append(o)
    outs, table = index_order_pipeline(batch, table0, entries)
    assert outs == want_outs
    assert {k: v for k, v in table.items() if v is not None} == {k: v for k, v in want_table.items() if v is not None}
