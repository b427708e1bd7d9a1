"""Long pipelined runs against the oracle.

Traffic reaches the engine through the pipelined submission (the pinned ring, `submit_device`), whose host-side
state machine picks the K1 pipeline per batch from the residue feedback, overlaps stage 2 of a batch with the tail
of the previous one behind PEND bits, drains that overlap, rotates four scratch sets, and grows, purges or sweeps
the table between batches while PEND bits and marks of earlier batches are still in flight.  Every scenario here
compares every row bit-exact with ONE oracle store that replays the same rows in submission order, whatever
pipeline sequence the timing of the run produced.  The engine statistics asserted on (`path_switches`, `drains`,
`index_batches`, `grows`, `purges`) only prove that the machinery was really exercised: they are lower bounds.

At the end of a run the engine's counters (allowed / denied / errors / len / expired_hits) are compared with the
oracle: they are added up separately by every decide kernel and feed the metrics and the adaptive sweep policy,
and no result comparison can catch a miscount."""
import numpy as np
import pytest

import oracle
import throttlecrab_b200 as tc
import traces
from gpu_util import engine_requests, first_mismatch

pytestmark = pytest.mark.gpu

T0 = traces.T0
MS = 1_000_000
P0, P3 = 0, 3                       # traces.POLICIES rows: (100, 1000, 60 s) and (5, 10, 60 s)


def k1_modes(*names):
    """pytest params for `k1_path, index_min`: the conftest modes, plus "adaptive-small" -- the adaptive choice
    for batches from 512 rows on (GCRA_INDEX_MIN=512, GCRA_ADAPTIVE=1, read by gcra_create)."""
    out = []
    for n in names:
        out.append(pytest.param("auto", "512", id=n) if n == "adaptive-small" else pytest.param(n, None, id=n))
    return out


def set_index_min(monkeypatch, index_min):
    if index_min is not None:
        monkeypatch.setenv("GCRA_INDEX_MIN", index_min)
        monkeypatch.setenv("GCRA_ADAPTIVE", "1")


def check_universe(key_ids):
    ids = np.unique(np.asarray(key_ids, np.uint64))
    assert len(np.unique(tc.hash_key_ids(ids))) == len(ids), "64-bit key hashes collide inside the trace"


def ring_run(ring, batches, fill, now_of, at_boundary=None):
    """Submit `batches` (a list of row counts) through `ring`, paced as a server drives it: after submitting batch
    t, wait for batch t - slots + 1, so that the residue feedback of earlier batches can reach the host before the
    next submissions.  `fill(t, slot_array)` writes batch t's rows, `now_of(t)` is its submit clock and
    `at_boundary(t)` runs before batch t is submitted.  Returns the results of all batches, concatenated."""
    S = ring.slots
    out = np.empty(sum(batches), tc.RES_DTYPE)
    off = np.concatenate([[0], np.cumsum(batches)])

    def collect(j):
        ring.wait(j % S)
        out[off[j]:off[j + 1]] = ring.res[j % S][:batches[j]]

    for t, n in enumerate(batches):
        if at_boundary is not None:
            at_boundary(t)
        fill(t, ring.req[t % S][:n])
        ring.submit(t % S, n, now_of(t))
        if t - S + 1 >= 0:
            collect(t - S + 1)
    for j in range(max(len(batches) - S + 1, 0), len(batches)):
        collect(j)
    return out


def assert_counters(st, want, ora, require_expired=True):
    """The engine's counters against the results and the oracle store that produced them (require_expired: the
    trace must write over an expired entry at least once)."""
    s = st.stats()
    ok = want["status"] == 0
    got = {f: s[f] for f in ("allowed", "denied", "errors", "len", "expired_hits")}
    exp = {"allowed": int(want["allowed"].sum()), "denied": int((ok & (want["allowed"] == 0)).sum()),
           "errors": int((~ok).sum()), "len": ora.len(), "expired_hits": ora.expired_writes()}
    assert got == exp, (got, exp)
    assert exp["expired_hits"] > 0 or not require_expired      # the counted event really happens in the trace


# ---------------------------------------------------------------------------------------------------------------
# scenario 1 / 3: phases that move the adaptive K1 choice at the production thresholds (2^15-row batches)
# ---------------------------------------------------------------------------------------------------------------
T = 1 << 15
BURST_KEYS, BURST_ROWS = 2048, 16
SAT_KEYS = 50
MIXED_BURST_KEYS = 328
ZIPF_KEYS = 200_000
PHASES = [("burst", 25), ("saturated", 40), ("mixed", 25), ("zipf", 15), ("burst", 20)]


def phase_trace():
    """The rows of every batch (trace key ids, policy index, quantity) and one clock per batch.  The residue
    fractions are the oracle's (rows behind the first state change of their key in the batch):
    burst      2048 fresh P0 keys x 16 rows, q = 1: every row changes its key's state (94 %);
    saturated  50 P3 keys, exhausted in their first batch: nothing changes any more (0 %);
    mixed      328 fresh burst-spending keys x 16 rows among the saturated rows (15 %: between 1/8 and 1/4, so the
               index-order pipeline stays and drains the overlap);
    zipf       config2 ticks over 200 K fresh keys (policy = key % 8): keys spend their bursts (60 % -> 40 %)."""
    rng = np.random.default_rng(11)
    batches, now, fresh, zipf_tick = [], T0, 10_000_000, 0

    def burst_keys(n):
        nonlocal fresh
        fresh += n
        return np.repeat(np.arange(fresh - n, fresh, dtype=np.uint64), BURST_ROWS)

    for name, count in PHASES:
        for _ in range(count):
            now += MS
            if name == "burst":
                key = burst_keys(BURST_KEYS)
                rng.shuffle(key)
                pol, q = np.full(T, P0), np.ones(T, np.int64)
            elif name in ("saturated", "mixed"):
                key = (5_000_000 + rng.integers(0, SAT_KEYS, T)).astype(np.uint64)
                pol, q = np.full(T, P3), np.ones(T, np.int64)
                if name == "mixed":
                    b = burst_keys(MIXED_BURST_KEYS)
                    key[:len(b)] = b
                    pol[:len(b)] = P0
                    perm = rng.permutation(T)
                    key, pol = key[perm], pol[perm]
            else:
                z = traces.config2(n_keys=ZIPF_KEYS, n_ticks=1, tick_size=T, start_tick=zipf_tick)
                zipf_tick += 1
                key, pol, q = z["key"], (z["key"] % np.uint64(8)).astype(np.int64), z["quantity"]
            batches.append((key, pol, q, now))
    return batches


def full_rows(key, pol, q, now, policies=traces.POLICIES):
    req = np.zeros(len(key), traces.REQ_DTYPE)
    req["key"] = key
    p = policies[pol]
    req["max_burst"], req["count_per_period"], req["period"] = p[:, 0], p[:, 1], p[:, 2]
    req["quantity"] = q
    req["now_ns"] = now
    return req


def assert_adaptive_machinery(s, n_batches):
    assert s["path_switches"] >= 2, s
    assert 0 < s["index_batches"] < n_batches, s
    assert s["drains"] >= 1, s


@pytest.mark.parametrize("k1_path", ["auto", "index", "sort"], indirect=True)
def test_adaptive_switching_48_byte_ring(k1_path):
    """The phases of `phase_trace` through a 3-slot 48-byte ring.  In the default mode the residue feedback sends
    the first bursts to the sort pipeline (31-batch hold), the saturated batches come back to the index-order
    pipeline with the overlap on, the mixed batches keep it and drain the overlap, and the Zipf batches switch to
    the sort pipeline again."""
    batches = phase_trace()
    req = np.concatenate([full_rows(*b) for b in batches])
    check_universe(req["key"])
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=400_000, created_ns=T0, p0=10**9)
    want = ora.replay(req)
    ereq = engine_requests(req)
    st = tc.ManualStore(capacity=400_000, created_ns=T0, max_batch=T)
    ring = tc.Ring(tc.RateLimiter(st), slots=3, slot_capacity=T)

    def fill(t, dst):
        dst[:] = ereq[t * T:(t + 1) * T]

    got = ring_run(ring, [T] * len(batches), fill, lambda t: batches[t][3])
    bad = first_mismatch(want, got, req)
    assert bad is None, bad
    assert_counters(st, want, ora)
    s = st.stats()
    print("48-byte ring, %s: %s" % (k1_path, {f: s[f] for f in ("path_switches", "drains", "index_batches")}))
    if k1_path == "auto":
        assert_adaptive_machinery(s, len(batches))
    elif k1_path == "index":
        assert s["index_batches"] == len(batches) and s["drains"] >= 1, s


# scenario 3: the same phases as 16-byte requests (policy index + per-call clock)
I32_MAX = 2**31 - 1
POLICY_TABLE = np.concatenate([traces.POLICIES, [(0, 10, 60),                  # 8: invalid (max_burst = 0)
                                                 (2**32, 1, 2**63 - 1)]])      # 9: Duration * u32 overflows
NPOL = len(POLICY_TABLE)


@pytest.mark.parametrize("k1_path", ["auto", "index", "sort"], indirect=True)
def test_adaptive_switching_16_byte_ring(k1_path):
    """The phases of the 48-byte test through a compact ring (`parse_request<true>` in ingest, pass A, pass B,
    pass C and the by-row tail).  Sprinkled into every batch: the invalid and the overflowing policy, policy
    indices at and beyond the table (GCRA_INTERNAL, all-zero results, not replayed by the oracle), negative
    quantities and 2^31 - 1.  One batch has a negative per-call clock."""
    assert oracle.derive(*POLICY_TABLE[9])[0] == 3 and tc.derive_params(*[int(x) for x in POLICY_TABLE[9]])[0] == 3
    rng = np.random.default_rng(12)
    batches = phase_trace()
    neg_batch = 50                                       # saturated phase: index-order unless only sorting
    rows16, full, foreign = [], [], []
    for t, (key, pol, q, now) in enumerate(batches):
        pol, q = pol.astype(np.int64).copy(), q.copy()
        edge = rng.random(T)
        pol[edge < 0.002] = 8
        pol[(edge >= 0.002) & (edge < 0.004)] = 9
        far = (edge >= 0.004) & (edge < 0.006)           # (quantities >= 0: the policy check is what fails)
        neg = (edge >= 0.006) & (edge < 0.008)
        q[neg] = rng.choice([-1, -2**31], int(neg.sum()))
        q[(edge >= 0.008) & (edge < 0.009)] = I32_MAX
        r16 = np.zeros(T, tc.REQ16_DTYPE)
        r16["key_hash"] = tc.hash_key_ids(key)
        r16["quantity"] = q
        r16["policy"] = np.where(far, rng.choice([NPOL, NPOL + 1, 2**32 - 1], T), pol)
        rows16.append(r16)
        clock = -1 - 5 * MS if t == neg_batch else now
        full.append(full_rows(key[~far], pol[~far], q[~far], clock, POLICY_TABLE))
        foreign.append(far)
    req = np.concatenate(full)
    check_universe(req["key"])
    far = np.concatenate(foreign)
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=400_000, created_ns=T0, p0=10**9)
    want = np.zeros(len(far), tc.RES_DTYPE)
    want["status"][far] = tc.INTERNAL
    want[~far] = ora.replay(req)
    st = tc.ManualStore(capacity=400_000, created_ns=T0, max_batch=T)
    lim = tc.RateLimiter(st)
    pol = np.zeros(NPOL, tc.POLICY_DTYPE)
    pol["max_burst"], pol["count_per_period"], pol["period"] = POLICY_TABLE.T
    lim.set_policies(pol)
    ring = tc.Ring(lim, slots=4, slot_capacity=T, compact=True)

    def fill(t, dst):
        dst[:] = rows16[t]

    got = ring_run(ring, [T] * len(batches), fill,
                   lambda t: -1 - 5 * MS if t == neg_batch else batches[t][3])
    bad = first_mismatch(want, got)
    assert bad is None, bad
    nb = got[neg_batch * T:(neg_batch + 1) * T]
    assert (nb["status"] != 0).all() and (nb["status"] == tc.INTERNAL).sum() > T // 2
    assert set(np.unique(want["status"])) == {0, 1, 2, 3}
    assert_counters(st, want, ora)
    s = st.stats()
    print("16-byte ring, %s: %s" % (k1_path, {f: s[f] for f in ("path_switches", "drains", "index_batches")}))
    if k1_path == "auto":
        assert_adaptive_machinery(s, len(batches))


# ---------------------------------------------------------------------------------------------------------------
# scenario 2: hundreds of small batches -- PEND chains and forced drains
# ---------------------------------------------------------------------------------------------------------------
LONG_BATCHES = 420
TOGGLER_ROWS, SPENDER_ROWS = 64, 40


def long_trace():
    """420 batches of 2048-4096 rows, one clock per batch advancing 20 ms.  In every batch: a max_burst = 1 key with
    zero-quantity rows, whose state toggles on every row (it is in every residue, and deferred from tail to tail),
    and a P0 key that spends its burst across batch boundaries and then one token every third batch; the other rows
    are uniform over 100 K keys (policy = key % 8, the trace quantity mix)."""
    rng = np.random.default_rng(13)
    sizes = rng.integers(2048, 4097, LONG_BATCHES)
    parts = []
    for t, n in enumerate(sizes):
        req = np.zeros(n, traces.REQ_DTYPE)
        bg = rng.integers(0, 100_000, n).astype(np.uint64)
        req["key"] = bg
        traces.fill_policy(req, (bg % np.uint64(8)).astype(np.int64))
        req["quantity"] = traces.quantities(rng.integers(0, 2**63, n, dtype=np.uint64))
        rows = rng.permutation(n)
        tog, spend = rows[:TOGGLER_ROWS], rows[TOGGLER_ROWS:TOGGLER_ROWS + SPENDER_ROWS]
        req["key"][tog] = 1_000_000
        req["max_burst"][tog], req["count_per_period"][tog], req["period"][tog] = 1, 3, 3600
        req["quantity"][tog] = 0
        req["key"][spend] = 1_000_001
        req["max_burst"][spend], req["count_per_period"][spend], req["period"][spend] = traces.POLICIES[P0]
        req["quantity"][spend] = 1
        req["now_ns"] = T0 + (t + 1) * 20 * MS
        parts.append(req)
    return parts


@pytest.mark.parametrize("k1_path,index_min", k1_modes("auto", "index", "sort", "adaptive-small"),
                         indirect=["k1_path"])
def test_long_runs_ring_and_device(k1_path, index_min, monkeypatch):
    """420 ragged batches, once through a paced 3-slot ring and once submitted back to back with `submit_device`
    and joined at the end: both bit-exact to the oracle, with exact counters.  The first and the last batch of the
    second run split off their first 200 rows as a blocking in-stream batch (the one-CTA small-batch kernel); a
    blocking batch orders itself after everything, which restarts the count towards the forced drain, so there are
    no others.  With the residue far below 1/8, the index-order runs give up the overlap every 65th batch."""
    import torch
    set_index_min(monkeypatch, index_min)
    parts = long_trace()
    req = np.concatenate(parts)
    check_universe(np.append(np.arange(100_000), [1_000_000, 1_000_001]))
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=110_000, created_ns=T0, p0=10**9)
    want = ora.replay(req)
    ereq = engine_requests(req)
    sizes = [len(p) for p in parts]
    off = np.concatenate([[0], np.cumsum(sizes)])
    n_batches = len(parts)
    stats = {}

    # (a) the ring
    st = tc.ManualStore(capacity=110_000, created_ns=T0, max_batch=4096)
    ring = tc.Ring(tc.RateLimiter(st), slots=3, slot_capacity=4096)

    def fill(t, dst):
        dst[:] = ereq[off[t]:off[t + 1]]

    got = ring_run(ring, sizes, fill, lambda t: int(parts[t]["now_ns"][0]))
    bad = first_mismatch(want, got, req)
    assert bad is None, "ring: " + bad
    assert_counters(st, want, ora)
    stats["ring"] = st.stats()
    st.close()

    # (b) submit_device back to back, joined at the end
    st = tc.ManualStore(capacity=110_000, created_ns=T0, max_batch=4096)
    lim = tc.RateLimiter(st)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    with torch.cuda.stream(stream):
        d_req = torch.from_numpy(ereq.view(np.uint8)).to(dev)
        d_res = torch.zeros(len(req) * 32, dtype=torch.uint8, device=dev)
        stream.synchronize()
        for t in range(n_batches):
            a, b = int(off[t]), int(off[t + 1])
            if t in (0, n_batches - 1):
                lim.rate_limit_batch_device(200, d_req[a * 48:].data_ptr(), d_res[a * 32:].data_ptr(),
                                            stream.cuda_stream)
                a += 200
            lim.submit_device(b - a, d_req[a * 48:].data_ptr(), d_res[a * 32:].data_ptr(), stream.cuda_stream)
        lim.join(stream.cuda_stream)
        stream.synchronize()
    got = d_res.cpu().numpy().view(tc.RES_DTYPE)
    bad = first_mismatch(want, got, req)
    assert bad is None, "submit_device: " + bad
    assert_counters(st, want, ora)
    stats["device"] = st.stats()
    print("long runs, %s: %s" % (k1_path if index_min is None else "adaptive-small",
                                 {k: {f: s[f] for f in ("path_switches", "drains", "index_batches")}
                                  for k, s in stats.items()}))
    if k1_path == "index" or index_min is not None:
        for k, s in stats.items():
            assert s["drains"] >= n_batches // 64, (k, s)
            assert s["index_batches"] > n_batches // 2, (k, s)


# ---------------------------------------------------------------------------------------------------------------
# scenario 4: growth, purges and sweeps between pipelined batches
# ---------------------------------------------------------------------------------------------------------------
def arriving_keys_trace():
    """Keys arrive progressively (as in test_tight_table_stash_and_growth), so a 16-entry tight table grows many
    times while old keys stay hot; clocks jump so that entries expire between sweeps."""
    n_keys, n = 20_000, 200_000
    rng = np.random.default_rng(14)
    req = np.zeros(n, traces.REQ_DTYPE)
    req["key"] = (rng.integers(0, n_keys, n) * np.linspace(0.01, 1.0, n)).astype(np.uint64)
    traces.fill_policy(req, (req["key"] % np.uint64(8)).astype(np.int64))
    req["quantity"] = rng.choice([0, 1, 1, 1, 2, 5], n)
    req["now_ns"] = T0 + np.cumsum(rng.choice([0, 1000, 2_000_000, 700_000_000], n))
    return req, n_keys


def test_growth_purge_and_sweeps_between_pipelined_batches(k1_path):
    """A tight table (GCRA_FLAG_TIGHT_TABLE) fed through a 3-slot ring in 2048-row batches: the table grows and
    purges between pipelined batches, and every third batch boundary sweeps both the engine and the oracle at the
    clock of the batch before.  Then the same rows through a PeriodicStore that sweeps on its own policy from the
    ring's clock."""
    req, n_keys = arriving_keys_trace()
    check_universe(np.arange(n_keys))
    ereq = engine_requests(req)
    B, every = 2048, 3
    sizes = [min(B, len(req) - a) for a in range(0, len(req), B)]
    def first_now(t):                   # the submit clock: no row of batch t or later is older
        return int(req["now_ns"][t * B])

    def sweep_now(t):                   # sweeps at boundary t use the clock of the last row before it
        return int(req["now_ns"][t * B - 1])

    def fill(t, dst):
        dst[:] = ereq[t * B:t * B + len(dst)]

    # oracle: the same rows, swept at the same boundaries
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=16, created_ns=T0, p0=10**9)
    want = np.empty(len(req), tc.RES_DTYPE)
    o_swept = {}
    for t in range(len(sizes)):
        if t and t % every == 0:
            o_swept[t] = (ora.force_sweep(sweep_now(t)), ora.len())
        want[t * B:t * B + sizes[t]] = ora.replay(req[t * B:t * B + sizes[t]])

    st = tc.ManualStore(capacity=16, created_ns=T0, max_batch=B, flags=tc._native.FLAG_TIGHT_TABLE)
    ring = tc.Ring(tc.RateLimiter(st), slots=3, slot_capacity=B)
    e_swept = {}

    def boundary(t):
        if t and t % every == 0:
            e_swept[t] = (st.sweep(sweep_now(t)), st.len())

    got = ring_run(ring, sizes, fill, first_now, boundary)
    bad = first_mismatch(want, got, req)
    assert bad is None, bad
    assert e_swept == o_swept
    assert sum(r for r, _ in o_swept.values()) > 0
    s = st.stats()
    print("tight table, %s: %s" % (k1_path, {f: s[f] for f in ("grows", "purges", "index_batches", "drains",
                                                                  "stash_entries", "sweeps")}))
    assert s["grows"] >= 2 and s["purges"] >= 1, s
    assert s["len"] == ora.len()
    st.close()

    # a PeriodicStore sweeping on its own policy (every 60 s of the ring's clock)
    st = tc.PeriodicStore(capacity=16, created_ns=T0, max_batch=B, flags=tc._native.FLAG_TIGHT_TABLE, p0=60)
    ring = tc.Ring(tc.RateLimiter(st), slots=3, slot_capacity=B)
    got = ring_run(ring, sizes, fill, first_now)
    bad = first_mismatch(want, got, req)
    assert bad is None, "PeriodicStore: " + bad
    assert st.stats()["sweeps"] > 0
    last = int(req["now_ns"][-1])
    st.sweep(last)
    ora.force_sweep(last)
    assert st.len() == ora.len()
    hashes = tc.hash_key_ids(np.arange(n_keys))
    for k in range(0, n_keys, 97):
        assert st.peek(int(hashes[k])) == ora.entry("k:%d" % k), k
