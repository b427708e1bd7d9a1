"""Which runs are hot, who decides them, and what the side streams leave behind, against the oracle.

Stage 2 of a sorted batch (csrc/gcra_b200.cu, `enqueue_decide_sorted_t`) lists the hot runs with `list_runs_kernel`,
starts the one-CTA and the cluster hot-run kernels on two engine-wide side streams, decides everything else with
`decide_kernel` on the batch's stream and joins the side streams through events.  Listing and skipping go through the
same `decide_chunk` code: a run is hot iff its LONG_RUN_MIN-th row is on the same key.  If the two disagreed by one
row, a row would be decided twice or never written; if a launch grid (`long_grid`, `clusters`, capped by how many runs
the batch can hold) were one short, a run would be left to nobody.

The boundary scenarios place every run at a chosen sorted position: a save of the table (one key word per slot, in
slot order) tells the test each key's slot, and the sort order of a batch is the slot order.  Each engine under test
loads that file, so all of them sort the batch alike.  In the index-order pipeline only the residue is sorted (a key's
rows behind its first state change), so each run also has a twin one row longer, whose residue run has the same
length, placed by filler keys of two rows (one residue row each).

Every row, the final entry of every key of the batch and the counters are compared bit-exact with one oracle store
replaying the same rows in submission order."""
import functools

import numpy as np
import pytest

import oracle
import throttlecrab_b200 as tc
import traces
from gpu_util import engine_requests, first_mismatch
from kernel_geometry import GIANT_RUN_MIN, LONG_RUN_MIN
from test_gpu_background_snapshot import read_snapshot
from test_gpu_pipelined_runs import assert_counters, check_universe

pytestmark = pytest.mark.gpu

T0 = traces.T0
MS, S = 1_000_000, 1_000_000_000
P0, P3, P6 = 0, 3, 6                     # traces.POLICIES: (100, 1000, 60 s), (5, 10, 60 s), (1, 3, 3600 s)
P_INVALID = len(traces.POLICIES)         # max_burst = 0: GCRA_INVALID_RATE_LIMIT
POLICY_TABLE = np.concatenate([traces.POLICIES, [(0, 10, 60)]])
FORMATS = ("48", "16/32", "16/16")       # request / result bytes
POOL = 8000                              # keys whose slots the boundary scenarios know
CHUNK = 32                               # rows of one warp chunk of decide_chunk


def policies():
    pol = np.zeros(len(POLICY_TABLE), tc.POLICY_DTYPE)
    pol["max_burst"], pol["count_per_period"], pol["period"] = POLICY_TABLE.T
    return pol


def hot_rows(rng, n):
    """(policy, quantity) of a run of n rows on one key: the first row spends a token (a state change, so the index-order
    residue is the other n - 1 rows), then a mix that keeps changing the state (P0 spends, P6 with q = 0 toggles) and
    denies (P3 after its burst)"""
    pol = rng.choice([P0, P3, P6], n)
    q = rng.choice([0, 0, 1, 2], n)
    pol[0], q[0] = P0, 1
    return pol.astype(np.int64), q.astype(np.int64)


def interleave(rng, runs):
    """The rows of `runs` [(key, policy[], quantity[])] in one random order that keeps each key's rows in order."""
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


def full_rows(key, pol, q, now):
    req = np.zeros(len(key), traces.REQ_DTYPE)
    req["key"] = key
    p = POLICY_TABLE[pol]
    req["max_burst"], req["count_per_period"], req["period"] = p[:, 0], p[:, 1], p[:, 2]
    req["quantity"], req["now_ns"] = q, now
    return req


class Batch:
    def __init__(self, key, pol, q, now):
        self.key, self.pol, self.q, self.now = key, pol, q, int(now)
        self.req = full_rows(key, pol, q, now)


def run_batch(lim, b, fmt):
    """one blocking batch in format `fmt`: 32-byte result rows (16/16: expanded on the host)"""
    if fmt == "48":
        return lim.rate_limit_batch(engine_requests(b.req))
    r16 = np.zeros(len(b.key), tc.REQ16_DTYPE)
    r16["key_hash"] = tc.hash_key_ids(b.key)
    r16["quantity"], r16["policy"] = b.q, b.pol
    if fmt == "16/32":
        return lim.rate_limit_batch16(r16, b.now)
    return tc.expand_results16(r16, b.now, policies(), lim.rate_limit_batch16(r16, b.now, compact_results=True))


def new_engine(max_batch, snapshot=None):
    st = tc.ManualStore(capacity=20_000, created_ns=T0, max_batch=max_batch)
    lim = tc.RateLimiter(st)
    lim.set_policies(policies())
    if snapshot is not None:
        st.load(snapshot)
    return st, lim


def check_batches(batches, fmt, max_batch, snapshot=None, pre=()):
    """`batches` through a fresh engine (loaded from `snapshot`, which holds the table after the `pre` batches), one
    blocking call each: every row, the entry of every key and the counters against one oracle replay of pre + batches"""
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=20_000, created_ns=T0, p0=10**9)
    want = [ora.replay(b.req) for b in list(pre) + list(batches)]
    st, lim = new_engine(max_batch, snapshot)
    for t, b in enumerate(batches):
        got = run_batch(lim, b, fmt)
        bad = first_mismatch(want[len(pre) + t], got, b.req)
        assert bad is None, "batch %d (%s): %s" % (t, fmt, bad)
    keys = np.unique(np.concatenate([b.key for b in batches]))
    for k, h in zip(keys.tolist(), tc.hash_key_ids(keys).tolist()):
        assert st.peek(int(h)) == ora.entry("k:%d" % k), k
    assert_counters(st, np.concatenate(want), ora, require_expired=False)
    st.close()


# ---------------------------------------------------------------------------------------------------------------
# runs at chosen sorted positions
# ---------------------------------------------------------------------------------------------------------------
def mix64(x):
    """gcra_device.cuh stored_key: the key word a key hash is kept under in the table"""
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(30))
        x = x * np.uint64(0xbf58476d1ce4e5b9)
        x = x ^ (x >> np.uint64(27))
        x = x * np.uint64(0x94d049bb133111eb)
        x = x ^ (x >> np.uint64(31))
    return np.where(x < 2, x + np.uint64(2), x)


@functools.lru_cache(maxsize=None)
def claimed_pool(path):
    """A table holding the POOL keys (one allowed row each at T0), saved to `path`: (the claiming batch, the pool key
    ids in slot order).  Engines that load the file sort every batch of these keys alike."""
    key = np.arange(1, POOL + 1, dtype=np.uint64) * np.uint64(7919)
    check_universe(key)
    pre = Batch(key, np.full(POOL, P0), np.zeros(POOL, np.int64), T0)
    st, lim = new_engine(1 << 16)
    assert first_mismatch(oracle.OracleStore(oracle.PERIODIC, capacity=20_000, created_ns=T0, p0=10**9).replay(pre.req),
                          run_batch(lim, pre, "48")) is None
    st.save(path)
    st.close()
    _, words, _, _ = read_snapshot(path)
    slot = {int(w): s for s, w in enumerate(words.tolist())}
    slots = np.array([slot[int(w)] for w in mix64(tc.hash_key_ids(key)).tolist()])
    return pre, key[np.argsort(slots)]


class Layout:
    """Runs laid out in slot order: `sort` and `res` are the rows before the next key in the sorted batch and in the
    index-order residue.  Filler keys: 'A' has one row (sort only), 'B' two (its second row is residue)."""

    def __init__(self, pool, rng):
        self.pool, self.rng, self.next = pool, rng, 0
        self.runs, self.sort, self.res = [], 0, 0
        self.hot = []                    # (key, rows, sorted start, residue start)

    def take(self):
        k = self.pool[self.next]
        self.next += 1
        return k

    def filler(self, kind):
        k = self.take()
        if kind == "A":
            self.runs.append((k, np.array([P3]), np.array([1])))
            self.sort += 1
        else:
            self.runs.append((k, np.array([P0, P3]), np.array([1, 1])))
            self.sort, self.res = self.sort + 2, self.res + 1

    def run(self, n, lane=None, view="sort"):
        """a hot-row run of n rows, first padded with fillers so that it starts at `lane` of a chunk in `view`"""
        if lane is not None:
            if view == "sort":
                for _ in range((lane - self.sort) % CHUNK):
                    self.filler("A")
            else:
                for _ in range((lane - self.res) % CHUNK):
                    self.filler("B")
        k = self.take()
        self.runs.append((k, *hot_rows(self.rng, n)))
        self.hot.append((int(k), n, self.sort, self.res))
        self.sort, self.res = self.sort + n, self.res + n - 1

    def batch(self, now, errors=0):
        key, pol, q = interleave(self.rng, self.runs)
        if errors:
            # rows that fail validation sort to null_slot, behind every run
            at = self.rng.integers(0, len(key) + 1, errors)
            ek = np.asarray(self.pool[self.rng.integers(0, self.next, errors)], np.uint64)
            neg = np.arange(errors) % 2 == 0
            key = np.insert(key, at, ek)
            pol = np.insert(pol, at, np.where(neg, P0, P_INVALID))
            q = np.insert(q, at, np.where(neg, -1, 1))
        return Batch(key, pol, q, now)


def boundary_batches(pool):
    """(name, batch): runs of LONG_RUN_MIN - 1, LONG_RUN_MIN and LONG_RUN_MIN + 1 rows starting at every lane of a chunk
    (and their twins at every lane of the residue); a hot run ending the batch, with and without error rows behind
    it; hot runs back to back, from position 0, next to cluster runs."""
    rng = np.random.default_rng(31)
    out = []
    lay = Layout(pool, rng)
    for lane in range(CHUNK):
        for d in (-1, 0, 1):
            lay.run(LONG_RUN_MIN + d, lane, "sort")
            lay.run(LONG_RUN_MIN + d + 1, lane, "residue")
    sort_lanes = {(n, s % CHUNK) for _, n, s, _ in lay.hot}
    res_lanes = {(n - 1, r % CHUNK) for _, n, _, r in lay.hot}
    want = {(LONG_RUN_MIN + d, lane) for d in (-1, 0, 1) for lane in range(CHUNK)}
    assert sort_lanes >= want and res_lanes >= want
    out.append(("lanes", lay.batch(T0 + S)))
    for errors in (0, 40):
        for n in (LONG_RUN_MIN, LONG_RUN_MIN + 1):   # its LONG_RUN_MIN-th row is the last row (sorted; residue)
            lay = Layout(pool, rng)
            for _ in range(7):
                lay.filler("B")
            lay.run(300)
            lay.filler("A")
            lay.run(n)
            b = lay.batch(T0 + S, errors)
            assert lay.sort + errors == len(b.key) and lay.hot[-1][2] + n == lay.sort
            out.append(("last-%d-errors-%d" % (n, errors), b))
    lay = Layout(pool, rng)
    for n in (LONG_RUN_MIN, LONG_RUN_MIN, LONG_RUN_MIN + 1):      # three back to back from position 0
        lay.run(n)
    for _ in range(5):
        lay.filler("B")
    for n in (GIANT_RUN_MIN, LONG_RUN_MIN, LONG_RUN_MIN - 1, GIANT_RUN_MIN + 1, LONG_RUN_MIN, GIANT_RUN_MIN - 1):
        lay.run(n)
    lay.filler("A")
    lay.run(LONG_RUN_MIN + 1)
    lay.run(LONG_RUN_MIN)
    assert lay.hot[0][2] == 0
    out.append(("adjacent", lay.batch(T0 + S, 10)))
    return out


@pytest.mark.parametrize("fmt", FORMATS)
def test_runs_at_every_lane_and_edge(fmt, tmp_path_factory):
    """Runs of 255, 256 and 257 rows starting at each of the 32 lanes of a chunk, in the sorted batch and in the
    residue; a hot run whose 256th row is the batch's last (before the error rows, in the second batch); runs back to
    back from position 0 and beside cluster runs.  Each batch runs on its own engine loaded with the claimed table."""
    path = str(tmp_path_factory.getbasetemp() / "hot_run_listing_pool.gcra")
    pre, pool = claimed_pool(path)
    for name, b in boundary_batches(pool):
        check_universe(b.key)
        check_batches([b], fmt, 1 << 16, snapshot=path, pre=[pre])


# ---------------------------------------------------------------------------------------------------------------
# batch sizes at the launch caps: long_grid = min(SMs, n / LONG_RUN_MIN), clusters = max(min(16, n / GIANT_RUN_MIN), 1)
# ---------------------------------------------------------------------------------------------------------------
SHAPES = {
    "one-run-of-256": [LONG_RUN_MIN],                      # one CTA, no cluster launch; residue of 255
    "one-run-of-4095": [GIANT_RUN_MIN - 1],                # the first cluster launch, an empty giant list
    "one-run-of-4096": [GIANT_RUN_MIN],                    # clusters = 1
    "long-list-full": [LONG_RUN_MIN] * ((1 << 15) // LONG_RUN_MIN),    # 128 one-CTA runs in max_batch = 2^15
    "giant-list-full": [GIANT_RUN_MIN] * ((1 << 15) // GIANT_RUN_MIN),  # 8 cluster runs
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_batches_made_of_hot_runs(shape):
    """Batches made only of hot runs, with max_batch equal to the batch: the work lists full to their last entry and the
    grids at their caps.  Two batches of the same keys, one clock each."""
    rng = np.random.default_rng(len(shape))
    lengths = SHAPES[shape]
    keys = 9_000_000 + np.arange(len(lengths), dtype=np.uint64)
    check_universe(keys)
    batches = [Batch(*interleave(rng, [(k, *hot_rows(rng, n)) for k, n in zip(keys, lengths)]), T0 + (t + 1) * S)
               for t in range(2)]
    check_batches(batches, "48", sum(lengths))


@pytest.mark.parametrize("fmt", FORMATS[1:])
def test_batches_made_of_hot_runs_compact(fmt):
    """The full work lists in the 16-byte formats."""
    rng = np.random.default_rng(77)
    keys = 9_100_000 + np.arange(12, dtype=np.uint64)
    lengths = [GIANT_RUN_MIN] * 4 + [LONG_RUN_MIN] * 8
    check_universe(keys)
    b = Batch(*interleave(rng, [(k, *hot_rows(rng, n)) for k, n in zip(keys, lengths)]), T0 + S)
    check_batches([b], fmt, sum(lengths))


# ---------------------------------------------------------------------------------------------------------------
# what the side streams leave behind: back-to-back batches, then a Store-trait op and a background save
# ---------------------------------------------------------------------------------------------------------------
CTA_KEYS, CLUSTER_KEYS, BG_KEYS = 30, 4, 20_000
N_BEFORE, N_AFTER = 24, 4                 # batches before the Store-trait op and the save, and after them


@functools.lru_cache(maxsize=None)
def stream_trace():
    """28 batches at 1 ms steps: 10 one-CTA runs (of 30 recurring keys) and 1-2 cluster runs (of 4) in each, among 1500
    background rows."""
    rng = np.random.default_rng(41)
    batches = []
    for t in range(N_BEFORE + N_AFTER):
        runs = [(10_000_000 + k, *hot_rows(rng, int(rng.integers(LONG_RUN_MIN, 1500))))
                for k in rng.choice(CTA_KEYS, 10, replace=False)]
        runs += [(11_000_000 + k, *hot_rows(rng, int(rng.integers(GIANT_RUN_MIN, GIANT_RUN_MIN + 1000))))
                 for k in rng.choice(CLUSTER_KEYS, int(rng.integers(1, 3)), replace=False)]
        key, pol, q = interleave(rng, [(np.uint64(k), p, x) for k, p, x in runs])
        bg = rng.integers(0, BG_KEYS, 1500).astype(np.uint64)
        at = rng.integers(0, len(key) + 1, len(bg))
        key = np.insert(key, at, bg)
        pol = np.insert(pol, at, (bg % np.uint64(8)).astype(np.int64))
        q = np.insert(q, at, rng.choice([0, 1, 1, 2, 5], len(bg)))
        batches.append(Batch(key, pol, q, T0 + (t + 1) * MS))
    hot = [10_000_000 + k for k in range(CTA_KEYS)] + [11_000_000 + k for k in range(CLUSTER_KEYS)]
    check_universe(np.concatenate([np.arange(BG_KEYS), hot]))
    # the Store-trait op: a hot key of the last batch before it, and the oracle at that point (the cut of the save)
    last = batches[N_BEFORE - 1]
    cas_key = "k:%d" % int(last.key[np.isin(last.key, np.array(hot[CTA_KEYS:], np.uint64))][0])
    cas_now = last.now
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=40_000, created_ns=T0, p0=10**9)
    want = [ora.replay(b.req) for b in batches[:N_BEFORE]]
    v = ora.get(cas_key, cas_now)
    assert v is not None and ora.compare_and_swap_with_ttl(cas_key, v, v + 1000, 60 * S, cas_now) is True
    cut = {k: ora.entry("k:%d" % k) for k in hot}
    cut_len, cut_expired = ora.len(), ora.expired_writes()
    want += [ora.replay(b.req) for b in batches[N_BEFORE:]]
    return batches, hot, (cas_key, cas_now, v), want, ora, cut, (cut_len, cut_expired)


@pytest.mark.parametrize("transport", ["submit_device", "ring"])
def test_side_streams_before_a_store_op_and_a_save(transport, tmp_path):
    """The batches back to back, never joined: 24, then a Store-trait get and compare_and_swap_with_ttl on a cluster
    run's key, then save_begin, then 4 more batches, then save_wait.  With `submit_device` every batch is in flight
    until the end; through a 3-slot ring each slot is waited for only before its reuse.  The Store-trait op sees the
    24 batches; the file holds the table they and the op left; every row, entry and counter equals the oracle's."""
    import torch
    batches, hot, (cas_key, cas_now, v), want, ora, cut, (cut_len, cut_expired) = stream_trace()
    nmax = max(len(b.key) for b in batches)
    st = tc.ManualStore(capacity=40_000, created_ns=T0, max_batch=nmax)
    lim = tc.RateLimiter(st)
    got = [None] * len(batches)
    path = str(tmp_path / "hot.gcra")
    if transport == "ring":
        ring = tc.Ring(lim, slots=3, slot_capacity=nmax)

        def submit(t):
            if t >= 3:
                collect(t - 3)
            ring.req[t % 3][:len(batches[t].key)] = engine_requests(batches[t].req)
            ring.submit(t % 3, len(batches[t].key), batches[t].now)

        def collect(t):
            ring.wait(t % 3)
            got[t] = ring.res[t % 3][:len(batches[t].key)].copy()

        def finish():
            for t in range(max(len(batches) - 3, 0), len(batches)):
                collect(t)
    else:
        dev = torch.device("cuda", 0)
        stream = torch.cuda.Stream(dev)
        d_req = [torch.from_numpy(engine_requests(b.req).view(np.uint8)).to(dev) for b in batches]
        d_res = [torch.zeros(len(b.key) * 32, dtype=torch.uint8, device=dev) for b in batches]
        torch.cuda.synchronize()

        def submit(t):
            lim.submit_device(len(batches[t].key), d_req[t].data_ptr(), d_res[t].data_ptr(), stream.cuda_stream)

        def finish():
            lim.join(stream.cuda_stream)
            stream.synchronize()
            for t in range(len(batches)):
                got[t] = d_res[t].cpu().numpy().view(tc.RES_DTYPE)

    for t in range(N_BEFORE):
        submit(t)
    assert st.get(cas_key, cas_now) == v
    assert st.compare_and_swap_with_ttl(cas_key, v, v + 1000, 60 * S, cas_now) is True
    st.save_begin(path)
    for t in range(N_BEFORE, len(batches)):
        submit(t)
    assert st.save_wait() == cut_len
    finish()
    for t, b in enumerate(batches):
        bad = first_mismatch(want[t], got[t], b.req)
        assert bad is None, "batch %d: %s" % (t, bad)
    hashes = tc.hash_key_ids(np.array(hot, np.uint64))
    for k, h in zip(hot, hashes.tolist()):
        assert st.peek(int(h)) == ora.entry("k:%d" % k), k
    assert_totals(st, want, ora.len(), ora.expired_writes())
    st.close()

    fresh = tc.ManualStore(capacity=100, created_ns=T0, max_batch=nmax)
    fresh.load(path)
    for k, h in zip(hot, hashes.tolist()):
        assert fresh.peek(int(h)) == cut[k], k
    assert_totals(fresh, want[:N_BEFORE], cut_len, cut_expired)
    fresh.close()


def assert_totals(st, want, n_entries, expired_hits):
    """the counters after the result rows `want` and the successful compare-and-swap, which counts as one allowed
    (mutating) operation, as the reference's stores count their operations for the sweep policies"""
    s, w = st.stats(), np.concatenate(want)
    ok = w["status"] == 0
    assert {f: s[f] for f in ("allowed", "denied", "errors", "len", "expired_hits")} == \
        {"allowed": int(w["allowed"].sum()) + 1, "denied": int((ok & (w["allowed"] == 0)).sum()),
         "errors": int((~ok).sum()), "len": n_entries, "expired_hits": expired_hits}
