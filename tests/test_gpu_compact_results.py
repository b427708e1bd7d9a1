"""16-byte results on the compact-request path, against the oracle and against the 32-byte path.

Two engines run the same compact trace: one returns gcra_result rows (32 bytes), the other gcra_result16 rows
(`cur`, status, allowed).  Every 16-byte row must carry the oracle's `cur` (rate_limiter.rs:208, read off the oracle's
store by oracle_cur.py), status and verdict; every row expanded on the host (gcra_expand_results16) must equal the
32-byte engine's row byte for byte; and the two engines must end with the same table (sampled gcra_peek, also against the oracle's entries), the same counters and
the same top denied keys (the metrics pass reads status and allowed at their 16-byte offsets).  The traces reach every
kernel that writes a result row of a single-GPU batch: the one-CTA small batch, ingest / probe error rows, the sorted
decide and its residue tail by row id, the hot-run kernels (one CTA and one cluster per run) with their finite-state
rounds, and pass B of the index-order pipeline.  (Pass C refuses residue rows only beyond max_batch, which a
single batch cannot reach.)"""
import functools

import numpy as np
import pytest

import oracle
import oracle_cur
import throttlecrab_b200 as tc
import traces

pytestmark = pytest.mark.gpu

T0 = traces.T0
MS = 1_000_000
I32_MAX = 2**31 - 1
P0, P3, P6 = 0, 3, 6                # traces.POLICIES: (100, 1000, 60), (5, 10, 60), (1, 3, 3600)
POLICY_TABLE = np.concatenate([traces.POLICIES, [(0, 10, 60),                  # 8: invalid (max_burst = 0)
                                                 (2**32, 1, 2**63 - 1)]])      # 9: Duration * u32 overflows
NPOL = len(POLICY_TABLE)
# gcra_get_stats fields that follow from the decisions alone.  Not stash_entries: when two new keys race for the last
# free slot of a bucket within one batch, which of them lands in the stash is up to the hardware; and on the ring not
# the pipeline statistics (index_batches, residue_*, drains, path_switches), which follow the residue feedback's timing.
STAT_DECISIONS = ("len", "occupied_slots", "table_slots", "allowed", "denied", "errors", "expired_hits", "sweeps",
                  "swept", "grows", "purges")
STAT_BLOCKING = STAT_DECISIONS + ("index_batches", "residue_rows", "residue_batches", "drains", "path_switches")


def policies():
    pol = np.zeros(NPOL, tc.POLICY_DTYPE)
    pol["max_burst"], pol["count_per_period"], pol["period"] = POLICY_TABLE.T
    return pol


class Batch:
    """One compact batch: trace key ids, policy indices (>= NPOL: beyond the table), quantities, one clock."""

    def __init__(self, key, pol, q, now):
        self.key = np.asarray(key, np.uint64)
        self.pol = np.asarray(pol, np.int64)
        self.q = np.asarray(q, np.int64)
        self.now = int(now)
        self.req16 = np.zeros(len(self.key), tc.REQ16_DTYPE)
        self.req16["key_hash"] = tc.hash_key_ids(self.key)
        self.req16["quantity"] = self.q
        self.req16["policy"] = self.pol

    def far(self):
        return self.pol >= NPOL


def sprinkle(rng, key, pol, q):
    """Edge rows in a batch: the invalid and the overflowing policy, indices beyond the table (with q >= 0, so that
    the policy check is what fails), negative quantities and 2^31 - 1."""
    pol, q = pol.copy(), q.copy()
    e = rng.random(len(key))
    pol[e < 0.002] = 8
    pol[(e >= 0.002) & (e < 0.004)] = 9
    far = (e >= 0.004) & (e < 0.006)
    pol[far] = rng.choice([NPOL, NPOL + 1, 2**32 - 1], int(far.sum()))
    q[far] = np.abs(q[far])
    neg = (e >= 0.006) & (e < 0.008)
    q[neg] = rng.choice([-1, -2**31], int(neg.sum()))
    q[(e >= 0.008) & (e < 0.009)] = I32_MAX
    return key, pol, q


def oracle_run(batches, capacity, boundary=None):
    """The oracle over the batches in order (rows beyond the table are refused with GCRA_INTERNAL and not replayed):
    (32-byte rows, cur, the store).  boundary(store, t) runs before batch t."""
    ora = oracle.OracleStore(oracle.PERIODIC, capacity=capacity, created_ns=T0, p0=10**9)
    want, cur = [], []
    for t, b in enumerate(batches):
        if boundary is not None:
            boundary(ora, t)
        far = b.far()
        req = np.zeros(int((~far).sum()), traces.REQ_DTYPE)
        req["key"] = b.key[~far]
        p = POLICY_TABLE[b.pol[~far]]
        req["max_burst"], req["count_per_period"], req["period"] = p[:, 0], p[:, 1], p[:, 2]
        req["quantity"] = b.q[~far]
        req["now_ns"] = b.now
        w = np.zeros(len(b.key), tc.RES_DTYPE)
        c = np.zeros(len(b.key), np.int64)
        w["status"][far] = tc.INTERNAL
        w[~far], c[~far] = oracle_rows(ora, req)
        want.append(w)
        cur.append(c)
    return np.concatenate(want), np.concatenate(cur), ora


def oracle_rows(ora, req):
    out, cur = oracle_cur.replay_cur(ora, req)
    return out.view(tc.RES_DTYPE), cur


def new_engine(capacity, max_batch, flags=0):
    st = tc.ManualStore(capacity=capacity, created_ns=T0, max_batch=max_batch, flags=flags)
    lim = tc.RateLimiter(st)
    lim.set_policies(policies())
    st.track_denied(4096)
    return st, lim


def expand(batches, res16, table=None):
    table = policies() if table is None else table
    out, a = [], 0
    for b in batches:
        out.append(tc.expand_results16(b.req16, b.now, table, res16[a:a + len(b.key)]))
        a += len(b.key)
    return np.concatenate(out)


def first_bad(a, b):
    x = a.view(np.uint8).reshape(len(a), -1)
    y = b.view(np.uint8).reshape(len(b), -1)
    bad = np.nonzero((x != y).any(axis=1))[0]
    return None if len(bad) == 0 else int(bad[0])


def assert_pair(batches, want, cur, res32, res16, st32, st16, ora, sample_keys, stat_fields=STAT_BLOCKING, table=None):
    """16-byte rows == the oracle's (cur, status, allowed); expanded rows == the 32-byte engine's == the oracle's;
    the two engines' tables, counters and top denied keys agree (and the tables with the oracle's entries).
    `table`: the policy table both engines ran with (default: this file's)."""
    assert len(res16) == len(res32) == len(want)
    got = np.stack([res16["cur_tat_ns"], res16["status"].astype(np.int64), res16["allowed"].astype(np.int64)], 1)
    exp = np.stack([cur, want["status"].astype(np.int64), want["allowed"].astype(np.int64)], 1)
    bad = np.nonzero((got != exp).any(axis=1))[0]
    assert len(bad) == 0, "16-byte row %d: engine %s, oracle (cur, status, allowed) %s" % (bad[0], got[bad[0]], exp[bad[0]])
    i = first_bad(want, res32)
    assert i is None, "32-byte row %d: oracle %s engine %s" % (i, want[i], res32[i])
    full = expand(batches, res16, table)
    i = first_bad(res32, full)
    assert i is None, "expanded row %d: 32-byte engine %s expanded %s" % (i, res32[i], full[i])
    s32, s16 = st32.stats(), st16.stats()
    s32, s16 = {f: s32[f] for f in stat_fields}, {f: s16[f] for f in stat_fields}
    assert s32 == s16, (s32, s16)
    assert st32.top_denied(64) == st16.top_denied(64)
    assert len(st16.top_denied(64)[0]) > 0
    hashes = tc.hash_key_ids(np.asarray(sample_keys, np.uint64))
    for k, h in zip(sample_keys, hashes):
        e = st16.peek(int(h))
        assert e == st32.peek(int(h)) == ora.entry("k:%d" % k), k
    assert set(np.unique(want["status"]).tolist()) >= {0, 1, 2, 3}
    assert want["allowed"].any() and ((want["status"] == 0) & (want["allowed"] == 0)).any()


def check_universe(keys):
    ids = np.unique(np.asarray(keys, np.uint64))
    assert len(np.unique(tc.hash_key_ids(ids))) == len(ids), "64-bit key hashes collide inside the trace"


# ---------------------------------------------------------------------------------------------------------------
# batch sizes 1, 200 (single-CTA kernel), 4096 and 2^15 + 1, through the device-resident entry points
# ---------------------------------------------------------------------------------------------------------------
SIZES = [1, 200, 4096, (1 << 15) + 1] * 3
TOGGLER, SPENDER = 1_000_000, 1_000_001


@functools.lru_cache(maxsize=None)
def sizes_trace():
    """Uniform keys over 3000 (policy = key % 8); in the two larger sizes a max_burst = 1 key with zero quantities
    whose state toggles on every row (a long run of 300 rows at 4096, a giant run of 5000 at 2^15 + 1: finite-state
    rounds), and a P0 key spending its burst (500 rows: the residue of the index-order pipeline)."""
    rng = np.random.default_rng(21)
    batches, now = [], T0
    for n in SIZES:
        now += 50 * MS
        key = rng.integers(0, 3000, n).astype(np.uint64)
        pol = (key % np.uint64(8)).astype(np.int64)
        q = traces.quantities(rng.integers(0, 2**63, n, dtype=np.uint64))
        if n >= 4096:
            rows = rng.permutation(n)
            tog = rows[:300 if n == 4096 else 5000]
            spend = rows[len(tog):len(tog) + 500]
            key[tog], pol[tog], q[tog] = TOGGLER, P6, 0
            key[spend], pol[spend], q[spend] = SPENDER, P0, 1
        batches.append(Batch(*sprinkle(rng, key, pol, q), now))
    want, cur, ora = oracle_run(batches, 4000)
    return batches, want, cur, ora


def test_batch_sizes_device(k1_path):
    import torch
    batches, want, cur, ora = sizes_trace()
    check_universe(np.append(np.arange(3000), [TOGGLER, SPENDER]))
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    out = {}
    for r16 in (False, True):
        st, lim = new_engine(4000, 1 << 16)
        rsz = 16 if r16 else 32
        res = []
        with torch.cuda.stream(stream):
            for b in batches:
                d_req = torch.from_numpy(b.req16.view(np.uint8)).to(dev)
                d_res = torch.zeros(len(b.key) * rsz, dtype=torch.uint8, device=dev)
                stream.synchronize()
                lim.rate_limit_batch16_device(len(b.key), d_req.data_ptr(), b.now, d_res.data_ptr(), stream.cuda_stream,
                                              compact_results=r16)
                stream.synchronize()
                res.append(d_res.cpu().numpy().view(tc.RES16_DTYPE if r16 else tc.RES_DTYPE))
        out[r16] = (st, np.concatenate(res))
    (st32, res32), (st16, res16) = out[False], out[True]
    assert_pair(batches, want, cur, res32, res16, st32, st16, ora, list(range(0, 3000, 7)) + [TOGGLER, SPENDER])
    if k1_path == "index":
        assert st16.stats()["index_batches"] == 2 * len(SIZES) // 4


# ---------------------------------------------------------------------------------------------------------------
# 2^20-row Zipf ticks over fresh keys, through the host-buffer entry points
# ---------------------------------------------------------------------------------------------------------------
ZIPF_KEYS = 1_000_000


@functools.lru_cache(maxsize=None)
def zipf_trace():
    """Two config2 ticks of 2^20 rows over 1 M keys that start without entries: the hot keys spend their bursts
    inside the tick (the hottest has ~73 K rows: a giant run, a residue tail), then saturate."""
    tr = traces.config2(n_keys=ZIPF_KEYS, n_ticks=2, tick_size=1 << 20)
    rng = np.random.default_rng(22)
    batches = []
    for t in range(2):
        sl = tr[t * (1 << 20):(t + 1) * (1 << 20)]
        key = sl["key"].copy()
        batches.append(Batch(*sprinkle(rng, key, (key % np.uint64(8)).astype(np.int64), sl["quantity"].copy()),
                             int(sl["now_ns"][0])))
    want, cur, ora = oracle_run(batches, ZIPF_KEYS)
    return batches, want, cur, ora


def test_zipf_tick_host(k1_path):
    batches, want, cur, ora = zipf_trace()
    u, c = np.unique(batches[0].key, return_counts=True)
    assert c.max() > 4096
    check_universe(u)
    out = {}
    for r16 in (False, True):
        st, lim = new_engine(ZIPF_KEYS, 1 << 20)
        out[r16] = (st, np.concatenate([lim.rate_limit_batch16(b.req16, b.now, compact_results=r16) for b in batches]))
    (st32, res32), (st16, res16) = out[False], out[True]
    hot = u[np.argsort(-c)[:50]].tolist()
    assert_pair(batches, want, cur, res32, res16, st32, st16, ora, hot + u[::4999].tolist())
    if k1_path != "sort":
        assert st16.stats()["index_batches"] == 2


# ---------------------------------------------------------------------------------------------------------------
# a tight table that grows and purges between batches
# ---------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def tight_trace():
    """Keys arrive progressively (a 16-entry tight table grows many times); every batch also has fresh keys whose
    only request is denied (q = 20 > max_burst: a slot without an entry, reclaimed by a purge); clocks jump so that
    entries expire and every third batch boundary sweeps."""
    rng = np.random.default_rng(23)
    n_keys, B, n_batches = 20_000, 2048, 90
    batches, now, fresh = [], T0, 10_000_000
    for t in range(n_batches):
        now += int(rng.choice([1000, 2 * MS, 700 * MS, 20_000 * MS]))
        key = (rng.integers(0, n_keys, B) * (t + 1) / n_batches).astype(np.uint64)
        pol = (key % np.uint64(8)).astype(np.int64)
        q = rng.choice([0, 1, 1, 1, 2, 5], B)
        key[:40] = np.arange(fresh, fresh + 40, dtype=np.uint64)
        fresh += 40
        pol[:40], q[:40] = 2, 20                     # (10, 100, 60): denied, no entry
        batches.append(Batch(*sprinkle(rng, key, pol, q), now))

    def boundary(ora, t):
        if t and t % 3 == 0:
            ora.force_sweep(batches[t - 1].now)
    want, cur, ora = oracle_run(batches, 16, boundary)
    return batches, want, cur, ora, fresh


def test_tight_table_grows_and_purges(k1_path):
    batches, want, cur, ora, fresh = tight_trace()
    check_universe(np.append(np.arange(20_000), np.arange(10_000_000, fresh)))
    out = {}
    for r16 in (False, True):
        st, lim = new_engine(16, 2048, flags=tc._native.FLAG_TIGHT_TABLE)
        res = []
        for t, b in enumerate(batches):
            if t and t % 3 == 0:
                st.sweep(batches[t - 1].now)
            res.append(lim.rate_limit_batch16(b.req16, b.now, compact_results=r16))
        out[r16] = (st, np.concatenate(res))
    (st32, res32), (st16, res16) = out[False], out[True]
    assert_pair(batches, want, cur, res32, res16, st32, st16, ora, list(range(0, 20_000, 97)))
    s = st16.stats()
    assert s["grows"] >= 2 and s["purges"] >= 1 and s["sweeps"] > 0, s
    assert s["len"] == ora.len()


# ---------------------------------------------------------------------------------------------------------------
# the ring: mode 2 against mode 1 over 72 pipelined 2^15-row slots with overlapped tails
# ---------------------------------------------------------------------------------------------------------------
T = 1 << 15
RING_BATCHES = 72
SAT_KEYS, BURST_KEYS, BURST_ROWS = 50, 328, 16


@functools.lru_cache(maxsize=None)
def ring_trace():
    """Saturated P3 keys with 328 fresh burst-spending P0 keys x 16 rows in every batch (a residue of ~15 %: the
    index-order pipeline keeps overlapping stage 2 with the previous tail) and a toggling max_burst = 1 key."""
    rng = np.random.default_rng(24)
    batches, now, fresh = [], T0, 10_000_000
    for _ in range(RING_BATCHES):
        now += MS
        key = (5_000_000 + rng.integers(0, SAT_KEYS, T)).astype(np.uint64)
        pol, q = np.full(T, P3), np.ones(T, np.int64)
        b = np.repeat(np.arange(fresh, fresh + BURST_KEYS, dtype=np.uint64), BURST_ROWS)
        fresh += BURST_KEYS
        key[:len(b)], pol[:len(b)] = b, P0
        key[len(b):len(b) + 64], pol[len(b):len(b) + 64], q[len(b):len(b) + 64] = TOGGLER, P6, 0
        perm = rng.permutation(T)
        batches.append(Batch(*sprinkle(rng, key[perm], pol[perm], q[perm]), now))
    want, cur, ora = oracle_run(batches, 200_000)
    return batches, want, cur, ora, fresh


def ring_run(ring, batches):
    """Submit every batch through `ring`, paced as a server drives it (wait for batch t - slots + 1 after submitting
    batch t); returns the results, concatenated."""
    S = ring.slots
    out = []

    def collect(j):
        ring.wait(j % S)
        out.append(ring.res[j % S][:len(batches[j].key)].copy())

    for t, b in enumerate(batches):
        ring.req[t % S][:len(b.key)] = b.req16
        ring.submit(t % S, len(b.key), b.now)
        if t - S + 1 >= 0:
            collect(t - S + 1)
    for j in range(max(len(batches) - S + 1, 0), len(batches)):
        collect(j)
    return np.concatenate(out)


def test_ring_mode2_against_mode1(k1_path):
    batches, want, cur, ora, fresh = ring_trace()
    check_universe(np.concatenate([5_000_000 + np.arange(SAT_KEYS), np.arange(10_000_000, fresh), [TOGGLER]]))
    out = {}
    for mode in (True, 2):
        st, lim = new_engine(200_000, T)
        ring = tc.Ring(lim, slots=4, slot_capacity=T, compact=mode)
        assert ring.res[0].dtype == (tc.RES16_DTYPE if mode == 2 else tc.RES_DTYPE)
        assert (st._L.gcra_ring_results(st._h, 0) is None) == (mode == 2)
        assert (st._L.gcra_ring_results16(st._h, 0) is None) == (mode != 2)
        out[mode] = (st, ring_run(ring, batches))
    (st32, res32), (st16, res16) = out[True], out[2]
    assert_pair(batches, want, cur, res32, res16, st32, st16, ora,
                list(range(5_000_000, 5_000_000 + SAT_KEYS)) + list(range(10_000_000, fresh, 101)) + [TOGGLER],
                stat_fields=STAT_DECISIONS)
    s = st16.stats()
    print("ring mode 2, %s: %s" % (k1_path, {f: s[f] for f in ("path_switches", "drains", "index_batches")}))
    if k1_path == "index":
        assert s["index_batches"] == RING_BATCHES, s
