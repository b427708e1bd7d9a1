"""Shapes that stress the stable radix sort of the slot keys (one digit-count launch, then one sweep per pass with
decoupled look-back over 4096-key tiles), through the public API.

Every row of a scenario is compared bit-exact with ONE oracle store that replays the same rows in submission order.
The sort must reproduce the one stable order of (slot << 32 | row) by slot, so any misplaced key -- a wrong tile
offset, a digit base, a tile boundary, a pass count -- shows up as a request decided against the wrong state.
The sort serves the sort pipeline (every batch) and the index-order pipeline's tail (its residue, whose size only
the device knows); the conftest modes run both."""
import numpy as np
import pytest

import oracle
import throttlecrab_b200 as tc
import traces
from gpu_util import engine_requests, first_mismatch

pytestmark = pytest.mark.gpu

T0 = traces.T0
MS = 1_000_000
TILE = 4096                         # keys per sweep tile (SORT_TILE)


def rows(key, now_ns, policy=None, quantity=1):
    req = np.zeros(len(key), traces.REQ_DTYPE)
    req["key"] = key
    traces.fill_policy(req, (req["key"] % np.uint64(8)).astype(np.int64) if policy is None else np.broadcast_to(policy, len(key)))
    req["quantity"] = quantity
    req["now_ns"] = now_ns
    return req


def check_universe(key_ids):
    ids = np.unique(np.asarray(key_ids, np.uint64))
    assert len(np.unique(tc.hash_key_ids(ids))) == len(ids), "64-bit key hashes collide inside the trace"


def run_batches(st, capacity, batches):
    """Each array of `batches` is one rate_limit_batch call on `st`; all rows against one oracle store."""
    req = np.concatenate(batches)
    check_universe(req["key"])
    lim = tc.RateLimiter(st)
    ereq = engine_requests(req)
    res = np.empty(len(req), tc.RES_DTYPE)
    a = 0
    for b in batches:
        lim.rate_limit_batch(ereq[a:a + len(b)], out=res[a:a + len(b)])
        a += len(b)
    want = oracle.OracleStore(oracle.PERIODIC, capacity=capacity, created_ns=T0, p0=10**9).replay(req)
    bad = first_mismatch(want, res, req)
    assert bad is None, bad
    return want


def test_one_key_in_every_row():
    """2^20 rows on one key: every tile holds a single digit, so each tile's offset of that digit comes from the
    longest look-back chain there is; in the index-order pipeline all rows but the first are the residue."""
    n = 1 << 20
    st = tc.ManualStore(capacity=1000, created_ns=T0, max_batch=n)
    rng = np.random.default_rng(1)
    q = rng.choice([0, 1, 1, 2], n)
    want = run_batches(st, 1000, [rows(np.full(n, 7, np.uint64), T0 + MS, policy=0, quantity=1),
                                  rows(np.full(n, 7, np.uint64), T0 + 5_000 * MS, policy=0, quantity=q)])
    assert want["allowed"].sum() > 0 and (want["allowed"] == 0).sum() > 0


@pytest.mark.parametrize("n", [256, TILE - 1, TILE, TILE + 1, (1 << 20) + 1])
def test_tile_boundaries(n):
    """Batch sizes around the tile (a partial last tile, an exact one, one key in the last tile), the smallest
    batch that is sorted, and one key past 2^20 (257 tiles).  Keys repeat, so equal slots meet across tiles."""
    rng = np.random.default_rng(n)
    n_keys = max(n // 3, 8)
    st = tc.ManualStore(capacity=n_keys, created_ns=T0, max_batch=n)
    batches = []
    for t in range(3):
        key = rng.integers(0, n_keys, n).astype(np.uint64)
        batches.append(rows(key, T0 + (t + 1) * 40 * MS, quantity=rng.choice([0, 1, 1, 1, 2, 5], n)))
    run_batches(st, n_keys, batches)


def test_uniform_keys_over_a_large_space():
    """2^19-row batches of uniform keys drawn from 2^40 ids: nearly every row has a key of its own, the digits of
    a tile spread over all bins, and the table is large enough for three passes."""
    n = 1 << 19
    rng = np.random.default_rng(3)
    st = tc.ManualStore(capacity=3 * n, created_ns=T0, max_batch=n)
    batches = []
    for t in range(3):
        key = rng.integers(0, 1 << 40, n).astype(np.uint64)
        if t == 2:
            key[: n // 2] = batches[0]["key"][: n // 2]        # revisit earlier keys
        batches.append(rows(key, T0 + (t + 1) * MS))
    run_batches(st, 3 * n, batches)
    assert st.stats()["table_slots"] > 1 << 18              # > 18 slot bits: three passes of at most 9 bits


def test_tight_table_grows_between_batches():
    """GCRA_FLAG_TIGHT_TABLE from 16 entries, batches whose keys reach further each time: the table grows between
    batches, so the slot bits and the number of passes (1 -> 2 -> 3) change from one batch to the next."""
    rng = np.random.default_rng(4)
    st = tc.ManualStore(capacity=16, created_ns=T0, max_batch=1 << 17, flags=tc._native.FLAG_TIGHT_TABLE)
    batches = []
    for t, (size, reach) in enumerate([(1 << 12, 40), (1 << 12, 300), (1 << 13, 3000), (1 << 15, 30_000),
                                       (1 << 17, 1_000_000), (1 << 17, 1_000_000), (1 << 17, 1_000_000)]):
        key = rng.integers(0, reach, size).astype(np.uint64)
        batches.append(rows(key, T0 + (t + 1) * 20 * MS, quantity=rng.choice([0, 1, 1, 2], size)))
    run_batches(st, 16, batches)
    s = st.stats()
    assert s["grows"] >= 3
    assert s["table_slots"] > 1 << 18


@pytest.mark.parametrize("k1_path", ["index"], indirect=True)
def test_index_order_residue_sizes(k1_path):
    """Index-order batches whose residue (the rows behind the first state change of their key) is empty, one row,
    and most of the batch: the tail sorts a count it only finds on the device, 0 included."""
    B = 1 << 14
    rng = np.random.default_rng(6)
    st = tc.ManualStore(capacity=1 << 15, created_ns=T0, max_batch=B)
    sat = (1_000 + rng.integers(0, 50, B)).astype(np.uint64)
    batches = [
        rows(sat, T0 + MS, policy=3),                                  # 50 keys (burst 5) exhausted: large residue
        rows(rng.permutation(sat), T0 + MS, policy=3),                 # all denied, nothing changes: residue 0
        rows(rng.permutation(sat), T0 + MS, policy=3),                 # again, behind an empty residue
    ]
    one = np.arange(10_000, 10_000 + B, dtype=np.uint64)
    one[B - 1] = one[B // 2]                                           # one key twice: residue 1
    batches.append(rows(one, T0 + 2 * MS, policy=0))
    burst = np.repeat(np.arange(50_000, 50_000 + B // 16, dtype=np.uint64), 16)
    batches.append(rows(rng.permutation(burst), T0 + 3 * MS, policy=0))   # 16 rows per fresh key: residue 15/16
    batches.append(rows(sat, T0 + 3 * MS, policy=3))                      # residue 0 after the large one
    batches.append(rows(rng.permutation(burst), T0 + 4 * MS, policy=0))
    run_batches(st, 1 << 15, batches)
    assert st.stats()["index_batches"] >= len(batches)
