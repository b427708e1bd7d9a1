"""The peer-memory tick (gcra_p2p_*) under skew, with `world` engines in one process on one GPU: one key flooding a
whole multi-GPU tick, a residue larger than the engine's batch capacity, a table that fills up inside a tick, an
empty rank -- and, on one engine, the wrap of the 32-bit batch epoch.  Every decision is checked against ONE oracle
store fed the union trace in global order; where the engine may refuse rows (GCRA_INTERNAL), the oracle replays
only the others (a refused row leaves no trace) and the refused rows themselves are checked against the rule that
refuses them.

The p2p scenarios run tests/p2p_loopback_worker.py in a child process with CUDA_DEVICE_MAX_CONNECTIONS=32 (see
test_gpu_sharded.test_peer_memory_pipeline_loopback_on_one_gpu).  A segmented tick always takes the index-order
pipeline, so the K1 pipeline is pinned to the engine's own choice: forcing one would run the same kernels again."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu


def run_worker(*args, timeout=1500):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "p2p_loopback_worker.py")] + [str(a) for a in args],
                         capture_output=True, text=True, timeout=timeout, env=env)
    assert out.returncode == 0 and "loopback ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    report = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])
    print(report)
    return report


# One key in every row of a tick whose owner batch (all segments together) spans 32768 256-row tiles: pass A adds 2
# per tile to the key's batch counter, 65536 in all -- the case a 16-bit counter reads as 0 ("alone on its key").
# Tick 1 on the fresh key (policy P0: burst 100), tick 2 1 ms later (saturated: all denied), tick 3 1 s later
# (about 16 tokens back).  max_batch = world x tick: the residue (every row behind the key's first state change)
# fits, so no row may be refused.
FLOOD = {
    "flood_2x2^22": (2, 1 << 22, ["--trace", "flood", "--n-ticks", 3, "--tick-ms", "0,1,1000"]),
    "flood_4x2^21": (4, 1 << 21, ["--trace", "flood", "--n-ticks", 3, "--tick-ms", "0,1,1000"]),
    # half the rows on the hot key, half on cold keys of the same owner: the hot key is in every tile among others
    "flood_mix_2x2^22": (2, 1 << 22, ["--trace", "flood_mix", "--n-ticks", 1, "--n-keys", 1_000_000]),
}


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
@pytest.mark.parametrize("name", list(FLOOD))
def test_flood_at_batch_counter_boundary(name, k1_path):
    world, tick, extra = FLOOD[name]
    # (capacity: every engine reserves table room for 1.25 x the rows it submits, up to 5.2 M, without growing)
    args = [world, tick, 0, "--max-batch", world * tick, "--capacity", 6_000_000] + extra
    rep = run_worker(*args)           # (the worker requires every row bit-identical, zero GCRA_INTERNAL)
    assert rep["refused"] == [0] * len(rep["rows"]) and rep["rows"] == [world * tick] * len(rep["rows"])
    assert all(e == 0 for tick_errors in rep["errors_delta"] for e in tick_errors)
    assert rep["len"] and sum(rep["len"]) == rep["oracle_len"]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_residue_beyond_max_batch_is_refused_exactly(k1_path):
    """4 ranks x 2^16 rows on one fresh key whose burst admits them all: every row changes the key's state, so all
    rows but the key's first go to the owner's residue -- 2^18 - 1 rows for a residue buffer of max_batch = 2^16.
    resolve_kernel answers GCRA_INTERNAL to the residue rows whose place in batch order is max_batch or later;
    those are the LAST rows of the tick in global order.  The next tick (2^14 rows per rank) fits and is exact."""
    world, tick, mb = 4, 1 << 16, 1 << 16
    rep = run_worker(world, tick, 0, "--trace", "flood", "--ticks", "%d/%d" % (tick, tick // 4), "--n-ticks", 2,
                     "--max-batch", mb, "--flood-policy", "10000000,1000,1", "--refusable")
    n = world * tick
    residue = n - 1                                  # every row behind row 0, the key's first state change
    expect = residue - mb
    assert expect > 0
    assert rep["refused"][0] == expect
    assert (rep["refused_first"][0], rep["refused_last"][0]) == (n - expect, n - 1)
    # only the key's owner refused anything, and counted each refusal as an error
    assert sorted(rep["errors_delta"][0]) == [0] * (world - 1) + [expect]
    assert rep["refused"][1] == 0 and rep["errors_delta"][1] == [0] * world
    assert rep["len"] and sum(rep["len"]) == rep["oracle_len"] == 1


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_table_full_inside_a_tick_with_an_empty_rank(k1_path):
    """Rank 0 submits nothing, and its engine starts with room for about 1 K keys; ranks 1-3 each send 2^15
    distinct new keys that rank 0 owns.  The owner reserves table room for what it submitted itself (0 rows +
    slack), so most new keys find no slot: those rows are refused, every other row is exact.  The next tick
    (only the admitted keys, sent again by the same ranks) finds the grown table and is exact."""
    world, tick = 4, 1 << 15
    rep = run_worker(world, tick, 0, "--trace", "fresh_to_owner", "--ticks", "0,%d" % tick, "--n-ticks", 2,
                     "--capacity", "1024,4000000", "--refusable")
    assert rep["rows"][0] == (world - 1) * tick
    assert rep["refused"][0] > 0, "the table never filled: this scenario tests nothing"
    assert rep["errors_delta"][0] == [rep["refused"][0], 0, 0, 0]
    assert rep["rows"][1] == rep["rows"][0] - rep["refused"][0]
    assert rep["refused"][1] == 0 and rep["errors_delta"][1] == [0] * world
    assert rep["len"][0] == rep["oracle_len"] == rep["rows"][1] and rep["len"][1:] == [0] * (world - 1)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_batch_epoch_wrap(k1_path, monkeypatch):
    """The index-order pipeline tags its per-slot marks with a 32-bit batch epoch; when the epoch wraps, every
    mark is cleared.  An engine started 4 batches before the wrap (GCRA_EPOCH0) runs 10 index-order batches of
    2^15 rows across it, with hot keys in every batch: bit-identical to the oracle and to an engine started at
    epoch 0."""
    import oracle
    import throttlecrab_b200 as tc
    import traces
    from gpu_util import engine_requests, first_mismatch
    n_keys, batch, n_batches = 40_000, 1 << 15, 10
    req = traces.config4(n_keys=n_keys, n_ticks=n_batches, tick_size=batch, hot=50)
    want = oracle.OracleStore(oracle.PERIODIC, capacity=n_keys, created_ns=traces.T0, p0=10**9).replay(req)
    ereq = engine_requests(req)
    got = {}
    for epoch0 in (2**32 - 4, None):
        if epoch0 is None:
            monkeypatch.delenv("GCRA_EPOCH0", raising=False)
        else:
            monkeypatch.setenv("GCRA_EPOCH0", str(epoch0))
        st = tc.ManualStore(capacity=n_keys, created_ns=traces.T0, max_batch=batch)
        lim = tc.RateLimiter(st)
        res = np.empty(len(req), tc.RES_DTYPE)
        for a in range(0, len(req), batch):
            lim.rate_limit_batch(ereq[a:a + batch], out=res[a:a + batch])
        assert st.stats()["index_batches"] == n_batches
        st.close()
        bad = first_mismatch(want, res, req)
        assert bad is None, "epoch0=%s: %s" % (epoch0, bad)
        got[epoch0] = res
    assert got[2**32 - 4].tobytes() == got[None].tobytes()
    assert want["allowed"].sum() > 0 and (want["allowed"] == 0).sum() > 0
