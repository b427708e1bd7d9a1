"""Entry points that fail return an error, release what they made and leave the engine usable: later calls succeed and
stay bit-identical to the oracle.  Failures come only from requests no H100 can satisfy or from values validation
rejects; nothing fills the device's memory and nothing faults.  The scenarios with a peer-memory loop-back run
tests/failed_calls_worker.py in a child process (see test_gpu_p2p_skew.py for why); they pin the K1 pipeline to the
engine's own choice."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu


def test_create_beyond_device_memory_fails_cleanly():
    """max_batch = 2^31: the request staging buffer alone is 96 GiB, after the streams, events and table were made.
    Every attempt fails; an engine made afterwards replays a trace bit-identically."""
    import throttlecrab_b200 as tc
    import traces
    from gpu_util import first_mismatch, replay_both
    for _ in range(3):
        with pytest.raises(RuntimeError):
            tc.ManualStore(capacity=1000, created_ns=traces.T0, max_batch=1 << 31)
    req = traces.config1(n=20_000)
    res_o, res_e, _, _ = replay_both(req, capacity=1000, batch=4096)
    assert first_mismatch(res_o, res_e, req) is None


def denied_counts(ereq, res):
    d = (res["status"] == 0) & (res["allowed"] == 0)
    keys, cnt = np.unique(ereq["key_hash"][d], return_counts=True)
    return {int(k): int(c) for k, c in zip(keys, cnt)}


def test_rejected_track_denied_keeps_counts():
    """gcra_track_denied(2^28) would need a table of 2^32 entries: rejected, and tracking goes on with the counts it
    had.  Batches of every pipeline (small, sort-size, index-order-size) stay exact and keep counting."""
    import oracle
    import throttlecrab_b200 as tc
    import traces
    from gpu_util import engine_requests, first_mismatch
    sizes = [20_000, 100, 4096, 1 << 15, 100]
    req = traces.config4(n_keys=60, n_ticks=1, tick_size=sum(sizes), hot=10)
    ereq = engine_requests(req)
    want = oracle.OracleStore(oracle.PERIODIC, capacity=1000, created_ns=traces.T0, p0=10**9).replay(req)
    st = tc.ManualStore(capacity=1000, created_ns=traces.T0, max_batch=1 << 15)
    lim = tc.RateLimiter(st)
    st.track_denied(100)
    res = np.empty(len(req), tc.RES_DTYPE)
    ends = np.cumsum(sizes)
    lim.rate_limit_batch(ereq[:ends[0]], out=res[:ends[0]])
    before = dict(st.top_denied(100)[0])
    assert before and before == denied_counts(ereq[:ends[0]], res[:ends[0]])
    with pytest.raises(tc.Internal, match="max_keys"):
        st.track_denied(1 << 28)
    assert dict(st.top_denied(100)[0]) == before
    for a, b in zip(ends[:-1], ends[1:]):
        lim.rate_limit_batch(ereq[a:b], out=res[a:b])
        assert dict(st.top_denied(100)[0]) == denied_counts(ereq[:b], res[:b])
    assert first_mismatch(want, res, req) is None
    st.track_denied(0)
    with pytest.raises(tc.Internal, match="track_denied first"):
        st.top_denied(10)


def run_worker(scenario, timeout=900):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "failed_calls_worker.py"), scenario],
                         capture_output=True, text=True, timeout=timeout, env=env)
    assert out.returncode == 0 and scenario + " ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_failed_p2p_prepare_leaves_the_engine_usable(k1_path):
    """gcra_p2p_prepare(world = 16, cap_rows = 2^24) needs an 80 GiB window and fails; the same engine then runs
    index-order batches and a 2-engine loop-back tick, both exact."""
    run_worker("p2p")


@pytest.mark.parametrize("k1_path", ["auto"], indirect=True)
def test_engine_lifecycle(k1_path):
    """20 rounds of 3 engines that use ring modes 0, 1 and 2, a policy table, denied tracking, a loop-back tick,
    snapshot save and restore and a growing table, then are destroyed: every call succeeds, every result is exact."""
    run_worker("lifecycle")
