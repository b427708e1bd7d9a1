"""Helpers shared by the GPU parity tests: engine vs oracle on the same trace."""
import numpy as np

import oracle
import throttlecrab_b200 as tc
import traces


def engine_requests(req):
    """Trace rows (key = key id) -> engine rows (key_hash = hash of "k:<id>")."""
    out = np.empty(len(req), tc.REQ_DTYPE)
    out["key_hash"] = tc.hash_key_ids(req["key"])
    for f in ("max_burst", "count_per_period", "period", "quantity", "now_ns"):
        out[f] = req[f]
    return out


def assert_universe_collision_free(n_keys):
    h = tc.hash_key_ids(np.arange(n_keys, dtype=np.uint64))
    assert len(np.unique(h)) == n_keys, "64-bit key hashes collide inside the synthetic universe"
    return h


def replay_both(req, capacity, batch, max_batch=None, store_cls=None, oracle_kind=oracle.PERIODIC,
                oracle_p0=10**9):
    """Run the whole trace through the oracle (one call at a time) and through the engine in
    batches of `batch`; returns (res_oracle, res_engine, oracle_store, engine_store)."""
    st_o = oracle.OracleStore(oracle_kind, capacity=capacity, created_ns=traces.T0, p0=oracle_p0)
    res_o = st_o.replay(req)
    store_cls = store_cls or tc.ManualStore
    st_e = store_cls(capacity=capacity, created_ns=traces.T0, max_batch=max_batch or max(batch, 4096))
    lim = tc.RateLimiter(st_e)
    ereq = engine_requests(req)
    res_e = np.empty(len(req), tc.RES_DTYPE)
    for a in range(0, len(req), batch):
        lim.rate_limit_batch(ereq[a:a + batch], out=res_e[a:a + batch])
    return res_o, res_e, st_o, st_e


def replay_skipping_refused(store, req, res_e, what=""):
    """For paths that may refuse rows (GCRA_INTERNAL: table full, residue beyond max_batch): feed the oracle `store`
    only the rows the engine did NOT refuse, and require each of them to be bit-identical.  A refused row leaves no
    trace in the engine, so this is exact.  Returns the indices of the refused rows."""
    refused = np.nonzero(res_e["status"] == tc.INTERNAL)[0]
    keep = np.ones(len(req), bool)
    keep[refused] = False
    res_o = store.replay(req[keep])
    bad = first_mismatch(res_o, res_e[keep], req[keep])
    assert bad is None, what + bad + " (%d refused rows skipped)" % len(refused)
    return refused


def first_mismatch(res_o, res_e, req=None):
    a = res_o.view(np.uint8).reshape(len(res_o), -1)
    b = res_e.view(np.uint8).reshape(len(res_e), -1)
    bad = np.nonzero((a != b).any(axis=1))[0]
    if len(bad) == 0:
        return None
    i = int(bad[0])
    return "row %d of %d mismatching rows: oracle=%s engine=%s req=%s" % (
        i, len(bad), res_o[i], res_e[i], None if req is None else req[i])
