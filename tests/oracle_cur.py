"""`cur` of every decision (rate_limiter.rs:208: new_tat if allowed, else the tat the request started from), read off
the CPU oracle's own store around each call -- what a 16-byte engine result carries.

The oracle reports the 32-byte result only; its store holds the rest.  Per request, before the call,
Store::get (the oracle's `get`: the value of a live entry, rate_limiter.rs:151) gives the stored tat; after the call:
  allowed  -> cur = new_tat, which the call has just written (the entry's tat);
  denied   -> cur = the tat the request started from: max(stored, now - dvt) when the entry was live, else now - ei
              (rate_limiter.rs:158-166, saturating; ei / dvt from the oracle's own derivation);
  an error -> 0 (no decision).
Whatever this derives is checked where it is used: the 32-byte result expanded from it must equal the oracle's row."""
import numpy as np

import oracle

I64_MAX, I64_MIN = 2**63 - 1, -2**63


def _sat(x):
    return I64_MAX if x > I64_MAX else I64_MIN if x < I64_MIN else x


def rate_limit_cur(store, key, max_burst, count, period, quantity, now):
    """store.rate_limit(...) -> ((status, allowed, remaining, reset_after, retry_after), cur)"""
    stored = store.get(key, now)
    res = store.rate_limit(key, max_burst, count, period, quantity, now)
    if res[0] != 0:
        return res, 0
    if res[1]:
        return res, store.entry(key)[0]
    _, ei, dvt = oracle.derive(max_burst, count, period)
    return res, (max(stored, _sat(now - dvt)) if stored is not None else _sat(now - ei))


def replay_cur(store, req):
    """store.replay(req) one request at a time (key string "k:<id>"), also returning every request's cur."""
    req = np.ascontiguousarray(req, oracle.REQ_DTYPE)
    cols = [req[f].tolist() for f in ("key", "max_burst", "count_per_period", "period", "quantity", "now_ns")]
    rows, cur = [], []
    for k, b, c, p, q, now in zip(*cols):
        r, x = rate_limit_cur(store, "k:%d" % k, b, c, p, q, now)
        rows.append(r)
        cur.append(x)
    out = np.zeros(len(req), oracle.RES_DTYPE)
    if rows:
        st, al, rem, reset, retry = zip(*rows)
        out["status"], out["allowed"] = st, al
        out["remaining"], out["reset_after_ns"], out["retry_after_ns"] = rem, reset, retry
    return out, np.array(cur, np.int64)
