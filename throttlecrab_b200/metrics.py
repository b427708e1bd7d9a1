"""The server's GET /metrics (throttlecrab-server/src/metrics.rs): Prometheus text of the requests per transport, the
allowed, denied and error totals, and the top denied keys by name.

The rings decide most requests on the GPU and never hand their key strings to the host, so the counts and the names
come from the engine: with ring metrics on (gcra_ring_metrics) every ring submit counts its rows per transport and
names its denied keys from the slot's input, and the denied-key table (gcra_track_denied) counts the denials of every
batch.  What the host decides on its general paths (PING, a request that is not plain, a gRPC call on the general
HTTP/2 path, ...) the drivers record here: resp.process_connections, http.process_connections,
grpc_transport.process_connections and mixed.process_connections take a Metrics as `metrics`, and a Metrics is the
callable that GET /metrics serves.

ShardedMetrics serves the same text for N engines of one hash-sharded table (mixed.process_connections_sharded): each
engine counts its own ring slots and names the keys its connections saw denied (gcra_ring_metrics_sharded), the
denied counts are on the keys' owners, and a scrape joins the three.

Differences from the reference: ties in the top list are ordered by smaller key hash (the reference's order is its
HashMap's), and the table is pruned to its top max_denied_keys entries when queried, not on each update, so with more
than 3 x max_denied_keys distinct denied keys between two scrapes the lists may differ.  With ShardedMetrics, an
engine whose connections see more distinct denied keys between two scrapes than its name table holds (16 x
max_denied_keys, at least 1,024) leaves some of them unnamed; ShardedMetrics.full counts their denied rows.
"""
import time

import numpy as np

from . import NAME_TOO_LONG, NAME_UNKNOWN

MAX_KEY_LENGTH = 256                  # metrics.rs:12
MAX_DENIED_KEYS_LIMIT = 10_000        # metrics.rs:17
TRANSPORTS = {"redis": 0, "resp": 0, "http": 1, "grpc": 2}     # the engine's order: GCRA_PROTO_* - 1


def escape_label(s):
    """metrics.rs:213-230: a Prometheus label value; control characters (char::is_control: U+0000-001F, U+007F-009F)
    other than \\n, \\r and \\t as \\x and their low byte"""
    out = []
    for ch in s:
        o = ord(ch)
        if ch == '"':
            out.append('\\"')
        elif ch == "\\":
            out.append("\\\\")
        elif ch == "\n":
            out.append("\\n")
        elif ch == "\r":
            out.append("\\r")
        elif ch == "\t":
            out.append("\\t")
        elif o <= 0x1F or 0x7F <= o <= 0x9F:
            out.append("\\x%02x" % (o & 0xFF))
        else:
            out.append(ch)
    return "".join(out)


class Metrics:
    """MetricsBuilder::new().max_denied_keys(n).build() over `limiter`'s engine (metrics.rs:100-142).  Creating one
    switches on the engine's denied tracking (max_denied_keys, clamped to 10,000; 0 turns the top-keys section off)
    and its ring metrics, and takes the start time.  The counters are the GPU's ring counts plus the events recorded
    here; call the object (or export_prometheus) for the text."""

    def __init__(self, limiter, max_denied_keys=100):
        self.limiter, self.store = limiter, limiter.store
        self.max_denied_keys = min(max(int(max_denied_keys), 0), MAX_DENIED_KEYS_LIMIT)
        self.start = time.monotonic()
        self.host = np.zeros((3, 3), np.uint64)        # [transport][allowed, denied, errors] decided on the host
        self.names = {}                                # key hash -> key bytes, of keys the host saw denied
        self._switch_on()

    def _switch_on(self):
        """denied tracking and ring metrics on the engine"""
        self.store.track_denied(self.max_denied_keys)
        self.store.ring_metrics(True)

    def record_request(self, transport, allowed, key=None):
        """record_request_with_key / record_request (metrics.rs:161-192) for a request decided on the host.  The engine
        decided it, so its denied-key table counted the denial already: only the key's name is kept here."""
        self.host[TRANSPORTS[transport], 0 if allowed else 1] += 1
        if not allowed and key is not None and self.max_denied_keys:
            kb = key.encode() if isinstance(key, str) else bytes(key)
            if len(kb) <= MAX_KEY_LENGTH:
                self.names[self.store.hash_key(kb)] = kb

    def record_error(self, transport):
        """record_error (metrics.rs:194-205)"""
        self.host[TRANSPORTS[transport], 2] += 1

    def counts(self):
        """[transport][allowed, denied, errors]: the rings' rows plus the host's events (Python ints)"""
        gpu = self._ring_counts()
        return [[int(gpu[t, j]) + int(self.host[t, j]) for j in range(3)] for t in range(3)]

    def _ring_counts(self):
        return np.asarray(self.store.ring_transport_counts(), np.uint64)

    def uptime_seconds(self):
        return int(time.monotonic() - self.start)

    def top_denied_keys(self):
        """[(key, count)], most denied first: every entry of the engine's table in gcra_top_denied's order, named by
        the rings or else by the host's records; keys longer than 256 bytes and keys without a name are left out"""
        if not self.max_denied_keys:
            return []
        # (every entry: the table holds at most 2 x max(16 x max_keys, 1024))
        top, _ = self.store.top_denied(self._table_entries())
        hashes = [h for h, _ in top]
        out = self._named(top, self.store.denied_names(hashes) if hashes else [])
        live = set(hashes)
        self.names = {h: n for h, n in self.names.items() if h in live}
        return out

    def _table_entries(self):
        return 2 * max(16 * self.max_denied_keys, 1024)

    def _named(self, top, names):
        """the top list's first max_denied_keys named entries: names[i] is top[i]'s ring name or marker, the host's
        records name the rest"""
        out = []
        for (h, count), name in zip(top, names):
            if name == NAME_TOO_LONG:
                continue
            if not isinstance(name, bytes):
                name = self.names.get(h)
            if name is None:
                continue
            out.append((name.decode("utf-8", "replace"), count))
            if len(out) == self.max_denied_keys:
                break
        return out

    def export_prometheus(self):
        """metrics.rs:233-310, byte for byte"""
        c = self.counts()
        by = [sum(row) for row in c]
        o = ["# HELP throttlecrab_uptime_seconds Time since server start in seconds\n",
             "# TYPE throttlecrab_uptime_seconds gauge\n",
             "throttlecrab_uptime_seconds %d\n\n" % self.uptime_seconds(),
             "# HELP throttlecrab_requests_total Total number of requests processed\n",
             "# TYPE throttlecrab_requests_total counter\n",
             "throttlecrab_requests_total %d\n\n" % sum(by),
             "# HELP throttlecrab_requests_by_transport Total requests by transport type\n",
             "# TYPE throttlecrab_requests_by_transport counter\n",
             'throttlecrab_requests_by_transport{transport="http"} %d\n' % by[1],
             'throttlecrab_requests_by_transport{transport="grpc"} %d\n' % by[2],
             'throttlecrab_requests_by_transport{transport="redis"} %d\n\n' % by[0]]
        for name, help_, j in (("allowed", "Total requests allowed", 0), ("denied", "Total requests denied", 1),
                               ("errors", "Total internal errors", 2)):
            o += ["# HELP throttlecrab_requests_%s %s\n" % (name, help_),
                  "# TYPE throttlecrab_requests_%s counter\n" % name,
                  "throttlecrab_requests_%s %d\n\n" % (name, sum(row[j] for row in c))]
        if self.max_denied_keys:
            o += ["# HELP throttlecrab_top_denied_keys Top keys by denial count\n",
                  "# TYPE throttlecrab_top_denied_keys gauge\n"]
            for rank, (key, count) in enumerate(self.top_denied_keys(), 1):
                o.append('throttlecrab_top_denied_keys{key="%s",rank="%d"} %d\n' % (escape_label(key), rank, count))
        return "".join(o)

    def __call__(self):
        return self.export_prometheus()


class ShardedMetrics(Metrics):
    """Metrics over the engines of one hash-sharded table, `limiters` in rank order (mixed.process_connections_sharded
    serves it as GET /metrics).  Creating one switches on denied tracking (max_denied_keys, clamped as Metrics does)
    and sharded ring metrics (gcra_ring_metrics_sharded) on every rank.  The counts are the sum of the ranks' GPU
    counts plus the events recorded here; record_request hashes with the ranks' shared seed.

    The top denied keys join what the ranks hold apart: every rank's top list (each query prunes that rank's table by
    gcra_top_denied's rule), merged (sharded.merge_top_denied: the lists hold disjoint keys, each counted on its
    owner); each hash named by the first rank whose connections named it, or else by the host's records; a hash that
    any rank marks too long, or that nobody named, is left out.  Then every rank keeps the names of the hashes that
    survived their owner's pruning, and forgets the rest.  `full` is the ranks' denied rows, since the scrape before,
    whose key found its name table full (those keys may go unnamed): rows, not keys, so a hot key left out counts
    once per denial."""

    def __init__(self, limiters, max_denied_keys=100):
        self.limiters = list(limiters)
        self.stores = [lim.store for lim in self.limiters]
        self.full = 0
        super().__init__(self.limiters[0], max_denied_keys)    # (store: rank 0's, whose hash_key is every rank's)

    def _switch_on(self):
        for st in self.stores:
            st.track_denied(self.max_denied_keys)
            st.ring_metrics_sharded(True, self.max_denied_keys)

    def _ring_counts(self):
        return sum((np.asarray(st.ring_transport_counts(), np.uint64) for st in self.stores),
                   np.zeros((3, 3), np.uint64))

    def top_denied_keys(self):
        from .sharded import merge_top_denied          # (sharded imports torch: only ShardedMetrics needs it)
        if not self.max_denied_keys:
            return []
        k = self.max_denied_keys
        lists = [st.top_denied(self._table_entries())[0] for st in self.stores]
        top = merge_top_denied(lists, sum(len(lst) for lst in lists))
        hashes = [h for h, _ in top]
        per_rank = [st.denied_names(hashes) for st in self.stores] if hashes else []
        names = []
        for got in zip(*per_rank):
            if any(g == NAME_TOO_LONG for g in got):
                names.append(NAME_TOO_LONG)
            else:
                names.append(next((g for g in got if isinstance(g, bytes)), NAME_UNKNOWN))
        out = self._named(top, names)
        # (gcra_top_denied's pruning: a list of more than 3 x k entries kept its first k, any other list all of them)
        keep = sorted({h for lst in lists for h, _ in (lst[:k] if len(lst) > 3 * k else lst)})
        self.full = sum(st.ring_names_keep(keep) for st in self.stores)
        live = set(keep)
        self.names = {h: n for h, n in self.names.items() if h in live}
        return out
