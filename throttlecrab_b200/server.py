"""The rate-limiting server: throttlecrab-server's command line over the engine's mixed ring.

    python -m throttlecrab_b200.server --redis --http --grpc

listens on the Redis (RESP), HTTP and gRPC ports the reference listens on and answers every connection against one
table.  The sockets, the connections' buffers and the serving rounds are native (gcra_server_*, include/gcra_b200.h):
a connection's bytes go from its socket into the mixed ring's pinned input, the GPU parses, decides and answers its
plain requests, and the replies go from the ring's mapped output to the socket.  What the ring does not take (PING,
QUIT, GET /health, GET /metrics, a gRPC connection's preface, SETTINGS and HPACK inserts, a malformed request) comes
back here through one callback, to the general paths the Python drivers use: resp.general, http.general and
grpc_transport.Connection.general.  A serve is exactly mixed.process_connections over the connections' pending bytes.

With several devices (--device 0,1,...) the server runs one engine per entry, the engines sharing one hash-sharded
table over peer memory (sharded.connect_local): connections are placed round-robin by accept order, each engine's
mixed ring parses its own connections and routes their rows to their keys' owners, and a serve is exactly
mixed.process_connections_sharded over the engines' connections (gcra_server_create_sharded).

Configuration mirrors config.rs: the same flags, THROTTLECRAB_* environment variables and defaults, CLI over env over
default; one addition, --device / THROTTLECRAB_DEVICE.  --buffer-size bounds the reference's actor channel; here it is
the ring's row_capacity, the most requests one submit decides.

Persistence (SNAPSHOT_FLAGS, off by default; the reference keeps its state in memory only): with --snapshot-dir the
server restores the directory's committed snapshot into its engines before it binds a port, saves in the background
every --snapshot-interval seconds between serves, and saves once more at shutdown (persist.SnapshotDir).
"""
import argparse
import ctypes as C
import logging
import os
import signal
import sys
import time
from dataclasses import dataclass

import numpy as np

from . import (AdaptiveStore, PeriodicStore, ProbabilisticStore, RateLimiter, MixedRing, Internal, GRPC_CONN_DTYPE,
               PROTO_RESP, PROTO_HTTP, PROTO_GRPC)
from . import grpc_transport as _gt
from . import http as _http
from . import mixed as _mixed
from . import resp as _resp
from .metrics import Metrics, ShardedMetrics, MAX_DENIED_KEYS_LIMIT
from .persist import SnapshotDir, SnapshotError

MAX_CONNS = 16384             # connections per ring submit: more open connections take several submits per round
IN_CAPACITY = 16 << 20        # bytes of requests per ring submit (256 full connection buffers)
MAX_BUFFER_SIZE = 1 << 20     # the largest row_capacity: the engine's default max_batch
READ_PAUSE, OUT_BOUND = 512 << 10, 1 << 20     # GCRA_SERVER_READ_PAUSE, GCRA_SERVER_OUT_BOUND
# Engines of one process wait for each other in kernels, and a wait kernel must not sit in a hardware queue ahead of
# the kernel it waits for: several engines need at least this many (INTEGRATION.md, "Serving from N engines")
MIN_DEVICE_CONNECTIONS = 32

PROTOCOLS = {"redis": PROTO_RESP, "http": PROTO_HTTP, "grpc": PROTO_GRPC}
_NAMES = {"redis": "Redis", "http": "HTTP", "grpc": "gRPC"}

# config.rs Args: (flag, environment variable, default, help)
FLAGS = [
    ("--http", "THROTTLECRAB_HTTP", False, "Enable HTTP transport"),
    ("--http-host", "THROTTLECRAB_HTTP_HOST", "0.0.0.0", "HTTP host"),
    ("--http-port", "THROTTLECRAB_HTTP_PORT", 8080, "HTTP port"),
    ("--grpc", "THROTTLECRAB_GRPC", False, "Enable gRPC transport"),
    ("--grpc-host", "THROTTLECRAB_GRPC_HOST", "0.0.0.0", "gRPC host"),
    ("--grpc-port", "THROTTLECRAB_GRPC_PORT", 8070, "gRPC port"),
    ("--redis", "THROTTLECRAB_REDIS", False, "Enable Redis protocol transport"),
    ("--redis-host", "THROTTLECRAB_REDIS_HOST", "0.0.0.0", "Redis host"),
    ("--redis-port", "THROTTLECRAB_REDIS_PORT", 6379, "Redis port"),
    ("--store", "THROTTLECRAB_STORE", "periodic", "Store type: periodic, probabilistic, adaptive"),
    ("--store-capacity", "THROTTLECRAB_STORE_CAPACITY", 100_000, "Initial store capacity"),
    ("--store-cleanup-interval", "THROTTLECRAB_STORE_CLEANUP_INTERVAL", 300,
     "Cleanup interval for periodic store (seconds)"),
    ("--store-cleanup-probability", "THROTTLECRAB_STORE_CLEANUP_PROBABILITY", 10_000,
     "Cleanup probability for probabilistic store (1 in N)"),
    ("--store-min-interval", "THROTTLECRAB_STORE_MIN_INTERVAL", 5,
     "Minimum cleanup interval for adaptive store (seconds)"),
    ("--store-max-interval", "THROTTLECRAB_STORE_MAX_INTERVAL", 300,
     "Maximum cleanup interval for adaptive store (seconds)"),
    ("--store-max-operations", "THROTTLECRAB_STORE_MAX_OPERATIONS", 1_000_000,
     "Maximum operations before cleanup for adaptive store"),
    ("--buffer-size", "THROTTLECRAB_BUFFER_SIZE", 100_000,
     "Rows one ring submit decides (the reference's channel buffer size)"),
    ("--max-denied-keys", "THROTTLECRAB_MAX_DENIED_KEYS", 100,
     "Maximum number of denied keys to track in metrics (0 to disable, max: 10000)"),
    ("--log-level", "THROTTLECRAB_LOG_LEVEL", "info", "Log level: error, warn, info, debug, trace"),
    ("--device", "THROTTLECRAB_DEVICE", 0,
     "CUDA device of the engine, or a comma-separated list: one engine per entry (repeats allowed)"),
]
# additions of this server, not of config.rs: persistence, off unless --snapshot-dir is given
SNAPSHOT_FLAGS = [
    ("--snapshot-dir", "THROTTLECRAB_SNAPSHOT_DIR", None,
     "Directory to restore the limits from at start and save them to (unset: state is not persisted)"),
    ("--snapshot-interval", "THROTTLECRAB_SNAPSHOT_INTERVAL", 60,
     "Seconds between background saves to the snapshot directory (0: save only at shutdown)"),
]
STORE_TYPES = ("periodic", "probabilistic", "adaptive")
NO_TRANSPORT = ("At least one transport must be specified.\n\n"
                "Available transports:\n"
                "  --http       Enable HTTP transport\n"
                "  --grpc       Enable gRPC transport\n"
                "  --redis      Enable Redis protocol transport\n"
                "Example:\n"
                "  python -m throttlecrab_b200.server --http --http-port 7070\n"
                "  python -m throttlecrab_b200.server --http --grpc --redis\n\n"
                "For more information, try '--help'")
_FALSEY = {"", "0", "n", "no", "f", "false", "off"}     # clap's reading of a boolean flag's environment variable


class ConfigError(Exception):
    """a configuration the server refuses: `status` is the exit status"""

    def __init__(self, message, status):
        super().__init__(message)
        self.status = status


@dataclass
class Config:
    http: bool
    http_host: str
    http_port: int
    grpc: bool
    grpc_host: str
    grpc_port: int
    redis: bool
    redis_host: str
    redis_port: int
    store: str
    store_capacity: int
    store_cleanup_interval: int
    store_cleanup_probability: int
    store_min_interval: int
    store_max_interval: int
    store_max_operations: int
    buffer_size: int
    max_denied_keys: int
    log_level: str
    device: object                    # an int, or a tuple of them for several engines (--device 0,1)
    snapshot_dir: object = None       # a path, or None: no persistence
    snapshot_interval: int = 60

    def devices(self):
        """the engines' devices, one per engine"""
        return self.device if isinstance(self.device, tuple) else (self.device,)

    def listens(self):
        """[(transport, host, port)] of the enabled transports"""
        return [(t, getattr(self, t + "_host"), getattr(self, t + "_port")) for t in ("http", "grpc", "redis")
                if getattr(self, t)]


def _dest(flag):
    return flag[2:].replace("-", "_")


def _devices(text, origin):
    """--device with a comma-separated list: a tuple of device indices"""
    out = []
    for part in text.split(","):
        if not part.strip():
            raise ConfigError("invalid value '%s' for '--device': an empty entry (%s)" % (text, origin), 2)
        try:
            v = int(part)
        except ValueError:
            raise ConfigError("invalid value '%s' for '--device': '%s' is not a number (%s)" % (text, part, origin), 2)
        if v < 0:
            raise ConfigError("invalid value '%s' for '--device': %d is out of range (%s)" % (text, v, origin), 2)
        out.append(v)
    return tuple(out)


def _value(flag, default, text, origin):
    if flag == "--device" and "," in text:
        return _devices(text, origin)
    if isinstance(default, bool):
        return text.strip().lower() not in _FALSEY
    if isinstance(default, int):
        try:
            v = int(text)
        except ValueError:
            raise ConfigError("invalid value '%s' for '%s': not a number (%s)" % (text, flag, origin), 2)
        if v < 0 or (flag.endswith("-port") and v > 65535):
            raise ConfigError("invalid value '%s' for '%s': out of range (%s)" % (text, flag, origin), 2)
        return v
    if flag == "--snapshot-dir" and not text:
        raise ConfigError("invalid value '' for '--snapshot-dir': an empty path (%s)" % origin, 2)
    if flag == "--store" and text.lower() not in STORE_TYPES:
        raise ConfigError("invalid value '%s' for '--store': Invalid store type: %s. Valid options are: periodic, "
                          "probabilistic, adaptive" % (text, text), 2)
    return text.lower() if flag == "--store" else text


def env_vars_text():
    """--list-env-vars: every THROTTLECRAB_* variable, what it sets and its default"""
    lines = ["ThrottleCrab environment variables (CLI arguments take precedence over them):", ""]
    for flag, env, default, help_ in FLAGS + SNAPSHOT_FLAGS:
        value = "true|false" if isinstance(default, bool) else "<%s>" % flag.rsplit("-", 1)[-1]
        lines.append("  %-48s %s [default: %s]" % (env + "=" + value, help_, str(default).lower()))
    return "\n".join(lines) + "\n"


def parse_config(argv=None, environ=None):
    """config.rs Config::from_env_and_args: CLI over environment over default.  Returns a Config, or None after
    --list-env-vars printed the variables; ConfigError for a configuration the reference refuses."""
    environ = os.environ if environ is None else environ
    ap = argparse.ArgumentParser(prog="python -m throttlecrab_b200.server",
                                 description="Rate limiting server on the GPU.  At least one transport must be "
                                             "specified.  CLI arguments take precedence over THROTTLECRAB_* "
                                             "environment variables.")
    for flag, env, default, help_ in FLAGS + SNAPSHOT_FLAGS:
        if isinstance(default, bool):
            ap.add_argument(flag, action="store_const", const=True, default=None, help=help_ + " [env: %s]" % env)
        else:
            ap.add_argument(flag, default=None, help=help_ + " [env: %s] [default: %s]" % (env, default))
    ap.add_argument("--list-env-vars", action="store_true", help="List all environment variables and exit")
    a = ap.parse_args(argv)
    if a.list_env_vars:
        sys.stdout.write(env_vars_text())
        return None
    kw = {}
    for flag, env, default, _ in FLAGS + SNAPSHOT_FLAGS:
        cli = getattr(a, _dest(flag))
        if cli is not None:
            kw[_dest(flag)] = cli if isinstance(default, bool) else _value(flag, default, cli, "argument")
        elif env in environ:
            kw[_dest(flag)] = _value(flag, default, environ[env], "environment variable " + env)
        else:
            kw[_dest(flag)] = default
    cfg = Config(**kw)
    if not 0 <= cfg.max_denied_keys <= MAX_DENIED_KEYS_LIMIT:
        raise ConfigError("invalid value '%d' for '--max-denied-keys': %d is not in 0..=%d"
                          % (cfg.max_denied_keys, cfg.max_denied_keys, MAX_DENIED_KEYS_LIMIT), 2)
    if not 1 <= cfg.buffer_size <= MAX_BUFFER_SIZE:
        raise ConfigError("invalid value '%d' for '--buffer-size': the ring's row capacity is 1..=%d"
                          % (cfg.buffer_size, MAX_BUFFER_SIZE), 2)
    if not (cfg.http or cfg.grpc or cfg.redis):
        raise ConfigError(NO_TRANSPORT, 1)
    conns = environ.get("CUDA_DEVICE_MAX_CONNECTIONS")
    if len(cfg.devices()) > 1 and conns is not None and not (conns.strip().isdigit() and
                                                              int(conns) >= MIN_DEVICE_CONNECTIONS):
        raise ConfigError("CUDA_DEVICE_MAX_CONNECTIONS=%s: several engines need at least %d (their kernels wait for "
                          "each other, and a waiting kernel must not hold the hardware queue of the one it waits for)"
                          % (conns, MIN_DEVICE_CONNECTIONS), 2)
    return cfg


def make_store(cfg, device=None, capacity=None):
    """store.rs create_rate_limiter: the configured store type, built by its builder (on `device` with `capacity`,
    default cfg's)"""
    if cfg.store == "periodic":
        b = PeriodicStore.builder().cleanup_interval(cfg.store_cleanup_interval)
    elif cfg.store == "probabilistic":
        b = ProbabilisticStore.builder().cleanup_probability(cfg.store_cleanup_probability)
    else:
        b = AdaptiveStore.builder().min_interval(cfg.store_min_interval).max_interval(cfg.store_max_interval) \
            .max_operations(cfg.store_max_operations)
    return b.capacity(cfg.store_capacity if capacity is None else capacity) \
        .device(cfg.device if device is None else device).build()


class GeneralPathError(RuntimeError):
    """a general-path call failed: its connection was closed, every other connection was served"""


class _General(C.Structure):
    _fields_ = [("consumed", C.c_uint64), ("out", C.c_void_p), ("out_len", C.c_uint64), ("close", C.c_uint32),
                ("plain_ready", C.c_uint32)]


class _Listen(C.Structure):
    _fields_ = [("protocol", C.c_uint32), ("port", C.c_uint16), ("reserved", C.c_uint16), ("host", C.c_char_p)]


_GENERAL_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int64,
                          C.c_void_p, C.POINTER(_General))
_COUNTERS = ("open", "accepted", "closed", "bytes_read", "bytes_written", "rounds", "submits", "general_calls",
             "general_errors", "full_closed", "peak_unsent")


class Server:
    """Listeners and connections served through `ring`, a MixedRing (its slot 0 is the server's), with the general
    paths deciding on the ring's limiter and `metrics` (a metrics.Metrics of the same engine, or None) serving GET
    /metrics.  `listens` is a list of (transport, host, port), transport "redis", "http" or "grpc"; port 0 binds an
    ephemeral port (port(transport) tells it).  read / serve / poll run in the caller's thread; see gcra_server_* in
    include/gcra_b200.h for what each does.

    `ring` may also be a list of MixedRings in rank order, of engines connected over peer memory
    (sharded.connect_local) whose rings are switched to peer-memory ticks (peer_memory(True)): the server then places
    connection id on rank id % len(rings), a serve is mixed.process_connections_sharded over the ranks' connections,
    the general paths decide on mixed.OwnerRouter of the rings' limiters, and `metrics` must be None or a
    metrics.ShardedMetrics of those limiters in rank order (ValueError otherwise)."""

    def __init__(self, ring, listens, metrics=None):
        rings = list(ring) if isinstance(ring, (list, tuple)) else None
        if rings is not None:
            if not rings:
                raise ValueError("no ring")
            limiters = [r.lim for r in rings]
            _mixed.check_sharded_metrics(metrics, limiters)
            self.rings, self.ring, self.limiter = rings, rings[0], _mixed.OwnerRouter(limiters)
        else:
            self.rings, self.ring, self.limiter = [ring], ring, ring.lim
        self.metrics = metrics
        self.store = self.ring.store
        self._L, self._h = self.ring._L, self.ring._h
        self._grpc = {}                                     # connection id -> grpc_transport.Connection
        self._keep, self._error = None, None
        self._cb = _GENERAL_FN(self._general)
        arr = (_Listen * max(len(listens), 1))()
        for i, (t, host, port) in enumerate(listens):
            if t not in PROTOCOLS:
                raise ValueError("transport must be 'redis', 'http' or 'grpc', not %r" % (t,))
            arr[i].protocol, arr[i].port, arr[i].host = PROTOCOLS[t], int(port), host.encode()
        srv = C.c_void_p()
        self._srv = None
        if rings is None:
            self.store._check(self._L.gcra_server_create(self._h, arr, len(listens), self._cb, None, C.byref(srv)))
        else:
            hs = (C.c_void_p * len(rings))(*[r._h.value for r in rings])
            self.store._check(self._L.gcra_server_create_sharded(hs, len(rings), arr, len(listens), self._cb, None,
                                                                 C.byref(srv)))
        self._srv = srv

    def port(self, transport):
        return int(self._L.gcra_server_port(self._srv, PROTOCOLS[transport]))

    def read(self, timeout_ms=0):
        self.store._check(self._L.gcra_server_read(self._srv, int(timeout_ms)))

    def serve(self, now_ns):
        self._check(self._L.gcra_server_serve(self._srv, int(now_ns)))

    def poll(self, timeout_ms, now_ns):
        self._check(self._L.gcra_server_poll(self._srv, int(timeout_ms), int(now_ns)))

    def stats(self):
        out = (C.c_uint64 * len(_COUNTERS))()
        self.store._check(self._L.gcra_server_stats(self._srv, out))
        return dict(zip(_COUNTERS, (int(v) for v in out)))

    def close(self):
        if getattr(self, "_srv", None):
            self._L.gcra_server_destroy(self._srv)
            self._srv = None
        self._grpc.clear()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        err, self._error = self._error, None
        if rc != 0:
            text = self._L.gcra_last_error(self._h).decode()
            if err is not None:
                raise GeneralPathError("%s: %r" % (text, err)) from err
            raise Internal(text)

    def _general(self, ctx, cid, proto, data, n, now, grpc, out):
        """gcra_server_general_fn: one general-path call on connection `cid`'s pending bytes"""
        try:
            if not out:                                     # the connection closed
                self._grpc.pop(cid, None)
                return 0
            buf = C.string_at(data, n) if n else b""
            close, ready = False, False
            if proto == PROTO_GRPC:
                cn = self._grpc.get(cid)
                if cn is None:
                    cn = self._grpc[cid] = _gt.Connection()
                row = np.frombuffer((C.c_char * GRPC_CONN_DTYPE.itemsize).from_address(grpc), GRPC_CONN_DTYPE)[0]
                cn.take_state(row)
                cn.buf, cn.out = bytearray(buf), bytearray()
                cn.general(self.limiter, now, self.metrics)
                cn.state(row)
                consumed, reply, close, ready = n - len(cn.buf), bytes(cn.out), cn.closed, cn.plain_ready
            else:
                g = (_resp.general if proto == PROTO_RESP else _http.general)(buf, self.limiter, now, self.metrics)
                consumed, reply = (0, b"") if g is None else (g[0], g[1])
                close = g is not None and g[3] is not None
            self._keep = C.create_string_buffer(reply, len(reply)) if reply else None
            o = out[0]
            o.consumed, o.out_len, o.close, o.plain_ready = consumed, len(reply), int(close), int(ready)
            o.out = C.cast(self._keep, C.c_void_p) if reply else None
            return 0
        except Exception as e:                              # (reported by serve; the connection closes)
            if self._error is None:
                self._error = e
            return 1


def serve_config(cfg, log, snapshots=None):
    """build the stores, the rings, the metrics and the server of `cfg` -> (server, [store per engine]).  With
    `snapshots` (a persist.SnapshotDir) its committed generation is restored into the stores as soon as they are made,
    before anything else is built and before any port is bound; a failed restore closes the stores and raises
    persist.SnapshotError."""
    devices = cfg.devices()
    if len(devices) == 1:
        store = make_store(cfg)
        try:
            if snapshots is not None:
                snapshots.restore([store])
            lim = RateLimiter(store)
            ring = MixedRing(lim, 1, MAX_CONNS, IN_CAPACITY, cfg.buffer_size)
            metrics = Metrics(lim, cfg.max_denied_keys)
            srv = Server(ring, cfg.listens(), metrics)
        except Exception:
            store.close()
            raise
        stores = [store]
    else:
        srv, stores = _serve_sharded(cfg, devices, snapshots)
    for t, host, _ in cfg.listens():
        log.info("Starting %s transport on %s:%d", _NAMES[t], host, srv.port(t))
    log.info("ThrottleCrab server started with store type: %s", cfg.store.capitalize())
    log.info("Store capacity: %d, Buffer size: %d", cfg.store_capacity, cfg.buffer_size)
    if len(devices) > 1:
        log.info("Engines: %d, one table sharded over peer memory (%s)", len(devices),
                 ", ".join("rank %d on cuda:%d" % (r, d) for r, d in enumerate(devices)))
    return srv, stores


def _serve_sharded(cfg, devices, snapshots=None):
    """one engine per device, each with a 1/world share of the capacity (each restoring its shard of `snapshots`
    before the engines connect), connected over peer memory, each with its mixed ring switched to peer-memory ticks;
    ShardedMetrics; the server -> (server, stores).  A failed step closes what was made, in reverse order."""
    from .sharded import connect_local                 # (sharded imports torch: only several engines need it)
    world = len(devices)
    made = []                                          # what has a close(), in the order made
    try:
        for d in devices:
            made.append(make_store(cfg, d, -(-cfg.store_capacity // world)))
        if snapshots is not None:
            snapshots.restore(made)
        limiters = [RateLimiter(st) for st in made]
        connect_local(limiters, cfg.buffer_size)
        rings = [MixedRing(lim, 1, MAX_CONNS, IN_CAPACITY, cfg.buffer_size) for lim in limiters]
        for ring in rings:
            ring.peer_memory(True)
        metrics = ShardedMetrics(limiters, cfg.max_denied_keys)
        srv = Server(rings, cfg.listens(), metrics)
    except Exception:
        for x in reversed(made):
            x.close()
        raise
    return srv, made


def main(argv=None):
    try:
        cfg = parse_config(argv)
    except ConfigError as e:
        sys.stderr.write("Error: %s\n" % e)
        return e.status
    if cfg is None:
        return 0
    snapshots = None
    if cfg.snapshot_dir is not None:
        try:                                           # (before any CUDA work: a locked directory refuses the start)
            snapshots = SnapshotDir(cfg.snapshot_dir, cfg.store)
        except SnapshotError as e:
            sys.stderr.write("Error: %s\n" % e)
            return e.status
    if len(cfg.devices()) > 1:
        # read when the process first touches CUDA, which nothing imported so far has done (parse_config refused a
        # value below MIN_DEVICE_CONNECTIONS)
        os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", str(MIN_DEVICE_CONNECTIONS))
    level = {"trace": logging.DEBUG, "warn": logging.WARNING}.get(cfg.log_level.lower(),
                                                                     getattr(logging, cfg.log_level.upper(), None))
    logging.basicConfig(stream=sys.stdout, level=level if isinstance(level, int) else logging.INFO,
                        format="%(asctime)s %(levelname)s throttlecrab: %(message)s")
    log = logging.getLogger("throttlecrab")
    stop = []
    for sig in (signal.SIGINT, signal.SIGTERM):
        signal.signal(sig, lambda s, _f: stop.append(s))
    status = 0
    try:
        if snapshots is not None:
            snapshots.log = log
        try:
            srv, stores = serve_config(cfg, log, snapshots)
        except SnapshotError as e:                     # (the stores are closed and no port was bound)
            sys.stderr.write("Error: %s\n" % e)
            return e.status
        try:
            interval = cfg.snapshot_interval
            due = time.monotonic() + interval
            # A signal is seen here, between polls, never inside one: a poll ends every tick it started on every
            # engine, so no engine is left owing its peers a tick at exit, and a save begun here is one cut of the
            # whole table.
            while not stop:
                try:
                    srv.poll(100, time.time_ns())
                except GeneralPathError as e:
                    log.warning("%s", e)
                if snapshots is not None:
                    snapshots.poll()
                    if interval and time.monotonic() >= due:
                        snapshots.begin()
                        due = time.monotonic() + interval
            log.info("Received %s, initiating graceful shutdown...", signal.Signals(stop[0]).name)
            srv.close()
            if snapshots is not None:
                t0 = time.monotonic()
                try:
                    g = snapshots.save()
                    log.info("Saved snapshot generation %d to %s in %.3f s", g, snapshots.path, time.monotonic() - t0)
                except SnapshotError as e:
                    log.error("%s", e)
                    status = 1
        finally:
            srv.close()                                # (the server before the engines whose rings it drives)
            for store in reversed(stores):
                store.close()
    finally:
        if snapshots is not None:
            snapshots.close()
    log.info("ThrottleCrab server shutdown complete")
    return status


if __name__ == "__main__":
    sys.exit(main())
