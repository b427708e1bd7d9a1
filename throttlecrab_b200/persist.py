"""The server's snapshot directory (--snapshot-dir): restore the table at start, save it in the background while
serving, save it once more at shutdown.  One SnapshotDir works over the server's stores in rank order, one engine or N.

    <dir>/LOCK                   flock'ed by the serving process for its whole life
    <dir>/MANIFEST               JSON: format, generation, world, files, entries, time, store
    <dir>/gen-<G>/rank<r>.gcra   generation G's file of rank r (store.save_begin: snapshot format version 3)

The manifest is the commit point.  A generation's files are all written (every rank's save_wait succeeded) and its
directory is fsynced before the manifest is written to a temporary file, fsynced, renamed over MANIFEST and the
directory fsynced; only then are the other generations deleted.  A save interrupted anywhere therefore leaves the
previous complete generation as the one MANIFEST names, and a restore never mixes two cuts.

Restore inserts every file of the committed generation into every new rank r of world M (store.restore(f, r, M)), so
the engine count may change between runs.  Nothing here imports torch or touches CUDA: the stores do.
"""
import fcntl
import json
import os
import re
import shutil
import time

from . import Internal

FORMAT = 1
MANIFEST = "MANIFEST"
_GEN = re.compile(r"gen-(\d+)$")


class SnapshotError(Exception):
    """a snapshot directory the server refuses to start with: `status` is the exit status"""

    def __init__(self, message, status=1):
        super().__init__(message)
        self.status = status


def _fsync_dir(path):
    fd = os.open(path, os.O_RDONLY | os.O_DIRECTORY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def _rank_file(r):
    return "rank%d.gcra" % r


class SnapshotDir:
    """The snapshot directory at `path`, created if missing and locked (SnapshotError, status 2, when another process
    holds it).  `store` is the configured store type, recorded in the manifest.  `log` takes info / warning.

    restore(stores) loads the committed generation and keeps `stores` (rank order) for the saves; begin() starts a
    background save at a serve boundary, poll() commits it once every rank's file is written, save() is the
    shutdown save.  close() releases the lock."""

    def __init__(self, path, store="", log=None):
        self.path, self.store_type, self.log = os.path.abspath(path), store, log
        self.stores = []
        self.generation = 0            # the committed generation (0: none)
        self._next = 1                 # the next generation a save writes (a failed one's number is not reused)
        self._pending = None           # a save in flight: {"gen": G, "left": set of ranks, "error": text or None}
        self._lock = None
        try:
            os.makedirs(self.path, exist_ok=True)
            fd = os.open(os.path.join(self.path, "LOCK"), os.O_RDWR | os.O_CREAT, 0o644)
        except OSError as e:
            raise SnapshotError("snapshot directory %s: %s" % (self.path, e), 2)
        try:
            fcntl.flock(fd, fcntl.LOCK_EX | fcntl.LOCK_NB)
        except OSError:
            os.close(fd)
            raise SnapshotError("snapshot directory %s is in use by another process (LOCK is held)" % self.path, 2)
        self._lock = fd

    def close(self):
        if self._lock is not None:
            os.close(self._lock)                       # (releases the flock)
            self._lock = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- restore ------------------------------------------------------------------------------------------------------
    def manifest(self):
        """the committed manifest, checked, or None when there is none; SnapshotError when it cannot be used"""
        p = os.path.join(self.path, MANIFEST)
        try:
            with open(p, "rb") as f:
                raw = f.read()
        except FileNotFoundError:
            return None
        except OSError as e:
            raise SnapshotError("snapshot manifest %s: %s" % (p, e))
        try:
            m = json.loads(raw)
        except ValueError as e:
            raise SnapshotError("snapshot manifest %s is malformed: %s" % (p, e))
        if not isinstance(m, dict) or m.get("format") != FORMAT:
            raise SnapshotError("snapshot manifest %s: unknown format %r (this build reads format %d)"
                                % (p, m.get("format") if isinstance(m, dict) else m, FORMAT))
        g, w, files, entries = m.get("generation"), m.get("world"), m.get("files"), m.get("entries")
        ok = (type(g) is int and g >= 1 and type(w) is int and w >= 1 and isinstance(files, list)
              and len(files) == w and all(isinstance(f, str) and f and os.path.basename(f) == f and f not in (".", "..")
                                          for f in files)
              and isinstance(entries, list) and len(entries) == w and all(type(n) is int and n >= 0 for n in entries))
        if not ok:
            raise SnapshotError("snapshot manifest %s is malformed: %r" % (p, m))
        return m

    def restore(self, stores):
        """Insert the committed generation into `stores` (rank order; each empty, as made) and keep them for the
        saves -> the manifest, or None when the directory holds none (the stores start empty).  SnapshotError when
        the manifest or a file cannot be used: the caller must not serve, since starting empty would reset every
        limit.  After a restore (or finding no manifest), generation directories the manifest does not name are
        deleted."""
        self.stores = list(stores)
        m = self.manifest()
        if m is None:
            if self.log:
                self.log.info("Snapshot directory %s holds no snapshot: starting empty", self.path)
            self._prune()                              # (a first save that never committed)
            return None
        gen = os.path.join(self.path, "gen-%d" % m["generation"])
        paths = [os.path.join(gen, f) for f in m["files"]]
        for p in paths:
            if not os.path.isfile(p):
                raise SnapshotError("snapshot generation %d lists %s, which is missing" % (m["generation"], p))
        t0, world, restored, conflicts = time.monotonic(), len(self.stores), 0, 0
        for r, st in enumerate(self.stores):
            for p in paths:
                try:
                    n, c = st.restore(p, r, world)
                except Internal as e:
                    raise SnapshotError("snapshot restore of %s into rank %d of %d failed: %s" % (p, r, world, e))
                restored, conflicts = restored + n, conflicts + c
        self.generation = m["generation"]
        self._next = self.generation + 1
        if self.log:
            self.log.info("Restored snapshot generation %d: %d entries, %d conflicts, saved by %d engine(s) at %s, "
                          "into %d engine(s) in %.3f s", self.generation, restored, conflicts, m["world"],
                          time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime(m.get("time", 0))), world,
                          time.monotonic() - t0)
        self._prune()
        return m

    # -- saves --------------------------------------------------------------------------------------------------------
    def in_flight(self):
        return self._pending is not None

    def begin(self):
        """Begin a background save on every engine (call it between serves: then every engine has ended every tick
        it started and the ranks' files are one cut).  -> True when begun; False when a save is still in flight (this
        call is skipped) or it failed to begin (logged; the committed generation stays)."""
        if self._pending is not None:
            if self.log:
                self.log.info("Snapshot generation %d still in flight: skipping this interval", self._pending["gen"])
            return False
        g = self._next
        self._next += 1
        self._pending = {"gen": g, "left": set(), "error": None}
        try:
            os.mkdir(self._gen_dir(g))
        except OSError as e:
            self._pending["error"] = "cannot create %s: %s" % (self._gen_dir(g), e)
            self._finish()
            return False
        for r, st in enumerate(self.stores):
            try:
                st.save_begin(os.path.join(self._gen_dir(g), _rank_file(r)))
            except Internal as e:
                self._pending["error"] = "rank %d: %s" % (r, e)
                break
            self._pending["left"].add(r)
        if self._pending["error"] is not None:
            self._wait_left()
            self._finish()
            return False
        return True

    def poll(self):
        """Non-blocking: commit the save in flight once every rank's file is written -> the generation committed by
        this call, or None"""
        p = self._pending
        if p is None:
            return None
        for r in sorted(p["left"]):
            try:
                done = self.stores[r].save_poll()
            except Internal as e:
                done = True
                p["error"] = p["error"] or "rank %d: %s" % (r, e)
            if done:
                p["left"].discard(r)
        if p["left"]:
            return None
        return self._finish()

    def save(self):
        """The shutdown save: finish a save in flight, then save every engine and wait for it -> the committed
        generation.  SnapshotError when it fails (the previous generation stays committed)."""
        if self._pending is not None:
            self._wait_left()
            self._finish()
        if not self.begin():
            raise SnapshotError("snapshot save failed; generation %d stays committed" % self.generation)
        self._wait_left()
        g = self._finish()
        if g is None:
            raise SnapshotError("snapshot save failed; generation %d stays committed" % self.generation)
        return g

    def _gen_dir(self, g):
        return os.path.join(self.path, "gen-%d" % g)

    def _wait_left(self):
        p = self._pending
        for r in sorted(p["left"]):
            try:
                self.stores[r].save_wait()
            except Internal as e:
                p["error"] = p["error"] or "rank %d: %s" % (r, e)
        p["left"].clear()

    def _finish(self):
        """every rank of the pending save is done: commit it, or discard it -> the generation committed, or None"""
        p, self._pending = self._pending, None
        g, entries = p["gen"], []
        if p["error"] is None:
            try:
                entries = [int(st.save_wait()) for st in self.stores]     # (done: returns at once)
            except Internal as e:
                p["error"] = str(e)
        if p["error"] is None:
            try:
                self._commit(g, entries)
                return g
            except OSError as e:
                p["error"] = "commit: %s" % e
        if self.log:
            self.log.warning("Snapshot generation %d failed, discarded (generation %d stays committed): %s",
                             g, self.generation, p["error"])
        if os.path.isdir(self._gen_dir(g)):
            shutil.rmtree(self._gen_dir(g), ignore_errors=True)
        return None

    def _commit(self, g, entries):
        _fsync_dir(self._gen_dir(g))                   # the rank files' names, then the generation's own
        _fsync_dir(self.path)
        m = {"format": FORMAT, "generation": g, "world": len(self.stores),
             "files": [_rank_file(r) for r in range(len(self.stores))], "entries": entries, "time": time.time(),
             "store": self.store_type}
        tmp = os.path.join(self.path, MANIFEST + ".tmp")
        with open(tmp, "w") as f:
            json.dump(m, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, os.path.join(self.path, MANIFEST))
        _fsync_dir(self.path)
        self.generation = g
        self._prune()

    def _prune(self):
        """delete every generation directory but the committed one"""
        for name in os.listdir(self.path):
            m = _GEN.match(name)
            if m and int(m.group(1)) != self.generation and os.path.isdir(os.path.join(self.path, name)):
                shutil.rmtree(os.path.join(self.path, name), ignore_errors=True)
