"""--snapshot-dir / --snapshot-interval and the snapshot directory (persist.SnapshotDir) over fake stores: the flags,
the commit order (rank files, then the manifest's rename, then the pruning), saves that fail at begin, poll or wait,
leftover generations, refused manifests, restore across world sizes, the directory lock, and where serve_config
restores.  No device work."""
import fcntl
import json
import os
import subprocess
import sys

import pytest

from throttlecrab_b200 import Internal
from throttlecrab_b200 import persist as P
from throttlecrab_b200 import server as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- flags -----------------------------------------------------------------------------------------------------------
def test_flags_from_the_cli_the_environment_and_by_default():
    cfg = S.parse_config(["--http"], {})
    assert cfg.snapshot_dir is None and cfg.snapshot_interval == 60
    cfg = S.parse_config(["--http"], {"THROTTLECRAB_SNAPSHOT_DIR": "/e", "THROTTLECRAB_SNAPSHOT_INTERVAL": "5"})
    assert (cfg.snapshot_dir, cfg.snapshot_interval) == ("/e", 5)
    cfg = S.parse_config(["--http", "--snapshot-dir", "/c", "--snapshot-interval", "0"],
                         {"THROTTLECRAB_SNAPSHOT_DIR": "/e", "THROTTLECRAB_SNAPSHOT_INTERVAL": "5"})
    assert (cfg.snapshot_dir, cfg.snapshot_interval) == ("/c", 0)
    # an interval without a directory is accepted (and has no effect)
    assert S.parse_config(["--http", "--snapshot-interval", "7"], {}).snapshot_dir is None


def test_config_without_the_new_fields_still_builds():
    kw = {S._dest(f): d for f, _, d, _ in S.FLAGS}
    cfg = S.Config(**kw)
    assert cfg.snapshot_dir is None and cfg.snapshot_interval == 60


def test_list_env_vars_names_both():
    text = S.env_vars_text()
    assert "THROTTLECRAB_SNAPSHOT_DIR=<dir>" in text and "THROTTLECRAB_SNAPSHOT_INTERVAL=<interval>" in text
    assert "[default: 60]" in text.split("THROTTLECRAB_SNAPSHOT_INTERVAL", 1)[1].splitlines()[0]
    assert all(f not in [x[0] for x in S.FLAGS] for f in ("--snapshot-dir", "--snapshot-interval"))


@pytest.mark.parametrize("flag,value", [("--snapshot-interval", "-1"), ("--snapshot-interval", "x"),
                                        ("--snapshot-interval", "1.5"), ("--snapshot-dir", "")])
def test_malformed_values_are_refused_with_status_2(flag, value):
    env = {"THROTTLECRAB_" + flag[2:].upper().replace("-", "_"): value}
    for argv, environ in [([flag, value], {}), ([], env)]:
        with pytest.raises(S.ConfigError) as e:
            S.parse_config(["--http"] + argv, environ)
        assert e.value.status == 2 and flag in str(e.value)
    p = subprocess.run([sys.executable, "-m", "throttlecrab_b200.server", "--http", flag, value], cwd=ROOT,
                       capture_output=True, text=True, timeout=60)
    assert p.returncode == 2 and flag in p.stderr, p.stderr


# ---- the directory over fake stores ----------------------------------------------------------------------------------
class FakeStore:
    """save_begin writes the file at once (or fails); save_poll / save_wait report `fail_at`; restore records"""

    def __init__(self, rank, events, fail_at=None):
        self.rank, self.events, self.fail_at = rank, events, fail_at
        self.restored, self.inflight = [], False

    def save_begin(self, path):
        if self.fail_at == "begin":
            raise Internal("snapshot: cannot create a file next to " + path)
        with open(path, "wb") as f:
            f.write(b"rank%d" % self.rank)
        self.events.append(("file", os.path.relpath(path, os.path.dirname(os.path.dirname(path)))))
        self.inflight = True

    def save_poll(self):
        if self.fail_at == "poll" and self.inflight:
            raise Internal("snapshot: short write")
        return True

    def save_wait(self):
        self.inflight = False
        if self.fail_at in ("poll", "wait"):
            raise Internal("snapshot: fsync")
        return 10 + self.rank

    def restore(self, path, rank, world):
        self.restored.append((os.path.basename(os.path.dirname(path)) + "/" + os.path.basename(path), rank, world))
        return 1, 0


class Log:
    def __init__(self):
        self.lines = []

    def info(self, fmt, *a):
        self.lines.append(("info", fmt % a))

    def warning(self, fmt, *a):
        self.lines.append(("warning", fmt % a))


def _manifest(d):
    with open(os.path.join(d, "MANIFEST")) as f:
        return json.load(f)


def _gens(d):
    return sorted(n for n in os.listdir(d) if n.startswith("gen-"))


def _dir(tmp_path, world, events=None, fail=None, log=None):
    events = [] if events is None else events
    sd = P.SnapshotDir(str(tmp_path), "periodic", log)
    stores = [FakeStore(r, events, (fail or {}).get(r)) for r in range(world)]
    assert sd.restore(stores) is None
    return sd, stores, events


def test_commit_order_files_then_manifest_rename_then_pruning(tmp_path, monkeypatch):
    events = []
    sd, stores, _ = _dir(tmp_path, 3, events)
    assert sd.save() == 1
    real_replace, real_rmtree = os.replace, P.shutil.rmtree

    def replace(src, dst):
        if os.path.basename(dst) == "MANIFEST":
            with open(src) as f:
                events.append(("manifest", json.load(f)["generation"]))
        return real_replace(src, dst)

    def rmtree(path, *a, **kw):
        events.append(("prune", os.path.basename(path), _manifest(str(tmp_path))["generation"]))
        return real_rmtree(path, *a, **kw)
    monkeypatch.setattr(os, "replace", replace)
    monkeypatch.setattr(P.shutil, "rmtree", rmtree)
    events.clear()
    assert sd.begin() and sd.poll() == 2
    assert events == [("file", "gen-2/rank0.gcra"), ("file", "gen-2/rank1.gcra"), ("file", "gen-2/rank2.gcra"),
                      ("manifest", 2), ("prune", "gen-1", 2)]
    m = _manifest(str(tmp_path))
    assert m["format"] == P.FORMAT and m["world"] == 3 and m["store"] == "periodic"
    assert m["files"] == ["rank0.gcra", "rank1.gcra", "rank2.gcra"] and m["entries"] == [10, 11, 12]
    assert _gens(str(tmp_path)) == ["gen-2"] and not os.path.exists(os.path.join(str(tmp_path), "MANIFEST.tmp"))
    sd.close()


@pytest.mark.parametrize("stage", ["begin", "poll", "wait"])
@pytest.mark.parametrize("rank", [0, 1])
def test_a_failed_rank_discards_its_generation_and_keeps_the_previous_manifest(tmp_path, stage, rank):
    log = Log()
    sd, stores, _ = _dir(tmp_path, 2, log=log)
    assert sd.save() == 1
    before = _manifest(str(tmp_path))
    stores[rank].fail_at = stage
    if stage == "begin":
        assert not sd.begin()
    else:
        assert sd.begin()
        assert sd.poll() is None
    assert not sd.in_flight()
    assert _manifest(str(tmp_path)) == before and _gens(str(tmp_path)) == ["gen-1"]
    assert any(k == "warning" and "generation 2 failed" in t and "generation 1 stays" in t for k, t in log.lines)
    with pytest.raises(P.SnapshotError, match="generation 1 stays committed"):
        sd.save()                                      # (the shutdown save fails the same way)
    assert _manifest(str(tmp_path)) == before
    stores[rank].fail_at = None                        # the next interval tries again, under a new number
    assert sd.begin() and sd.poll() == 4 and _gens(str(tmp_path)) == ["gen-4"]
    sd.close()


def test_a_save_in_flight_makes_the_next_interval_skip(tmp_path):
    log = Log()
    sd, stores, _ = _dir(tmp_path, 2, log=log)
    stores[1].save_poll = lambda: False
    assert sd.begin() and sd.poll() is None and sd.in_flight()
    assert not sd.begin()                              # skipped, not queued
    assert any("still in flight" in t for _, t in log.lines)
    assert _gens(str(tmp_path)) == ["gen-1"] and not os.path.exists(os.path.join(str(tmp_path), "MANIFEST"))
    assert sd.save() == 2                              # the shutdown save commits the one in flight, then its own
    assert _manifest(str(tmp_path))["generation"] == 2 and _gens(str(tmp_path)) == ["gen-2"]
    sd.close()


def test_restore_from_world_w_into_world_m_calls_every_file_rank_and_world(tmp_path):
    for old, new in [(1, 1), (1, 2), (2, 1), (2, 3), (3, 2)]:
        d = tmp_path / ("%d-%d" % (old, new))
        sd, _, _ = _dir(d, old)
        g = sd.save()
        sd.close()
        log = Log()
        sd = P.SnapshotDir(str(d), "adaptive", log)
        stores = [FakeStore(r, []) for r in range(new)]
        assert sd.restore(stores)["world"] == old
        for r, st in enumerate(stores):
            assert st.restored == [("gen-%d/rank%d.gcra" % (g, f), r, new) for f in range(old)]
        assert sd.generation == g and any("Restored snapshot generation %d" % g in t for _, t in log.lines)
        assert sd.save() == g + 1 and _manifest(str(d))["world"] == new
        sd.close()


def test_a_generation_the_manifest_does_not_name_is_ignored_then_removed(tmp_path):
    sd, _, _ = _dir(tmp_path, 2)
    sd.save()
    sd.close()
    for g in (0, 2, 7):                                # an interrupted save's leftovers, older or newer
        os.mkdir(str(tmp_path / ("gen-%d" % g)))
        (tmp_path / ("gen-%d" % g) / "rank0.gcra").write_bytes(b"partial")
    sd = P.SnapshotDir(str(tmp_path), "periodic")
    stores = [FakeStore(r, []) for r in range(2)]
    sd.restore(stores)
    assert all(p.startswith("gen-1/") for st in stores for p, _, _ in st.restored)
    assert _gens(str(tmp_path)) == ["gen-1"]
    sd.close()


def test_no_manifest_starts_empty_and_removes_uncommitted_generations(tmp_path):
    os.mkdir(str(tmp_path / "gen-1"))
    sd = P.SnapshotDir(str(tmp_path / "new"), "periodic")          # a missing directory is created
    assert sd.restore([FakeStore(0, [])]) is None and os.path.isdir(str(tmp_path / "new"))
    sd.close()
    sd = P.SnapshotDir(str(tmp_path), "periodic")
    st = FakeStore(0, [])
    assert sd.restore([st]) is None and st.restored == [] and _gens(str(tmp_path)) == []
    assert sd.save() == 1
    sd.close()


@pytest.mark.parametrize("text,match", [
    ("{", "malformed"), ("[]", "unknown format"), ('{"format": 99}', "unknown format"),
    ('{"format": 1, "generation": 1, "world": 2, "files": ["rank0.gcra"], "entries": [1]}', "malformed"),
    ('{"format": 1, "generation": 1, "world": 1, "files": ["../x"], "entries": [1]}', "malformed"),
    ('{"format": 1, "generation": 0, "world": 1, "files": ["rank0.gcra"], "entries": [1]}', "malformed"),
    ('{"format": 1, "generation": 1, "world": 1, "files": ["rank0.gcra"], "entries": [-1]}', "malformed"),
])
def test_a_malformed_manifest_is_refused(tmp_path, text, match):
    (tmp_path / "MANIFEST").write_text(text)
    sd = P.SnapshotDir(str(tmp_path), "periodic")
    st = FakeStore(0, [])
    with pytest.raises(P.SnapshotError, match=match):
        sd.restore([st])
    assert st.restored == []
    sd.close()


def test_a_missing_file_is_refused_before_any_restore(tmp_path):
    sd, _, _ = _dir(tmp_path, 2)
    sd.save()
    sd.close()
    os.remove(str(tmp_path / "gen-1" / "rank1.gcra"))
    sd = P.SnapshotDir(str(tmp_path), "periodic")
    st = FakeStore(0, [])
    with pytest.raises(P.SnapshotError, match="rank1.gcra, which is missing"):
        sd.restore([st])
    assert st.restored == [] and _gens(str(tmp_path)) == ["gen-1"]
    sd.close()


def test_a_failed_restore_is_refused(tmp_path):
    sd, _, _ = _dir(tmp_path, 1)
    sd.save()
    sd.close()
    sd = P.SnapshotDir(str(tmp_path), "periodic")
    st = FakeStore(0, [])

    def bad(path, rank, world):
        raise Internal("snapshot: bad header")
    st.restore = bad
    with pytest.raises(P.SnapshotError, match="bad header"):
        sd.restore([st])
    assert sd.generation == 0
    sd.close()


# ---- the lock --------------------------------------------------------------------------------------------------------
def test_a_second_object_on_the_same_directory_is_refused(tmp_path):
    sd = P.SnapshotDir(str(tmp_path), "periodic")
    with pytest.raises(P.SnapshotError, match="in use by another process") as e:
        P.SnapshotDir(str(tmp_path), "periodic")
    assert e.value.status == 2
    sd.close()
    P.SnapshotDir(str(tmp_path), "periodic").close()   # released by close


def test_the_cli_exits_2_while_the_directory_is_locked(tmp_path):
    fd = os.open(str(tmp_path / "LOCK"), os.O_RDWR | os.O_CREAT)
    fcntl.flock(fd, fcntl.LOCK_EX)
    try:
        # (a CUDA-less machine would fail to make an engine instead: the refusal comes before any CUDA work)
        p = subprocess.run([sys.executable, "-m", "throttlecrab_b200.server", "--redis", "--snapshot-dir",
                            str(tmp_path)], cwd=ROOT, capture_output=True, text=True, timeout=60)
        assert p.returncode == 2 and "in use by another process" in p.stderr, (p.stdout, p.stderr)
        assert "gcra_create" not in p.stderr + p.stdout
    finally:
        os.close(fd)


# ---- serve_config ----------------------------------------------------------------------------------------------------
def _fakes(monkeypatch, calls, fail_restore=False):
    built = []

    class Fake:
        def __init__(self, **kw):
            self.kw = kw
            built.append(self)
            calls.append(("store", len(built) - 1))

        def close(self):
            calls.append(("close", built.index(self)))

        def restore(self, path, rank, world):
            calls.append(("restore", built.index(self), os.path.basename(path), rank, world))
            if fail_restore and rank == world - 1:
                raise Internal("snapshot: the file is truncated")
            return 0, 0
    for cls in (S.PeriodicStore, S.ProbabilisticStore, S.AdaptiveStore):
        monkeypatch.setattr(cls, "__init__", lambda self, **kw: Fake.__init__(self, **kw))
        monkeypatch.setattr(cls, "close", lambda self: Fake.close(self))
        monkeypatch.setattr(cls, "restore", lambda self, *a: Fake.restore(self, *a))
    monkeypatch.setattr(S, "RateLimiter", lambda st: calls.append(("limiter", built.index(st))) or ("lim", st))
    import throttlecrab_b200.sharded as sharded
    monkeypatch.setattr(sharded, "connect_local", lambda lims, cap: calls.append(("connect", len(lims))))

    class Ring:
        def __init__(self, lim, *geometry):
            calls.append(("ring", built.index(lim[1])))

        def peer_memory(self, on):
            pass
    monkeypatch.setattr(S, "MixedRing", Ring)
    monkeypatch.setattr(S, "ShardedMetrics", lambda lims, k: None)
    monkeypatch.setattr(S, "Metrics", lambda lim, k: None)

    class Srv:
        def __init__(self, rings, listens, metrics):
            calls.append(("server",))

        def port(self, t):
            return 1
    monkeypatch.setattr(S, "Server", Srv)
    return built


def _committed(path, world):
    sd = P.SnapshotDir(str(path), "periodic")
    sd.restore([FakeStore(r, []) for r in range(world)])
    sd.save()
    sd.close()


@pytest.mark.parametrize("devices", ["0", "0,0,1"])
def test_serve_config_restores_after_the_stores_and_before_everything_else(tmp_path, monkeypatch, devices):
    _committed(tmp_path, 2)
    calls = []
    _fakes(monkeypatch, calls)
    cfg = S.parse_config(["--http", "--device", devices, "--snapshot-dir", str(tmp_path)], {})
    sd = P.SnapshotDir(cfg.snapshot_dir, cfg.store)
    srv, stores = S.serve_config(cfg, Log(), sd)
    n = len(cfg.devices())
    restores = [("restore", r, "rank%d.gcra" % f, r, n) for r in range(n) for f in range(2)]
    assert calls[:n] == [("store", r) for r in range(n)] and calls[n:n + len(restores)] == restores
    rest = [c[0] for c in calls[n + len(restores):]]
    assert "restore" not in rest and "store" not in rest and rest[0] == "limiter" and rest[-1] == "server"
    assert sd.stores == stores and sd.generation == 1
    sd.close()


@pytest.mark.parametrize("devices", ["0", "0,0,1"])
def test_a_failed_restore_closes_every_store_in_reverse_and_builds_no_server(tmp_path, monkeypatch, devices):
    _committed(tmp_path, 1)
    calls = []
    _fakes(monkeypatch, calls, fail_restore=True)
    cfg = S.parse_config(["--http", "--device", devices, "--snapshot-dir", str(tmp_path)], {})
    sd = P.SnapshotDir(cfg.snapshot_dir, cfg.store)
    with pytest.raises(P.SnapshotError, match="truncated"):
        S.serve_config(cfg, Log(), sd)
    n = len(cfg.devices())
    assert calls[-n:] == [("close", r) for r in reversed(range(n))]
    assert not any(c[0] in ("limiter", "connect", "ring", "server") for c in calls), calls
    sd.close()
