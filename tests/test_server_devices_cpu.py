"""--device / THROTTLECRAB_DEVICE with several devices: the list's parsing, CLI over environment, the refusals and
their exit status, the CUDA_DEVICE_MAX_CONNECTIONS check, and one store per entry with the capacity split.  No device
work."""
import os
import subprocess
import sys

import pytest

from throttlecrab_b200 import server as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_device_lists_from_the_cli_and_the_environment():
    assert S.parse_config(["--http", "--device", "0,1,2"], {}).device == (0, 1, 2)
    assert S.parse_config(["--http"], {"THROTTLECRAB_DEVICE": "3,1"}).device == (3, 1)
    assert S.parse_config(["--http", "--device", "0,0"], {"THROTTLECRAB_DEVICE": "1,2,3"}).device == (0, 0)
    assert S.parse_config(["--http", "--device", "4"], {"THROTTLECRAB_DEVICE": "1,2"}).device == 4
    assert S.parse_config(["--http"], {"THROTTLECRAB_DEVICE": " 1 , 2 "}).devices() == (1, 2)


def test_a_single_value_stays_an_int():
    for argv, env in [([], {}), (["--device", "2"], {}), ([], {"THROTTLECRAB_DEVICE": "5"})]:
        cfg = S.parse_config(["--http"] + argv, env)
        assert type(cfg.device) is int and cfg.devices() == (cfg.device,)


@pytest.mark.parametrize("value", ["", "0,", ",0", "0,,1", "0,x", "a", "0,-1", "-2", "1.5"])
def test_malformed_lists_are_refused(value):
    for argv, env in [(["--device", value], {}), ([], {"THROTTLECRAB_DEVICE": value})]:
        with pytest.raises(S.ConfigError) as e:
            S.parse_config(["--http"] + argv, env)
        assert e.value.status == 2
        assert str(e.value).startswith("invalid value '%s' for '--device': " % value), str(e.value)


def test_too_few_device_connections_are_refused_for_several_engines():
    for v in ("8", "0", "x"):
        with pytest.raises(S.ConfigError) as e:
            S.parse_config(["--http", "--device", "0,1"], {"CUDA_DEVICE_MAX_CONNECTIONS": v})
        assert e.value.status == 2 and "CUDA_DEVICE_MAX_CONNECTIONS" in str(e.value)
    assert S.parse_config(["--http", "--device", "0,1"], {"CUDA_DEVICE_MAX_CONNECTIONS": "32"}).device == (0, 1)
    assert S.parse_config(["--http", "--device", "1"], {"CUDA_DEVICE_MAX_CONNECTIONS": "8"}).device == 1
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="8")
    p = subprocess.run([sys.executable, "-m", "throttlecrab_b200.server", "--http", "--device", "0,1"], cwd=ROOT,
                       capture_output=True, text=True, env=env, timeout=60)
    assert p.returncode == 2 and "CUDA_DEVICE_MAX_CONNECTIONS=8" in p.stderr, p.stderr
    p = subprocess.run([sys.executable, "-m", "throttlecrab_b200.server", "--http", "--device", "0,,1"], cwd=ROOT,
                       capture_output=True, text=True, timeout=60)
    assert p.returncode == 2 and "an empty entry" in p.stderr, p.stderr


def test_importing_the_server_touches_no_cuda():
    """main sets CUDA_DEVICE_MAX_CONNECTIONS after its imports: they must not have initialised CUDA (nor loaded the
    engine library, whose calls would)"""
    code = ("import sys; import throttlecrab_b200.server, throttlecrab_b200.sharded; "
            "from throttlecrab_b200 import _native; import torch; "
            "assert _native._lib is None and not torch.cuda.is_initialized(); print('clean')")
    p = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=120)
    assert p.returncode == 0 and "clean" in p.stdout, p.stderr


def test_one_store_per_device_with_the_capacity_split(monkeypatch):
    built, calls = [], []

    class Fake:
        def __init__(self, **kw):
            self.kw = kw
            built.append(self)

        def close(self):
            calls.append(("close", built.index(self)))
    for cls in (S.PeriodicStore, S.ProbabilisticStore, S.AdaptiveStore):
        monkeypatch.setattr(cls, "__init__", lambda self, **kw: Fake.__init__(self, **kw))
        monkeypatch.setattr(cls, "close", lambda self: Fake.close(self))
    monkeypatch.setattr(S, "RateLimiter", lambda st: ("lim", st))
    import throttlecrab_b200.sharded as sharded
    monkeypatch.setattr(sharded, "connect_local", lambda lims, cap: calls.append(("connect", len(lims), cap)))

    class Ring:
        def __init__(self, lim, *geometry):
            calls.append(("ring", built.index(lim[1]), geometry))

        def peer_memory(self, on):
            calls.append(("p2p", on))
    monkeypatch.setattr(S, "MixedRing", Ring)
    monkeypatch.setattr(S, "ShardedMetrics", lambda lims, k: calls.append(("metrics", len(lims), k)))

    class Srv:
        def __init__(self, rings, listens, metrics):
            calls.append(("server", len(rings)))

        def port(self, t):
            return 1
    monkeypatch.setattr(S, "Server", Srv)
    cfg = S.parse_config(["--http", "--store", "adaptive", "--store-capacity", "1001", "--device", "0,0,3",
                          "--store-min-interval", "13", "--buffer-size", "512"], {})
    log = type("Log", (), {"lines": [], "info": lambda self, *a: self.lines.append(a[0] % a[1:])})()
    srv, stores = S.serve_config(cfg, log)
    assert [st.kw for st in stores] == [dict(p0=13, p1=300, p2=1_000_000, capacity=334, device=d) for d in (0, 0, 3)]
    assert stores == built and all(type(st) is S.AdaptiveStore for st in built)
    assert calls == [("connect", 3, 512)] + [("ring", r, (1, S.MAX_CONNS, S.IN_CAPACITY, 512)) for r in range(3)] + \
        [("p2p", True)] * 3 + [("metrics", 3, 100), ("server", 3)]
    assert any("rank 0 on cuda:0, rank 1 on cuda:0, rank 2 on cuda:3" in ln for ln in log.lines), log.lines

    # a step that fails closes every store made so far, in reverse order, and raises
    built.clear()
    calls.clear()

    def no_device(self, **kw):
        if kw["device"] == 99:
            raise RuntimeError("no device 99")
        Fake.__init__(self, **kw)
    monkeypatch.setattr(S.PeriodicStore, "__init__", no_device)
    cfg = S.parse_config(["--http", "--device", "0,1,99"], {})
    with pytest.raises(RuntimeError, match="no device 99"):
        S.serve_config(cfg, log)
    assert calls == [("close", 1), ("close", 0)]
