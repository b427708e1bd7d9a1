"""The server's configuration against config.rs's, transcribed in tests/golden/server_config.json: every flag, its
THROTTLECRAB_* variable and default, CLI over environment over default, the refusals and their exit statuses,
--list-env-vars, and the store each --store builds.  No device work."""
import json
import os
import subprocess
import sys

import pytest

from throttlecrab_b200 import server as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "server_config.json")))


def _dest(flag):
    return flag[2:].replace("-", "_")


def test_every_flag_env_name_and_default_matches_the_reference():
    mine = {f: (e, d) for f, e, d, _ in S.FLAGS}
    for row in GOLDEN["flags"]:
        assert mine.pop(row["flag"]) == (row["env"], row["default"]), row
    assert list(mine) == ["--device"]                  # the one addition
    cfg = S.parse_config(["--http"], {})
    for row in GOLDEN["flags"]:
        want = True if row["flag"] == "--http" else row["default"]
        assert getattr(cfg, _dest(row["flag"])) == want, row
    assert cfg.device == 0 and S.STORE_TYPES == tuple(GOLDEN["store_types"])


@pytest.mark.parametrize("row", GOLDEN["flags"], ids=lambda r: r["flag"])
def test_cli_over_env_over_default(row):
    flag, env, default = row["flag"], row["env"], row["default"]
    if isinstance(default, bool):
        assert getattr(S.parse_config(["--redis", "--http", "--grpc"], {env: "false"}), _dest(flag)) is True
        on = S.parse_config(["--redis"] if flag != "--redis" else ["--http"], {env: "true"})
        assert getattr(on, _dest(flag)) is True
        off = S.parse_config(["--redis"] if flag != "--redis" else ["--http"], {env: "false"})
        assert getattr(off, _dest(flag)) is False
        return
    if flag == "--store":
        env_v, cli_v = "ADAPTIVE", "probabilistic"
        want_env = "adaptive"
    elif isinstance(default, int):
        env_v, cli_v = "7", "9"
        want_env = 7
    else:
        env_v, cli_v = "from-env", "from-cli"
        want_env = "from-env"
    assert getattr(S.parse_config(["--http"], {env: env_v}), _dest(flag)) == want_env
    want_cli = int(cli_v) if isinstance(default, int) else cli_v
    assert getattr(S.parse_config(["--http", flag, cli_v], {env: env_v}), _dest(flag)) == want_cli
    assert getattr(S.parse_config(["--http"], {}), _dest(flag)) == default


def test_transports_from_the_environment_and_their_listens():
    cfg = S.parse_config([], {"THROTTLECRAB_REDIS": "1", "THROTTLECRAB_REDIS_PORT": "7000",
                              "THROTTLECRAB_HTTP": "yes"})
    assert cfg.listens() == [("http", "0.0.0.0", 8080), ("redis", "0.0.0.0", 7000)]
    assert S.parse_config(["--grpc", "--grpc-host", "127.0.0.1"], {}).listens() == [("grpc", "127.0.0.1", 8070)]


def test_no_transport_is_refused_with_the_reference_error():
    with pytest.raises(S.ConfigError) as e:
        S.parse_config([], {"THROTTLECRAB_HTTP": "false"})
    assert str(e.value).startswith(GOLDEN["no_transport_error"])
    assert e.value.status == GOLDEN["no_transport_exit_status"]
    p = subprocess.run([sys.executable, "-m", "throttlecrab_b200.server"], cwd=ROOT, capture_output=True, text=True,
                       env={k: v for k, v in os.environ.items() if not k.startswith("THROTTLECRAB_")}, timeout=60)
    assert p.returncode == GOLDEN["no_transport_exit_status"]
    assert GOLDEN["no_transport_error"] in p.stderr


def test_out_of_range_and_malformed_values_are_refused():
    lo, hi = GOLDEN["max_denied_keys_range"]
    assert S.parse_config(["--http", "--max-denied-keys", str(hi)], {}).max_denied_keys == hi
    assert S.parse_config(["--http", "--max-denied-keys", str(lo)], {}).max_denied_keys == lo
    for argv, env in [(["--max-denied-keys", str(hi + 1)], {}), ([], {"THROTTLECRAB_MAX_DENIED_KEYS": "10001"}),
                      (["--store", "lru"], {}), ([], {"THROTTLECRAB_STORE": "lru"}),
                      (["--http-port", "x"], {}), (["--http-port", "65536"], {}), (["--buffer-size", "0"], {})]:
        with pytest.raises(S.ConfigError) as e:
            S.parse_config(["--http"] + argv, env)
        assert e.value.status == 2, (argv, env)


def test_list_env_vars_lists_every_variable_and_exits_zero():
    p = subprocess.run([sys.executable, "-m", "throttlecrab_b200.server", "--list-env-vars"], cwd=ROOT,
                       capture_output=True, text=True, timeout=60)
    assert p.returncode == 0
    for row in GOLDEN["flags"]:
        line = [ln for ln in p.stdout.splitlines() if ln.strip().startswith(row["env"] + "=")]
        assert len(line) == 1, row
        assert "[default: %s]" % str(row["default"]).lower() in line[0]


@pytest.mark.parametrize("store", GOLDEN["store_types"])
def test_store_built_per_store_flag(store, monkeypatch):
    built = {}

    def fake_init(self, **kw):
        built.update(kw, cls=type(self).__name__)
    for cls in (S.PeriodicStore, S.ProbabilisticStore, S.AdaptiveStore):
        monkeypatch.setattr(cls, "__init__", fake_init)
    cfg = S.parse_config(["--http", "--store", store, "--store-capacity", "123", "--store-cleanup-interval", "11",
                          "--store-cleanup-probability", "12", "--store-min-interval", "13",
                          "--store-max-interval", "14", "--store-max-operations", "15", "--device", "2"], {})
    S.make_store(cfg)
    want = {"periodic": ("PeriodicStore", {"p0": 11}), "probabilistic": ("ProbabilisticStore", {"p0": 12}),
            "adaptive": ("AdaptiveStore", {"p0": 13, "p1": 14, "p2": 15})}[store]
    assert built == dict(want[1], cls=want[0], capacity=123, device=2)
