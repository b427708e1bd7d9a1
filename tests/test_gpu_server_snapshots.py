"""The server's snapshot directory on the GPU (--snapshot-dir, persist.SnapshotDir).  Restart equivalence runs in a
child process (tests/server_snapshot_worker.py) with CUDA_DEVICE_MAX_CONNECTIONS=32, as the sharded server's tests do:
a server restarted into another world size answers byte for byte as a control server on one engine that never
stopped, after a shutdown save and after a background save whose cut is the serve boundary; a save that cannot create
its generation leaves serving and the committed generation alone.  Then the CLI: a truncated rank file refuses the
start before any port is bound, and limits survive SIGTERM and restarts with --device 0,0 and back."""
import json
import os
import re
import signal
import socket
import subprocess
import sys
import time

import pytest

from test_gpu_server import ROOT
from test_resp import _throttle

pytestmark = [pytest.mark.gpu, pytest.mark.parametrize("k1_path", ["auto"], indirect=True)]
HERE = os.path.dirname(os.path.abspath(__file__))


def _worker(*args):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    out = subprocess.run([sys.executable, os.path.join(HERE, "server_snapshot_worker.py")] + [str(a) for a in args],
                         capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0 and "server snapshot ok" in out.stdout, out.stdout[-3000:] + out.stderr[-5000:]


@pytest.mark.parametrize("old,new", [(1, 1), (1, 2), (2, 1), (2, 3), (3, 2)])
def test_a_restarted_server_answers_as_one_that_never_stopped(old, new):
    _worker("restart", old, new)


@pytest.mark.parametrize("world", [1, 2])
def test_a_failed_save_leaves_serving_and_the_committed_generation(world):
    _worker("failed", world)


# ---- the CLI ---------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _start(d, devices="0", interval=60, port=0):
    args = [sys.executable, "-m", "throttlecrab_b200.server", "--redis", "--redis-host", "127.0.0.1",
            "--redis-port", str(port), "--store-capacity", "1000", "--buffer-size", "4096", "--device", devices,
            "--snapshot-dir", d, "--snapshot-interval", str(interval)]
    env = {k: v for k, v in os.environ.items() if k != "CUDA_DEVICE_MAX_CONNECTIONS"}   # (the server sets it)
    return subprocess.Popen(args, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)


def _port(p):
    lines, t = [], time.time() + 120
    while time.time() < t:
        ln = p.stdout.readline()
        assert ln, "".join(lines)
        lines.append(ln)
        m = re.search(r"Starting Redis transport on 127\.0\.0\.1:(\d+)", ln)
        if m:
            return int(m.group(1)), lines
    raise AssertionError("".join(lines))


def _stop(p):
    p.send_signal(signal.SIGTERM)
    out = p.stdout.read()
    assert p.wait(60) == 0, out
    return out


def _end(p):
    """(cleanup after a failed assertion)"""
    if p.poll() is None:
        p.terminate()
        try:
            p.wait(30)
        except subprocess.TimeoutExpired:
            p.kill()
            p.wait(10)
    p.stdout.close()


def _throttles(port, key, n):
    """n THROTTLE key 2 1 3600 1 on one connection -> [allowed per call]: a new key's first two are allowed, the third
    is denied, and its entry lives two hours (with max_burst 1 the reference gives the entry no time to live)"""
    with socket.create_connection(("127.0.0.1", port), timeout=20) as s:
        s.sendall(_throttle(key, 2, 1, 3600, 1) * n)
        got = b""
        while got.count(b"*5\r\n") < n or not got.endswith(b"\r\n") or got.count(b"\r\n") < 6 * n:
            d = s.recv(4096)
            assert d, got
            got += d
    return [int(r.split(b"\r\n")[0][1:]) for r in got.split(b"*5\r\n")[1:]]


def _manifest(d):
    with open(os.path.join(d, "MANIFEST")) as f:
        return json.load(f)


def _two_gpus():
    import torch
    return torch.cuda.device_count() >= 2


def test_cli_keeps_limits_across_restarts_and_device_lists(tmp_path):
    d = str(tmp_path / "snap")
    p = _start(d, interval=1)
    try:
        port, _ = _port(p)
        assert _throttles(port, "k", 3) == [1, 1, 0]
        t = time.time() + 60
        while not (os.path.exists(os.path.join(d, "MANIFEST")) and _manifest(d)["generation"] >= 1):
            assert time.time() < t and p.poll() is None
            time.sleep(0.2)
        out = _stop(p)
        assert "Saved snapshot generation" in out, out
        assert _manifest(d)["world"] == 1
    finally:
        _end(p)
    for devices, world in [("0,0", 2)] + ([("0,1", 2)] if _two_gpus() else []) + [("0", 1)]:
        p = _start(d, devices)
        try:
            port, lines = _port(p)
            assert any("Restored snapshot generation" in ln for ln in lines), lines
            assert _throttles(port, "k", 1) == [0], devices                # still denied
            assert _throttles(port, "other", 1) == [1]
            _stop(p)
            m = _manifest(d)
            assert m["world"] == world and len(m["files"]) == world, (devices, m)
        finally:
            _end(p)


def test_cli_refuses_a_truncated_snapshot_before_binding(tmp_path):
    d = str(tmp_path / "snap")
    p = _start(d)
    try:
        port, _ = _port(p)
        assert _throttles(port, "k", 3) == [1, 1, 0]
        _stop(p)
    finally:
        _end(p)
    f = os.path.join(d, "gen-%d" % _manifest(d)["generation"], "rank0.gcra")
    with open(f, "r+b") as fh:
        fh.truncate(os.path.getsize(f) - 7)
    port = _free_port()
    p = _start(d, port=port)
    try:
        out, _ = p.communicate(timeout=120)
        assert p.returncode != 0 and "snapshot restore of" in out and "rank0.gcra" in out, out
        assert "Starting Redis transport" not in out
        with pytest.raises(OSError):
            socket.create_connection(("127.0.0.1", port), timeout=5).close()
    finally:
        _end(p)
    assert _manifest(d)["generation"] == 1 and os.path.getsize(f) > 0            # left for the operator
