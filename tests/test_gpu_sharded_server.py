"""The native server over several engines of one process (gcra_server_create_sharded, server.Server over a list of
mixed rings, --device 0,1,...).  Each case runs its engines in a child process (tests/sharded_server_worker.py) with
CUDA_DEVICE_MAX_CONNECTIONS=32, as test_gpu_sharded_rings.py does: engines of one process wait for each other in
kernels, and a wait kernel must not sit in a hardware queue ahead of the kernel it waits for.  Loop-back: 2 to 4
engines on GPU 0; with 2 GPUs, engine r on GPU r.  Then the CLI with --device 0,0 as a subprocess."""
import os
import re
import random
import signal
import socket
import subprocess
import sys
import time

import pytest

from test_gpu_server import ROOT, grpc_client
from test_http_cpu import body_of, request
from test_resp import _cmd, _throttle

pytestmark = [pytest.mark.gpu, pytest.mark.parametrize("k1_path", ["auto"], indirect=True)]
HERE = os.path.dirname(os.path.abspath(__file__))


def _worker(*args):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    out = subprocess.run([sys.executable, os.path.join(HERE, "sharded_server_worker.py")] + [str(a) for a in args],
                         capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0 and "sharded server ok" in out.stdout, out.stdout[-3000:] + out.stderr[-5000:]


@pytest.mark.parametrize("world", [2, 3, 4])
def test_serve_is_process_connections_sharded(world):
    """one serve against the replay (keys shared across ranks and transports, a hot key, GET /metrics naming a key
    that only a non-owner rank parsed, per-rank transport counts); against ONE engine where no slot fills; a rank with
    more connections than max_conns and more bytes than in_capacity while the others tick empty"""
    _worker("serve", world)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_byte_splits_across_reads_and_serves(world):
    _worker("splits", world)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_every_rank_sweeps(world):
    """a periodic store: serves past the cleanup interval shrink every rank's table, decisions as the replay's"""
    _worker("sweep", world)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_general_path_failure_on_rank_1(world):
    _worker("general", world)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_refusals_leave_nothing_open(world):
    _worker("refusals", world)


def _gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.skipif(_gpus() < 2, reason="needs 2 GPUs")
def test_serve_on_two_gpus():
    """--device 0,1: engine r on GPU r"""
    _worker("serve", 2, "--gpus")


def _cli(devices, env=None):
    args = [sys.executable, "-m", "throttlecrab_b200.server", "--redis", "--http", "--grpc", "--device", devices,
            "--buffer-size", "4096", "--store-capacity", "1000"]
    for t in ("redis", "http", "grpc"):
        args += ["--%s-host" % t, "127.0.0.1", "--%s-port" % t, "0"]
    return subprocess.Popen(args, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)


def test_subprocess_cli_with_two_engines():
    env = {k: v for k, v in os.environ.items() if k != "CUDA_DEVICE_MAX_CONNECTIONS"}   # (the server sets it)
    p = _cli("0,0", env)
    try:
        ports, lines, t = {}, [], time.time() + 120
        while len(ports) < 3 and time.time() < t:
            ln = p.stdout.readline()
            assert ln, "".join(lines)
            lines.append(ln)
            m = re.search(r"Starting (\w+) transport on 127\.0\.0\.1:(\d+)", ln)
            if m:
                ports[m.group(1)] = int(m.group(2))
        assert sorted(ports) == ["HTTP", "Redis", "gRPC"], lines
        lines.append(p.stdout.readline())
        lines.append(p.stdout.readline())
        lines.append(p.stdout.readline())
        assert any("rank 0 on cuda:0, rank 1 on cuda:0" in ln for ln in lines), lines

        def ask(port, data, until):
            with socket.create_connection(("127.0.0.1", port), timeout=20) as s:
                s.sendall(data)
                got = b""
                while not until(got):
                    d = s.recv(4096)
                    assert d, got
                    got += d
                return got
        r = ask(ports["Redis"], _throttle("sub", 3, 10, 60), lambda g: g.count(b"\r\n") >= 6)
        assert r.startswith(b"*5\r\n:1\r\n:3\r\n")                          # allowed, limit 3
        assert ask(ports["Redis"], _cmd("PING"), lambda g: b"\r\n" in g) == b"+PONG\r\n"
        h = ask(ports["HTTP"], request(body_of("sub", 3, 10, 60)), lambda g: b"\r\n\r\n" in g and g.endswith(b"}"))
        assert h.startswith(b"HTTP/1.1 200"), h
        g = ask(ports["gRPC"], grpc_client(random.Random(7), ["sub"], 0, tail=False), lambda g: b"grpc-status" in g)
        assert b"grpc-status" in g
        p.send_signal(signal.SIGTERM)
        assert p.wait(20) == 0
    finally:
        if p.poll() is None:
            p.kill()
            p.wait(10)
        p.stdout.close()


def test_subprocess_cli_refuses_a_bad_device_list():
    p = _cli("0,99")
    try:
        out, _ = p.communicate(timeout=120)
        assert p.returncode != 0 and "gcra_create failed" in out, out
    finally:
        if p.poll() is None:
            p.kill()
            p.wait(10)
