"""Sharded ring metrics (gcra_ring_metrics_sharded, gcra_ring_names_keep) and metrics.ShardedMetrics: ring metrics for
rings whose ticks are peer-memory ticks.  Each case runs its engines in a child process
(tests/sharded_ring_metrics_worker.py, tests/sharded_ring_metrics_ipc_worker.py) with CUDA_DEVICE_MAX_CONNECTIONS=32,
as tests/test_gpu_sharded_rings.py does: engines of one process wait for each other in kernels."""
import os
import subprocess
import sys

import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.parametrize("k1_path", ["auto"], indirect=True)]
HERE = os.path.dirname(os.path.abspath(__file__))


def _run(script, *args):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    out = subprocess.run([sys.executable, os.path.join(HERE, script)] + [str(a) for a in args],
                         capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0 and "sharded ring metrics ok" in out.stdout, out.stdout[-3000:] + out.stderr[-5000:]


def _worker(*args):
    _run("sharded_ring_metrics_worker.py", *args)


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_counts_and_names_per_rank(world):
    """fuzzed connections of every protocol, keys shared across ranks and transports, a hot key, a filling slot, empty
    ranks: each rank's transport counts equal its rows', each key denied through a rank is named there with its exact
    bytes (or too long) and no other is, the owners' merged top list equals one oracle replay's denied counts; replies,
    outcomes, final entries and launches (one more per submit with rows) against twins with sharded metrics off"""
    _worker("counts", world)


def test_world_1_text_equals_metrics():
    """ShardedMetrics([lim]) with ring p2p off serves the text Metrics serves on a twin engine"""
    _worker("world1_text", 1)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_sharded_driver_serves_get_metrics(world):
    """process_connections_sharded with a ShardedMetrics: GET /metrics against a model of metrics.rs"""
    _worker("driver", world)


@pytest.mark.parametrize("world", [2, 3])
def test_pruning_keeps_the_survivors_names(world):
    _worker("prune", world)


@pytest.mark.parametrize("world", [1, 2])
def test_a_full_name_table_counts_what_it_drops(world):
    _worker("full", world)


def test_refusals_leave_the_engines_usable():
    """ring metrics and sharded ring metrics in both orders, max_keys above 10,000, a keep while off"""
    _worker("refusals", 2)


def test_two_processes_on_one_gpu():
    """one engine per process over CUDA IPC windows: per-rank counts and names against one oracle"""
    _run("sharded_ring_metrics_ipc_worker.py", 2)


def _gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.skipif(_gpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("scenario", ["counts", "driver", "prune"])
def test_one_process_drives_two_gpus(scenario):
    _worker(scenario, 2, "--gpus")


@pytest.mark.skipif(_gpus() < 2, reason="needs 2 GPUs")
def test_two_processes_on_two_gpus():
    _run("sharded_ring_metrics_ipc_worker.py", 2, "--gpus")
