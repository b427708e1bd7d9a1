"""Rings over peer memory (gcra_ring_p2p, gcra_resp_ring_submit_route / _finish): N engines' mixed rings served
against one hash-sharded table.  Each case runs its engines in a child process (tests/sharded_rings_worker.py), so
that a tick a peer never delivers ends that process, not the test session.  Loop-back: 1 to 4 engines of one process
on one GPU, and 2 processes on one GPU (CUDA IPC windows).  With 2 GPUs: one process drives both (window pointers,
peer access), and 2 processes one GPU each (CUDA IPC).  The child runs with
CUDA_DEVICE_MAX_CONNECTIONS=32, as the other loop-back tests: engines of one process wait for each other in kernels,
and a wait kernel must not sit in a hardware queue ahead of the kernel it waits for."""
import os
import subprocess
import sys

import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.parametrize("k1_path", ["auto"], indirect=True)]
HERE = os.path.dirname(os.path.abspath(__file__))


def _worker(*args):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")     # see test_gpu_sharded.py's loop-back test
    out = subprocess.run([sys.executable, os.path.join(HERE, "sharded_rings_worker.py")] + [str(a) for a in args],
                         capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0 and "sharded rings ok" in out.stdout, out.stdout[-3000:] + out.stderr[-5000:]


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_ring_ticks_against_one_oracle(world):
    """fuzzed connections of every protocol, keys shared across ranks and transports, a hot key in every rank, one
    rank's slot filling (stop 3), ranks with 0 connections, 2 ring slots in flight per engine: outcomes, replies,
    final entries and counters against one oracle store"""
    _worker("ticks", world)


@pytest.mark.parametrize("world", [2, 3])
def test_seeded_engines(world):
    _worker("seeded", world)


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_ring_ticks_between_p2p_submit_ticks(world):
    """ring ticks and gcra_p2p_submit ticks as one tick sequence, mixed within a tick, more ticks in flight than
    P2P_DEPTH (world 1: bulk ticks of one rank, whose inbox view has an empty second segment)"""
    _worker("mixed_ticks", world)


@pytest.mark.parametrize("world", [2, 4])
def test_tight_table_grows_on_owners_between_ring_ticks(world):
    _worker("tight", world)


def test_world_1_equals_the_plain_ring():
    _worker("world1", 1)


def test_refusals_leave_the_engines_usable():
    """not connected, metrics on (both orders), row_capacity above the cap, differing seeds"""
    _worker("refusals", 2)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sharded_driver_equals_one_engine(world):
    """mixed.process_connections_sharded over `world` engines against process_connections(ring=None) on one engine
    over the joined connection list, general paths included"""
    _worker("driver", world)


def _ipc(*args):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    out = subprocess.run([sys.executable, os.path.join(HERE, "sharded_rings_ipc_worker.py")] + [str(a) for a in args],
                         capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0 and "sharded rings ok" in out.stdout, out.stdout[-3000:] + out.stderr[-5000:]


def test_ring_ticks_between_processes_on_one_gpu():
    """one engine per process, windows exchanged as CUDA IPC handles, every ring tick one gcra_resp_ring_submit,
    gcra_p2p_submit ticks of another process between them, against one oracle (both processes on GPU 0)"""
    _ipc(2)


def test_a_differing_seed_is_refused_through_ipc_windows():
    _ipc(2, "--bad-seed")


def _gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.skipif(_gpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("scenario", ["ticks", "driver"])
def test_one_process_drives_two_gpus(scenario):
    """engine r on GPU r, connected with window pointers: gcra_p2p_connect enables peer access"""
    _worker(scenario, 2, "--gpus")


@pytest.mark.skipif(_gpus() < 2, reason="needs 2 GPUs")
def test_ring_ticks_between_processes_on_two_gpus():
    """the same processes with engine r on GPU r: rows and results cross between the GPUs through IPC windows"""
    _ipc(2, "--gpus")
