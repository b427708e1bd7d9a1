import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device here")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


# Every GPU test runs three times: with the engine's own choice of K1 pipeline by batch size, with the
# index-order pipeline forced for every batch above 255 requests, and with the sort pipeline only
# (GCRA_INDEX_MIN is read by gcra_create; include/gcra_b200.h GCRA_FLAG_INDEX_PATH / GCRA_FLAG_SORT_PATH).
K1_PATHS = {"auto": None, "index": "256", "sort": "0"}


@pytest.fixture(autouse=True)
def k1_path(request, monkeypatch):
    mode = getattr(request, "param", "auto")
    if K1_PATHS[mode] is None:
        monkeypatch.delenv("GCRA_INDEX_MIN", raising=False)
    else:
        monkeypatch.setenv("GCRA_INDEX_MIN", K1_PATHS[mode])
    return mode


def pytest_generate_tests(metafunc):
    if metafunc.definition.get_closest_marker("gpu") and "k1_path" in metafunc.fixturenames:
        for m in metafunc.definition.iter_markers("parametrize"):      # a test may pick its own pipelines
            names = m.args[0] if isinstance(m.args[0], (list, tuple)) else [x.strip() for x in m.args[0].split(",")]
            if "k1_path" in names:
                return
        metafunc.parametrize("k1_path", list(K1_PATHS), indirect=True)
