"""Every CUDA resource of the host code has one owner (throttlecrab_b200/csrc/gcra_owned.cuh): no other source file
creates or releases one directly, so a failed call releases what it made and no entry point keeps a list of frees."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "throttlecrab_b200", "csrc")
OWNER = "gcra_owned.cuh"
RAW = re.compile(r"\b(cudaMalloc|cudaMallocHost|cudaHostAlloc|cudaFree|cudaFreeHost|cudaEventCreate\w*|cudaEventDestroy|"
                 r"cudaStreamCreate\w*|cudaStreamDestroy|cudaIpcCloseMemHandle)\s*\(")


def test_only_the_owner_header_creates_or_releases_cuda_resources():
    found = []
    for name in sorted(os.listdir(CSRC)):
        if name == OWNER or not name.endswith((".cu", ".cuh", ".inc")):
            continue
        with open(os.path.join(CSRC, name)) as f:
            for no, line in enumerate(f, 1):
                found += ["%s:%d: %s" % (name, no, m.group(1)) for m in RAW.finditer(line)]
    assert not found, "raw CUDA resource calls outside %s:\n%s" % (OWNER, "\n".join(found))


def test_the_owner_header_covers_every_kind():
    with open(os.path.join(CSRC, OWNER)) as f:
        src = f.read()
    for call in ("cudaMalloc(", "cudaHostAlloc(", "cudaFree", "cudaFreeHost", "cudaStreamCreateWithFlags(",
                 "cudaStreamDestroy", "cudaEventCreateWithFlags(", "cudaEventDestroy", "cudaIpcCloseMemHandle"):
        assert call in src, call
