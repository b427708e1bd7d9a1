"""K2 (expired-key sweep) on BASELINE.json configs[2]: 100 M resident keys, sweeps at expired fractions
0 / 1 / 50 / 100 % (bench.py: sweep_block); achieved HBM GB/s against the H100 SXM data-sheet peak.  One JSON line.
GCRA_SWEEP_MODE=0|1|2 selects the eviction store variant (csrc/gcra_kernels.cuh: sweep_kernel)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import throttlecrab_b200 as tc  # noqa: E402

keys = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000_000
peak = bench.PEAK_HBM_GBS
out = bench.sweep_block(tc, peak, 0, keys)
out["sweep_mode"] = int(os.environ.get("GCRA_SWEEP_MODE", "0"))
print(json.dumps(out), flush=True)
