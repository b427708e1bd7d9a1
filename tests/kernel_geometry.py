"""The hot-run geometry of the decide kernels, read from throttlecrab_b200/csrc/gcra_kernels.cuh.

The build passes none of GCRA_LONG_MIN, GCRA_GIANT_MIN or GCRA_CLUSTER as -D, so the defaults in the header are what
runs.  The CPU model of the hot-run kernel (test_algorithm_model.py) and the GPU scenarios built on it
(test_gpu_fsm_cycles.py, test_gpu_hot_run_listing.py) take their strides and thresholds from here, so that a change of
the kernels' geometry moves them too instead of leaving them aimed at positions that are no longer edges."""
import os
import re

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "throttlecrab_b200", "csrc",
                      "gcra_kernels.cuh")
PATTERNS = {
    "LONG_RUN_MIN": r"^#define GCRA_LONG_MIN (\d+)$",
    "GIANT_RUN_MIN": r"^#define GCRA_GIANT_MIN (\d+)$",
    "CLUSTER_CTAS": r"^#define GCRA_CLUSTER (\d+)$",
    "LONG_THREADS": r"^constexpr int LONG_THREADS = (\d+);",
    "SMALL_MAX": r"^constexpr u32 SMALL_MAX = (\d+);",
}
# the header must use the macros above, not literals: else the parsed defaults would not be what runs
USES = [r"^constexpr u32 LONG_RUN_MIN = GCRA_LONG_MIN;", r"^constexpr u32 GIANT_RUN_MIN = GCRA_GIANT_MIN;",
        r"^constexpr int CLUSTER_CTAS = GCRA_CLUSTER;"]


def parse(src):
    out = {}
    for name, pat in PATTERNS.items():
        m = re.findall(pat, src, re.M)
        if len(m) != 1:
            raise AssertionError("%s: expected one match of %r in %s, found %d" % (name, pat, HEADER, len(m)))
        out[name] = int(m[0])
    for pat in USES:
        if len(re.findall(pat, src, re.M)) != 1:
            raise AssertionError("expected one match of %r in %s" % (pat, HEADER))
    return out


with open(HEADER) as _f:
    GEOMETRY = parse(_f.read())

LONG_THREADS = GEOMETRY["LONG_THREADS"]          # threads of one hot-run CTA
CLUSTER_CTAS = GEOMETRY["CLUSTER_CTAS"]          # CTAs of one hot-run cluster
LONG_RUN_MIN = GEOMETRY["LONG_RUN_MIN"]          # a run of this many rows or more is hot: one CTA
GIANT_RUN_MIN = GEOMETRY["GIANT_RUN_MIN"]        # ... this many or more: one cluster
SMALL_MAX = GEOMETRY["SMALL_MAX"]                # batches of up to this many rows: the one-CTA small-batch kernel
CTA_STRIDE = LONG_THREADS                        # rows a one-CTA group decides per stride
CLUSTER_STRIDE = CLUSTER_CTAS * LONG_THREADS     # ... and a cluster
