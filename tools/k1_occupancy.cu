// Occupancy of the sort pipeline's decide kernels, compiled from the engine's own kernel header with the library's
// flags (tools/k1_timeline.py builds and runs it): one JSON object per kernel on stdout.
//   registers    per thread, as ptxas allocated them
//   cta_regs     registers one CTA takes from the SM's 65 536 (per-warp allocation in units of 256)
//   blocks_per_sm / clusters: cudaOccupancyMaxActiveBlocksPerMultiprocessor / cudaOccupancyMaxActiveClusters
#include <cstdio>

#include "../throttlecrab_b200/csrc/gcra_kernels.cuh"

using namespace gcra;

template <typename K>
static void report(const char *name, K kernel, int threads, int cluster) {
    cudaFuncAttributes a{};
    cudaFuncGetAttributes(&a, kernel);
    int blocks = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kernel, threads, 0);
    const int cta_regs = ((a.numRegs * 32 + 255) / 256) * 256 * (threads / 32);
    printf("{\"kernel\": \"%s\", \"threads\": %d, \"registers\": %d, \"local_bytes\": %zu, \"cta_regs\": %d, "
           "\"blocks_per_sm\": %d", name, threads, a.numRegs, a.localSizeBytes, cta_regs, blocks);
    if (cluster > 1) {
        if (cluster > 8) cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(16 * cluster);
        cfg.blockDim = dim3(threads);
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cluster;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int clusters = 0;
        const cudaError_t e = cudaOccupancyMaxActiveClusters(&clusters, kernel, &cfg);
        printf(", \"cluster\": %d, \"clusters\": %d", cluster, e == cudaSuccess ? clusters : -1);
    }
    printf("}\n");
}

int main() {
    report("decide_kernel<false, false>", decide_kernel<false, false>, DECIDE_THREADS, 1);
    report("decide_kernel<false, true>", decide_kernel<false, true>, DECIDE_THREADS, 1);
    report("list_runs_kernel", list_runs_kernel, DECIDE_THREADS, 1);
    report("decide_runs_kernel<1, false, false>", decide_runs_kernel<1, false, false>, LONG_THREADS, 1);
    report("decide_runs_kernel<CLUSTER_CTAS, false, false>", decide_runs_kernel<CLUSTER_CTAS, false, false>, LONG_THREADS,
           CLUSTER_CTAS);
    report("sort_sweep_kernel", sort_sweep_kernel, TILE_THREADS, 1);
    return cudaGetLastError() == cudaSuccess ? 0 : 1;
}
