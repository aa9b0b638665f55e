// The fp64 reduction of the preprocessing normalisations (preprocess.cu for LIDC, petct_preprocess.cu for PET-CT): a fixed number of
// partial sums, each a block's tree over its threads' sequential sums, then one block's tree over the partial sums.  The tree's shape
// depends only on the element count, so a volume reduces to the same bits on every run and every device.
#pragma once
#include <math.h>

#include "mdt_common.cuh"

namespace mdt {

constexpr int kRedBlocks = 1024;      // fixed number of partial sums, whatever the device
constexpr int kRedThreads = 256;

__device__ __forceinline__ double block_tree_sum(double v, double *sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int h = blockDim.x / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) sh[threadIdx.x] = __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + h]);
        __syncthreads();
    }
    return sh[0];
}

// one block of kRedBlocks threads: the tree over the partial sums.  pass 0: stats[0] = mean; pass 1: stats[1] = population std
// (static: one copy per including translation unit)
static __global__ void __launch_bounds__(kRedBlocks) red_final_kernel(const double *__restrict__ partial, long long n, int pass, double *__restrict__ stats) {
    __shared__ double sh[kRedBlocks];
    const double s = block_tree_sum(partial[threadIdx.x], sh);
    if (threadIdx.x == 0) stats[pass] = pass == 0 ? s / (double)n : sqrt(s / (double)n);
}

}  // namespace mdt
