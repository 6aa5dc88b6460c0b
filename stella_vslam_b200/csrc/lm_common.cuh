// lm_common.cuh -- pieces shared by the single-CTA Levenberg-Marquardt kernels: the pose optimiser (lba_kernels.cu) and the Sim3
// transform optimiser (transform_kernels.cu).
#pragma once

#include <cmath>

namespace b200 {

// RobustKernelHuber: rho[1] weight and rho[0] cost
__device__ __forceinline__ double huber_weight(double e2, double delta) { return (e2 <= delta * delta) ? 1.0 : delta / sqrt(e2); }
__device__ __forceinline__ double huber_cost(double e2, double delta) { return (e2 <= delta * delta) ? e2 : 2 * sqrt(e2) * delta - delta * delta; }

// sum of v over a CTA of kThreads threads in a fixed order: warp shuffle tree, then the warp leaders in index order.  out[0..N) is
// written by threads 0..N-1; scratch holds (kThreads / 32) * N doubles.
template <int kThreads, int N>
__device__ __forceinline__ void cta_sum(double (&v)[N], double* out, double* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < N; ++i) {
#pragma unroll
        for (int s2 = 16; s2 > 0; s2 >>= 1) v[i] += __shfl_down_sync(0xFFFFFFFFu, v[i], s2);
    }
    __syncthreads();
    if (lane == 0)
#pragma unroll
        for (int i = 0; i < N; ++i) scratch[warp * N + i] = v[i];
    __syncthreads();
    if (threadIdx.x < N) {
        double r = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) r += scratch[w * N + threadIdx.x];
        out[threadIdx.x] = r;
    }
    __syncthreads();
}

}  // namespace b200
