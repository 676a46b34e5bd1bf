// Fixed-order fp64 sums shared by the image-space losses (ssim.cu, smooth.cu).  Each loss kernel writes one partial
// per CTA with cta_partial, and reduce_partials_kernel sums the partials, both in a fixed order, so every loss value
// is deterministic run to run.
#pragma once
#include <cstddef>
#include <cuda_runtime.h>

namespace r3dg {
namespace {

constexpr int kReduceNT = 256;

// *dst = the CTA's sum of `acc` over its NT threads in a fixed order: butterfly within each warp, then the warps in
// index order.  Every thread of the CTA must call it.
template <int NT>
__device__ __forceinline__ void cta_partial(double acc, double* dst) {
    __shared__ double warp_sum[NT / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < NT / 32; ++w) s += warp_sum[w];
        *dst = s;
    }
}

// out[b] = sum(partial[b * per .. (b+1) * per)) / count, one CTA per output, fixed summation order
__global__ void __launch_bounds__(kReduceNT) reduce_partials_kernel(const double* __restrict__ partial, long long per,
                                                                   double count, float* __restrict__ out) {
    __shared__ double s[kReduceNT];
    const double* p = partial + (size_t)blockIdx.x * per;
    double acc = 0.0;
    for (long long i = threadIdx.x; i < per; i += kReduceNT) acc += p[i];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int o = kReduceNT / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[blockIdx.x] = (float)(s[0] / count);
}

}  // namespace
}  // namespace r3dg
