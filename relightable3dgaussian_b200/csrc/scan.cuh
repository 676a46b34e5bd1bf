// Single-CTA exclusive scan of per-block counts, shared by the row-compaction passes (compact.cu: one channel, the
// keep mask; densify.cu: several channels at once, one per output segment / counter).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace r3dg {

// sums: NCH channels of n block counts, channel c at sums + c * stride.  Each channel is replaced in place by its
// exclusive prefix; its total goes to totals[c].  One CTA of 1024 threads.  T = unsigned long long for totals that may
// exceed 2^32 (tsdf.cu's mesh counts).
template <int NCH, typename T = uint32_t>
__global__ void __launch_bounds__(1024) block_sums_scan_kernel(long long n, long long stride, T* __restrict__ sums,
                                                               T* __restrict__ totals) {
    __shared__ T s_warp[32];
    __shared__ T s_carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c = 0; c < NCH; ++c) {
        T* ch = sums + c * stride;
        if (threadIdx.x == 0) s_carry = 0;
        __syncthreads();
        for (long long base = 0; base < n; base += 1024) {
            const long long i = base + threadIdx.x;
            const T v = i < n ? ch[i] : T(0);
            T inc = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const T t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
            if (lane == 31) s_warp[warp] = inc;
            __syncthreads();
            if (warp == 0) {
                T w = s_warp[lane], winc = w;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const T t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
                s_warp[lane] = winc - w;                       // exclusive prefix of the warp totals
            }
            __syncthreads();
            const T excl = s_carry + s_warp[warp] + inc - v;
            if (i < n) ch[i] = excl;
            __syncthreads();
            if (threadIdx.x == 1023) s_carry = excl + v;
            __syncthreads();
        }
        if (threadIdx.x == 0) totals[c] = s_carry;
        __syncthreads();
    }
}

}  // namespace r3dg
