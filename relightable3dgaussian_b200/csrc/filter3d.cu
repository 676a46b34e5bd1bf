// Mip-Splatting's 3D smoothing filter (Yu et al., CVPR 2024): the per-Gaussian filter size f that the rasterizer's
// filter_3d input takes, from the highest sampling rate at which any training camera sees the Gaussian.  The host side
// is relightable3dgaussian_b200/filter3d.py.  Two launches, no host synchronisation:
//   filter3d_min_kernel     one thread per Gaussian, the cameras staged through shared memory in chunks: the least
//                           valid depth d_i (-1 when no camera sees the Gaussian) into `out`, and the largest d_i of
//                           the block into one word of tmp by atomicMax on the float bits (d > 0.2 > 0, so the bits
//                           order as the values);
//   filter3d_finish_kernel  f_i = (d_i / F) sqrt(0.2), unseen rows taking that largest d (0 when nothing is seen).
// min and max do not depend on the order of their operands, so the result is bitwise reproducible.
#include "common.cuh"
#include "kernels.h"

namespace r3dg {

#define F3D_THREADS 256
#define F3D_CHUNK 256           // cameras staged per round: 256 x 20 floats = 20 KB of shared memory
#define F3D_CAMF 20             // per camera: the view matrix with fx fy cx cy in its unused column, and 4 bounds

// a camera's record in shared memory: the view matrix at offsets 0..15 (xform_row_ reads m[r], m[4 + r], m[8 + r],
// m[12 + r] for r = 0, 1, 2), with column 3, which it never reads, replaced by fx, fy, cx, cy at 3, 7, 11, 15; then the
// bounds u_lo, u_hi, v_lo, v_hi at 16..19
__device__ __forceinline__ void stage_camera(float* s, const float* __restrict__ vm, const float* __restrict__ k) {
#pragma unroll
    for (int j = 0; j < 16; ++j) s[j] = vm[j];
    const double W = k[4], H = k[5];
    // the bounds as torch compares an fp32 tensor with a Python float: the double product rounded to fp32
    s[3] = k[0]; s[7] = k[1]; s[11] = k[2]; s[15] = k[3];
    s[16] = (float)(-0.15 * W); s[17] = (float)(W * 1.15);
    s[18] = (float)(-0.15 * H); s[19] = (float)(1.15 * H);
}

__global__ void __launch_bounds__(F3D_THREADS) filter3d_min_kernel(int P, int V, const float* __restrict__ means3D,
                                                                   const float* __restrict__ viewmatrices,
                                                                   const float* __restrict__ intrinsics,
                                                                   float* __restrict__ out, uint32_t* __restrict__ dmax) {
    __shared__ float sCam[F3D_CHUNK * F3D_CAMF];
    __shared__ uint32_t sMax;
    const int i = blockIdx.x * F3D_THREADS + threadIdx.x;
    float px = 0.f, py = 0.f, pz = 0.f;
    if (i < P) { px = means3D[3 * (size_t)i]; py = means3D[3 * (size_t)i + 1]; pz = means3D[3 * (size_t)i + 2]; }
    if (threadIdx.x == 0) sMax = 0u;
    float d = __int_as_float(0x7f800000);              // +inf: no valid camera yet
    for (int c0 = 0; c0 < V; c0 += F3D_CHUNK) {
        const int n = min(F3D_CHUNK, V - c0);
        __syncthreads();                               // the previous chunk is consumed
        for (int c = threadIdx.x; c < n; c += F3D_THREADS)
            stage_camera(sCam + c * F3D_CAMF, viewmatrices + 16 * (size_t)(c0 + c), intrinsics + 6 * (size_t)(c0 + c));
        __syncthreads();
        if (i < P) {
            for (int c = 0; c < n; ++c) {
                const float* m = sCam + c * F3D_CAMF;
                const float z = xform_row_(m, 2, px, py, pz);    // project_kernel's near-cull depth, bit for bit
                const float tx = xform_row_(m, 0, px, py, pz), ty = xform_row_(m, 1, px, py, pz);
                const float u = __fadd_rn(__fmul_rn(__fdiv_rn(tx, z), m[3]), m[11]);
                const float v = __fadd_rn(__fmul_rn(__fdiv_rn(ty, z), m[7]), m[15]);
                const bool valid = z > 0.2f && u >= m[16] && u <= m[17] && v >= m[18] && v <= m[19];
                if (valid) d = fminf(d, z);
            }
        }
    }
    const bool seen = i < P && d != __int_as_float(0x7f800000);
    if (i < P) out[i] = seen ? d : -1.0f;
    uint32_t b = seen ? __float_as_uint(d) : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) b = max(b, __shfl_xor_sync(0xffffffffu, b, o));
    if ((threadIdx.x & 31) == 0 && b) atomicMax(&sMax, b);
    __syncthreads();
    if (threadIdx.x == 0 && sMax) atomicMax(dmax, sMax);
}

__global__ void __launch_bounds__(256) filter3d_finish_kernel(int P, float F, float* __restrict__ f,
                                                              const uint32_t* __restrict__ dmax) {
    const float dm = __uint_as_float(*dmax);           // +0 when no Gaussian is seen: f = 0, the unfiltered model
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
        const float d = f[i];
        f[i] = __fmul_rn(__fdiv_rn(d < 0.0f ? dm : d, F), 0.44721359549995793928f);   // fp32 sqrt(0.2)
    }
}

size_t filter3d_tmp_bytes(int) { return 256; }

int launch_filter3d(int P, int V, const float* means3D, const float* viewmatrices, const float* intrinsics, float F,
                    float* out, void* tmp, size_t tmp_bytes, int sms, cudaStream_t stream) {
    if (P < 0 || !(F > 0.0f && F <= 3.402823466e38f)) return R3DG_ERR_BAD_ARG;
    if (P == 0) return 0;
    if (V < 1 || !means3D || !viewmatrices || !intrinsics || !out || !tmp || tmp_bytes < filter3d_tmp_bytes(P))
        return R3DG_ERR_BAD_ARG;
    uint32_t* dmax = (uint32_t*)tmp;
    R3DG_CUDA_TRY(cudaMemsetAsync(dmax, 0, sizeof(uint32_t), stream));
    filter3d_min_kernel<<<(P + F3D_THREADS - 1) / F3D_THREADS, F3D_THREADS, 0, stream>>>(P, V, means3D, viewmatrices,
                                                                                      intrinsics, out, dmax);
    R3DG_CUDA_TRY(cudaGetLastError());
    const int blocks = min((P + 255) / 256, 8 * sms);
    filter3d_finish_kernel<<<blocks, 256, 0, stream>>>(P, F, out, dmax);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
