// §8(f)2: the host-side epilogue the reference wraps around the rasterizer
// (gaussian_renderer/neilf.py:135-137, render.py:106-108):
//     rendered_feature = rendered_feature / rendered_opacity.clamp_min(1e-5) * (num_contrib > 0)
// In PyTorch this is 3 elementwise kernels forward over [S,H,W] (plus ~6 in autograd's backward, which
// also keeps two [S,H,W] intermediates alive).  Here: ONE pass forward, ONE pass backward, both
// HBM-bound (forward reads S+2 planes and writes S; backward reads 2S+2 and writes S+1), optional —
// the reference's unmodified render functions keep using PyTorch; `rasterizer.unpremultiply` opts in.
#include "common.cuh"
#include "kernels.h"

namespace r3dg {

__global__ void __launch_bounds__(256) unpremultiply_fwd_kernel(int S, long long HW, const float* __restrict__ feature,
                                                                const float* __restrict__ opacity,
                                                                const int32_t* __restrict__ n_contrib, float* __restrict__ out) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
        const float den = fmaxf(opacity[p], 1e-5f);
        const float m = n_contrib[p] > 0 ? 1.0f : 0.0f;
        for (int c = 0; c < S; ++c) out[c * HW + p] = mul_(div_(feature[c * HW + p], den), m);   // torch op order: (f / den) * mask
    }
}

// d_feature = g * m / den;  d_opacity = -(sum_c g_c * m * f_c) / den^2 where opacity >= 1e-5 (clamp_min passes its gradient there)
__global__ void __launch_bounds__(256) unpremultiply_bwd_kernel(int S, long long HW, const float* __restrict__ feature,
                                                                const float* __restrict__ opacity,
                                                                const int32_t* __restrict__ n_contrib, const float* __restrict__ g,
                                                                float* __restrict__ d_feature, float* __restrict__ d_opacity) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
        const float o = opacity[p];
        const float den = fmaxf(o, 1e-5f);
        const float m = n_contrib[p] > 0 ? 1.0f : 0.0f;
        const float inv = 1.0f / den;
        float acc = 0.0f;
        for (int c = 0; c < S; ++c) {
            const float gm = g[c * HW + p] * m;
            d_feature[c * HW + p] = gm * inv;
            acc += gm * feature[c * HW + p];
        }
        d_opacity[p] = o >= 1e-5f ? -acc * inv * inv : 0.0f;
    }
}

static int grid_for(long long n, int num_sms) {
    const long long want = (n + 255) / 256;
    return (int)(want < (long long)num_sms * 16 ? want : (long long)num_sms * 16);
}

int launch_unpremultiply_forward(int S, long long HW, const float* feature, const float* opacity, const int32_t* n_contrib,
                                 float* out, int num_sms, cudaStream_t stream) {
    if (S <= 0 || HW <= 0) return 0;
    unpremultiply_fwd_kernel<<<grid_for(HW, num_sms), 256, 0, stream>>>(S, HW, feature, opacity, n_contrib, out);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_unpremultiply_backward(int S, long long HW, const float* feature, const float* opacity, const int32_t* n_contrib,
                                  const float* g, float* d_feature, float* d_opacity, int num_sms, cudaStream_t stream) {
    if (HW <= 0) return 0;
    unpremultiply_bwd_kernel<<<grid_for(HW, num_sms), 256, 0, stream>>>(S, HW, feature, opacity, n_contrib, g, d_feature, d_opacity);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}


// ---------------------------------------------------------------------------------------------------------------
// §8(f)2, first half: the feature pack the reference's render functions build in front of the rasterizer
// (gaussian_renderer/neilf.py:110-126, render.py:88-93):
//     xyz_homo = cat([means3D, 1]);  depths = (xyz_homo @ world_view_transform)[:, 2:3];  depths2 = depths.square()
//     features = cat([depths, depths2, t_0, t_1, ...], dim=-1)
// = ones_like + cat + a [P,4]x[4,4] sgemm + slice + square + an 8-tensor cat forward, and the matching slice / matmul
// chain in autograd's backward (whose sliced cotangents are non-contiguous and get copied again).  Here: ONE pass
// forward (reads the sources once, writes [P,S] once) and ONE backward (reads dL/dfeatures once, writes every source
// gradient contiguous, plus dL/dmeans3D through the two depth channels).  Optional operator: the reference's own files
// keep their PyTorch expressions.
// ---------------------------------------------------------------------------------------------------------------
struct PackTable {
    int P, S, num, depth;                 // depth: 2 leading channels {z, z^2} from means3D / viewmatrix, or 0
    const float* means3D;
    const float* view;                    // [4,4] stored transposed (row-vector convention): z = x*v[2] + y*v[6] + z*v[10] + v[14]
    r3dg_pack_src src[R3DG_PACK_MAX];
    int offset[R3DG_PACK_MAX];            // first output channel of source k
};

__device__ __forceinline__ float view_depth(const float* __restrict__ v, const float* __restrict__ m) {
    // (xyz_homo @ V)[2] as the sgemm accumulates it: k = 0..3 in order
    return fmaf(1.0f, v[14], fmaf(m[2], v[10], fmaf(m[1], v[6], m[0] * v[2])));
}

__global__ void __launch_bounds__(256) pack_features_fwd_kernel(const PackTable t, float* __restrict__ out) {
    const long long total = (long long)t.P * t.S;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long p = i / t.S;
        const int c = (int)(i - p * t.S);
        float v = 0.0f;
        if (c < t.depth) {
            const float z = view_depth(t.view, t.means3D + 3 * p);
            v = c == 0 ? z : z * z;
        } else {
            int k = 0;
            while (k + 1 < t.num && c >= t.offset[k + 1]) ++k;
            v = t.src[k].ptr[p * t.src[k].width + (c - t.offset[k])];
        }
        out[i] = v;
    }
}

// one thread per (Gaussian, source): copies that source's slice of the cotangent row; source index == num means the
// depth channels -> dL/dmeans3D = (g_z + 2 z g_z2) * V[:3, 2]
__global__ void __launch_bounds__(256) pack_features_bwd_kernel(const PackTable t, const float* __restrict__ g,
                                                                float* __restrict__ d_means3D) {
    const long long total = (long long)t.P * t.S;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long p = i / t.S;
        const int c = (int)(i - p * t.S);
        const float gv = g[i];
        if (c < t.depth) {
            if (c == 0 && d_means3D) {
                const float z = view_depth(t.view, t.means3D + 3 * p);
                const float s = gv + 2.0f * z * g[i + 1];
                d_means3D[3 * p] = s * t.view[2]; d_means3D[3 * p + 1] = s * t.view[6]; d_means3D[3 * p + 2] = s * t.view[10];
            }
        } else {
            int k = 0;
            while (k + 1 < t.num && c >= t.offset[k + 1]) ++k;
            float* dst = const_cast<float*>(t.src[k].ptr);
            if (dst) dst[p * t.src[k].width + (c - t.offset[k])] = gv;
        }
    }
}

// dL/dviewmatrix of the depth channels, one partial sum per CTA of 256 Gaussians: column j of the stored matrix
// (elements 4j + 2) gets sum_g (g_z + 2 z g_z2) [m_g,1]_j, every other element 0.  Fixed order: a butterfly per warp,
// then the 8 warps in order.  work: [16][gridDim.x], one column per CTA.
__global__ void __launch_bounds__(256) pack_view_grad_kernel(const PackTable t, const float* __restrict__ g,
                                                             float* __restrict__ work) {
    __shared__ float part[4][8];
    const long long p = (long long)blockIdx.x * 256 + threadIdx.x;
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    if (p < t.P) {
        const float* m = t.means3D + 3 * p;
        const float z = view_depth(t.view, m);
        const float s = g[p * t.S] + 2.0f * z * g[p * t.S + 1];
        c[0] = s * m[0]; c[1] = s * m[1]; c[2] = s * m[2]; c[3] = s;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c[j] += __shfl_xor_sync(0xffffffffu, c[j], o);
        if ((threadIdx.x & 31) == 0) part[j][threadIdx.x >> 5] = c[j];
    }
    __syncthreads();
    if (threadIdx.x < 16) {
        const int k = threadIdx.x;
        float s = 0.f;
        if ((k & 3) == 2) {
            s = part[k >> 2][0];
#pragma unroll
            for (int w = 1; w < 8; ++w) s += part[k >> 2][w];
        }
        work[(size_t)k * gridDim.x + blockIdx.x] = s;
    }
}

static int make_table(PackTable& t, int P, int S, const float* means3D, const float* view, int num, const r3dg_pack_src* srcs,
                      bool need_ptr) {
    if (P < 0 || S <= 0 || num < 0 || num > R3DG_PACK_MAX) return R3DG_ERR_BAD_ARG;
    t.P = P; t.S = S; t.num = num; t.depth = (means3D && view) ? 2 : 0; t.means3D = means3D; t.view = view;
    int off = t.depth;
    for (int k = 0; k < num; ++k) {
        if (srcs[k].width <= 0 || (need_ptr && !srcs[k].ptr)) return R3DG_ERR_BAD_ARG;
        t.src[k] = srcs[k]; t.offset[k] = off; off += srcs[k].width;
    }
    return off == S ? 0 : R3DG_ERR_BAD_ARG;
}

int launch_pack_features_forward(int P, int S, const float* means3D, const float* view, int num, const r3dg_pack_src* srcs,
                                 float* out, int num_sms, cudaStream_t stream) {
    PackTable t;
    const int rc = make_table(t, P, S, means3D, view, num, srcs, true);
    if (rc != 0 || P == 0) return rc;
    pack_features_fwd_kernel<<<grid_for((long long)P * S, num_sms), 256, 0, stream>>>(t, out);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_pack_features_backward(int P, int S, const float* means3D, const float* view, const float* g, int num,
                                  const r3dg_pack_src* dsts, float* d_means3D, float* d_view, void* work, size_t work_bytes,
                                  int num_sms, cudaStream_t stream) {
    PackTable t;
    const int rc = make_table(t, P, S, means3D, view, num, dsts, false);
    if (rc != 0) return rc;
    const int nblk = (P + 255) / 256;
    if (d_view && (t.depth == 0 || !work || work_bytes < r3dg_raster_cam_grad_bytes(P, 1))) return R3DG_ERR_BAD_ARG;
    static_assert(16 * 2 <= kCamGradFloats, "the pack's [16][P / 256] partials fit in r3dg_raster_cam_grad_bytes(P, 1)");
    if (P == 0) {
        if (d_view) R3DG_CUDA_TRY(cudaMemsetAsync(d_view, 0, 16 * sizeof(float), stream));
        return 0;
    }
    pack_features_bwd_kernel<<<grid_for((long long)P * S, num_sms), 256, 0, stream>>>(t, g, d_means3D);
    R3DG_CUDA_TRY(cudaGetLastError());
    if (d_view) {
        pack_view_grad_kernel<<<nblk, 256, 0, stream>>>(t, g, (float*)work);
        R3DG_CUDA_TRY(cudaGetLastError());
        const CamGradOut o = {{d_view, nullptr, nullptr}, {16, 0, 0}};
        return launch_cam_grad_sum((const float*)work, nblk, 1, o, stream);
    }
    return 0;
}

}  // namespace r3dg
