// Real SH basis up to degree 3 and the rasterizer's SH -> RGB (forward.cu:20-71), shared by the projection
// (projection.cu) and the radiance bake (indirect.cu), so a bake colour is what the rasterizer would show from the
// ray origin.
#pragma once
#include "common.cuh"

namespace r3dg {

__constant__ float SH_C2c[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                -1.0925484305920792f, 0.5462742152960396f};
__constant__ float SH_C3c[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                                -0.5900435899266435f};

// w[k] = Y_k(x, y, z) for k < (deg + 1)^2 (entries beyond are not written); (x, y, z) is a unit vector.
__device__ __forceinline__ void sh_basis(int deg, float x, float y, float z, float (&w)[16]) {
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    w[0] = 0.28209479177387814f;
    if (deg > 0) {
        w[1] = -(0.4886025119029199f * y); w[2] = 0.4886025119029199f * z; w[3] = -(0.4886025119029199f * x);
        if (deg > 1) {
            w[4] = SH_C2c[0] * xy; w[5] = SH_C2c[1] * yz; w[6] = SH_C2c[2] * ((zz + zz) - xx - yy);
            w[7] = SH_C2c[3] * xz; w[8] = SH_C2c[4] * (xx - yy);
            if (deg > 2) {
                w[9] = SH_C3c[0] * y * fmaf(xx, 3.0f, -yy);
                w[10] = SH_C3c[1] * xy * z;
                w[11] = SH_C3c[2] * y * (fmaf(zz, 4.0f, -xx) - yy);
                w[12] = SH_C3c[3] * z * fmaf(yy, -3.0f, fmaf(xx, -3.0f, zz + zz));
                w[13] = SH_C3c[4] * x * (fmaf(zz, 4.0f, -xx) - yy);
                w[14] = SH_C3c[5] * z * (xx - yy);
                w[15] = SH_C3c[6] * x * fmaf(yy, -3.0f, xx);
            }
        }
    }
}

// SH -> RGB (forward.cu:20-71).  sh rows are [M][3] floats.
// `sh` points at coefficient 0 / channel 0 of this Gaussian; consecutive floats of its [M][3] row
// are `stride` apart (1 in global memory, PROJ_THREADS+1 in the transposed shared-memory slab);
// stride 0 = contiguous, 16-byte aligned row read with vector loads (row-major slab of the bulk-copy path).
__device__ __forceinline__ void sh_to_rgb(int deg, float px, float py, float pz,
                                          const float* __restrict__ campos,
                                          const float* __restrict__ sh, int stride, float* rgb,
                                          unsigned& clamped_bits) {
    const float dx = px - campos[0], dy = py - campos[1], dz = pz - campos[2];
    const float len = sqrt_(dot3_(dx, dx, dy, dy, dz, dz));
    const float x = div_(dx, len), y = div_(dy, len), z = div_(dz, len);
    float w[16];
    sh_basis(deg, x, y, z, w);
    const int n = (deg + 1) * (deg + 1);
    float res[3];
    if (stride == 0) {
        // row-major slab row (TMA bulk copy path): 16-byte vector reads, each consumed immediately.  Element
        // i = 3k + c adds w[k] * sh[k][c] to channel c in the same k order as below (same fma chain per channel).
        const float4* __restrict__ r4 = reinterpret_cast<const float4*>(sh);
        res[0] = res[1] = res[2] = 0.0f;
#pragma unroll
        for (int i4 = 0; i4 < 12; ++i4) {
            if (4 * i4 < 3 * n) {
                const float4 v4 = r4[i4];
                const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int i = 4 * i4 + e, k = i / 3, c = i - 3 * k;
                    if (k == 0) res[c] = w[0] * v[e];
                    else if (k < n) res[c] = fmaf(w[k], v[e], res[c]);
                }
            }
        }
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) res[c] = w[0] * sh[c * stride];
#pragma unroll
        for (int k = 1; k < 16; ++k) {
            if (k < n) {
#pragma unroll
                for (int c = 0; c < 3; ++c) res[c] = fmaf(w[k], sh[(3 * k + c) * stride], res[c]);
            }
        }
    }
    clamped_bits = 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        res[c] += 0.5f;
        if (res[c] < 0.0f) clamped_bits |= 1u << c;
        rgb[c] = fmaxf(res[c], 0.0f);
    }
}

}  // namespace r3dg
