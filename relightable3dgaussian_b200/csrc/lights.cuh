// Point and directional lights (include/r3dg_b200.h, LIGHTS): the light geometry shared by the shadow trace
// (lights_trace.cu) and the shading kernels (lights.cu).  Both must see the same direction l for a (Gaussian, light)
// pair, but the two files are compiled with different contraction settings (the trace with the bake's, the shading
// with the shading step's -fmad=false), so l is rounded op by op with explicit intrinsics.
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace r3dg {

#define LIGHT_R2_MIN 1e-8f          // floor of a point light's squared distance
#define LIGHT_EPS 1e-12f            // F.normalize eps
#define LIGHT_ORIGIN_OFFSET 0.05f   // shadow-ray origin m + 0.05 l (the visibility bake's offset)

// w = vec (directional) or vec - m (point); r2 = |w|^2 = (w0 w0 + w1 w1) + w2 w2; rn = sqrt(r2); l = w / max(rn, eps)
struct LightDir { float w[3], r2, rn, l[3]; };

__device__ __forceinline__ LightDir light_dir(int kind, const float* vec, float mx, float my, float mz) {
    LightDir d;
    d.w[0] = vec[0]; d.w[1] = vec[1]; d.w[2] = vec[2];
    if (kind != 0) { d.w[0] = sub_(d.w[0], mx); d.w[1] = sub_(d.w[1], my); d.w[2] = sub_(d.w[2], mz); }
    d.r2 = add_(add_(mul_(d.w[0], d.w[0]), mul_(d.w[1], d.w[1])), mul_(d.w[2], d.w[2]));
    d.rn = sqrt_(d.r2);
    const float den = fmaxf(d.rn, LIGHT_EPS);
    d.l[0] = div_(d.w[0], den); d.l[1] = div_(d.w[1], den); d.l[2] = div_(d.w[2], den);
    return d;
}

// host-side checks shared by both operations: K in range and every kind 0 or 1
inline bool lights_valid(int K, const int32_t* kind) {
    if (K < 0 || K > R3DG_MAX_LIGHTS || (K > 0 && !kind)) return false;
    for (int j = 0; j < K; ++j)
        if (kind[j] != 0 && kind[j] != 1) return false;
    return true;
}

// the host kind array as the kernels' argument: bit j set = light j is a point light
inline uint32_t point_mask(int K, const int32_t* kind) {
    uint32_t m = 0u;
    for (int j = 0; j < K; ++j) m |= (uint32_t)(kind[j] == 1) << j;
    return m;
}

}  // namespace r3dg
