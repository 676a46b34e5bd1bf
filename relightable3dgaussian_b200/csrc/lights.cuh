// Point and directional lights (include/r3dg_b200.h, LIGHTS): the light geometry shared by the shadow trace
// (lights_trace.cu) and the shading kernels (lights.cu).  Both must see the same direction l for a (Gaussian, light)
// pair, but the two files are compiled with different contraction settings (the trace with the bake's, the shading
// with the shading step's -fmad=false), so l is rounded op by op with explicit intrinsics.  The spot and rect lights
// (SHAPED LIGHTS) share their sample hash and sample points the same way.
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

// ---- spot and rect lights (SHAPED LIGHTS) ----
#define LIGHT_SPOT 2
#define LIGHT_RECT 3

// lowbias32 (C. Wellons' integer hash): the sample hash of a rect light
__host__ __device__ __forceinline__ uint32_t lowbias32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

// the per-(set, Gaussian row, light) hash state; sample q's jitter is lowbias32(h ^ 2q) and lowbias32(h ^ (2q + 1))
__device__ __forceinline__ uint32_t rect_hash(uint32_t seed, uint32_t g, uint32_t j) {
    return lowbias32(lowbias32(lowbias32(seed) ^ g) ^ j);
}

__device__ __forceinline__ float hash_unit(uint32_t h) { return (float)(h >> 8) * (1.0f / 16777216.0f); }   // exact

// Stratified sample q = i M + k of the rect (pos, u, v): s = -1 + (2i + 2 xi1) / M (stratum i of width 2/M, jittered
// over all of it), t likewise, and y = (pos + s u) + t v, rounded op by op (2 xi and 2i + 2 xi are exact)
__device__ __forceinline__ void rect_sample(const float* pos, const float* u, const float* v, int M, uint32_t h, int q,
                                            float& s, float& t, float* y) {
    const int i = q / M, k = q - (q / M) * M;
    const float xi1 = hash_unit(lowbias32(h ^ (2u * (uint32_t)q))), xi2 = hash_unit(lowbias32(h ^ (2u * (uint32_t)q + 1u)));
    const float fm = (float)M;
    s = add_(-1.0f, div_(add_((float)(2 * i), mul_(2.0f, xi1)), fm));
    t = add_(-1.0f, div_(add_((float)(2 * k), mul_(2.0f, xi2)), fm));
#pragma unroll
    for (int c = 0; c < 3; ++c) y[c] = add_(add_(pos[c], mul_(s, u[c])), mul_(t, v[c]));
}

// rays of a shaped light set (R of the header), -1 for a bad set: K out of range, a kind other than 2 or 3, M out of
// range or R above R3DG_MAX_SHAPED_RAYS
inline int shaped_rays(int K, const int32_t* kind, int M) {
    if (K < 0 || K > R3DG_MAX_LIGHTS || (K > 0 && !kind) || M < 1 || M > R3DG_MAX_RECT_SAMPLES) return -1;
    int R = 0;
    for (int j = 0; j < K; ++j) {
        if (kind[j] != LIGHT_SPOT && kind[j] != LIGHT_RECT) return -1;
        R += kind[j] == LIGHT_SPOT ? 1 : M * M;
    }
    return R > R3DG_MAX_SHAPED_RAYS ? -1 : R;
}

// the host kind array as the kernels' argument: bit j set = light j is a rect
inline uint32_t rect_mask(int K, const int32_t* kind) {
    uint32_t m = 0u;
    for (int j = 0; j < K; ++j) m |= (uint32_t)(kind[j] == LIGHT_RECT) << j;
    return m;
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

// ---- per-pixel lights (PIXEL LIGHTS) ----
// The set of a per-pixel light call: its R and the kernels' light masks
struct PixelLightSet {
    int R;
    bool shaped;                     // spots and rects (else directional and point lights)
    uint32_t dir_mask, point_mask, rect_mask;
};

// The checks the trace and the shading share, before any launch: 0 and the set, or the call's R3DG_ERR_* code.
// `shading`: also the light fields only the shading reads.
inline int pixel_light_set(const r3dg_pixel_light_args* a, bool shading, PixelLightSet& ls) {
    if (!a || a->V < 1 || a->V > R3DG_MAX_VIEWS || a->H < 1 || a->W < 1 || a->M < 1 || a->M > R3DG_MAX_RECT_SAMPLES)
        return R3DG_ERR_BAD_ARG;
    if (a->K < 0 || a->K > R3DG_MAX_LIGHTS || (a->K > 0 && !a->kind)) return R3DG_ERR_BAD_ARG;
    ls.shaped = a->K > 0 && (a->kind[0] == LIGHT_SPOT || a->kind[0] == LIGHT_RECT);
    ls.R = ls.shaped ? shaped_rays(a->K, a->kind, a->M) : (lights_valid(a->K, a->kind) ? a->K : -1);
    if (ls.R < 0) return R3DG_ERR_BAD_ARG;                 // a kind outside 0..3, mixed families, or R too large
    const uint32_t all = a->K == 32 ? 0xffffffffu : (1u << a->K) - 1u;
    ls.rect_mask = ls.shaped ? rect_mask(a->K, a->kind) : 0u;
    ls.point_mask = ls.shaped ? 0u : point_mask(a->K, a->kind);
    ls.dir_mask = ls.shaped ? 0u : all & ~ls.point_mask;
    if (!a->points) return R3DG_ERR_BAD_ARG;
    if (a->K > 0 && (!a->pos || (ls.rect_mask && (!a->a || !a->b)))) return R3DG_ERR_BAD_ARG;
    if (shading && a->K > 0 && (!a->color || (ls.shaped && (!a->a || ((all & ~ls.rect_mask) && !a->cone)))))
        return R3DG_ERR_BAD_ARG;
    if ((long long)a->V * a->H * a->W > 0x7fffffffLL) return R3DG_ERR_UNSUPPORTED;
    return 0;
}

}  // namespace r3dg
