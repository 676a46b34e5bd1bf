// The per-light code of the LIGHTS and SHAPED LIGHTS shading terms (include/r3dg_b200.h), shared by the per-Gaussian
// kernels (lights.cu) and the per-pixel ones (pixel_lights.cu): the lights in shared memory, each light's (or rect
// sample's) direction, weight and n . l, and the normalisation backwards.  Both files are compiled with -fmad=false,
// so a pixel taken as a row gets the row path's bits.
#pragma once
#include "brdf.cuh"
#include "lights.cuh"

namespace r3dg {

#define LS_THREADS 128
#define LS_WARPS (LS_THREADS / 32)

// The K lights in shared memory
struct LightSmem { float vec[3 * R3DG_MAX_LIGHTS], color[3 * R3DG_MAX_LIGHTS]; };

// A: an argument record with K and the light fields vec and color
template <class A>
__device__ __forceinline__ void stage_lights(const A& a, LightSmem& s) {
    for (int i = threadIdx.x; i < 3 * a.K; i += LS_THREADS) { s.vec[i] = a.vec[i]; s.color[i] = a.color[i]; }
    __syncthreads();
}

// The light's term before GGX: l, E and max(n . l, 0) (ndr: n . l before the clamp)
struct LightTerm { LightDir d; float E[3], r2c, ndr, ndi; };

__device__ __forceinline__ LightTerm light_term(int kind, const LightSmem& s, int j, const GaussianOperands& o, const float* m) {
    LightTerm t;
    t.d = light_dir(kind, s.vec + 3 * j, m[0], m[1], m[2]);
    t.r2c = fmaxf(t.d.r2, LIGHT_R2_MIN);
#pragma unroll
    for (int c = 0; c < 3; ++c) t.E[c] = kind == 0 ? s.color[3 * j + c] : s.color[3 * j + c] / t.r2c;
    t.ndr = o.n[0] * t.d.l[0] + o.n[1] * t.d.l[1] + o.n[2] * t.d.l[2];        // the shading step's n . w
    t.ndi = fmaxf(t.ndr, 0.f);
    return t;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// dL/dw of l = w / max(|w|, eps) (F.normalize: the norm's gradient is cut below eps)
__device__ __forceinline__ void normalize_backward(const LightDir& d, const float* dl, float* dw) {
    const float den = fmaxf(d.rn, LIGHT_EPS);
    const float ldl = d.rn >= LIGHT_EPS ? d.l[0] * dl[0] + d.l[1] * dl[1] + d.l[2] * dl[2] : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) dw[c] = (dl[c] - d.l[c] * ldl) / den;
}

// dL/dx of n = x / max(|x|, eps) for the cotangent dn (F.normalize: the norm's gradient is cut below eps)
__device__ __forceinline__ void normalize3_backward(const float* x, const float* dn, float* dx) {
    const float xn = sqrtf(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]), den = fmaxf(xn, LIGHT_EPS);
    const float ndn = xn >= LIGHT_EPS ? (x[0] * dn[0] + x[1] * dn[1] + x[2] * dn[2]) / den : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) dx[c] = (dn[c] - x[c] / den * ndn) / den;
}

// ==== spot and rect lights (SHAPED LIGHTS; DESIGN.md §4.28) ==================================================
// The backward accumulates each light's gradient over its samples as 16 intermediate values per light (SL_SLOTS);
// shaped_reduce_kernel (lights.cu) applies the light-level chain rule once (axis normalisation, u x v, n_e and A).
#define SL_SLOTS 16
// slots: 0-2 dL/dpos (= dL/dy summed), 3-5 dL/du through y (rect) or dL/da^ (spot), 6-8 dL/dv through y (rect) or
// dL/dcos_inner, dL/dcos_outer (spot, 6 and 7), 9-11 dL/dcolor, 12-14 dL/dn_e and 15 dL/dA (rect)

struct ShapedSmem {
    float L[9 * R3DG_MAX_LIGHTS];              // pos, a (axis or u), b (v)
    float color[3 * R3DG_MAX_LIGHTS];
    float dir[3 * R3DG_MAX_LIGHTS];            // rect: n_e;  spot: a^
    float sc[R3DG_MAX_LIGHTS];                 // rect: A;  spot: max(cos_inner - cos_outer, 1e-6)
    float co[R3DG_MAX_LIGHTS];                 // spot: cos_outer
    float live[R3DG_MAX_LIGHTS];               // spot: 1 where cos_inner - cos_outer >= 1e-6 (the clamp passes its gradient)
};

// A: an argument record with K and the light fields pos, a, b, color and cone
template <class A>
__device__ __forceinline__ void stage_shaped(const A& a, uint32_t rect_mask, ShapedSmem& s) {
    for (int i = threadIdx.x; i < 3 * a.K; i += LS_THREADS) {
        const int j = i / 3, c = i - 3 * j;
        const bool rect = (rect_mask >> j) & 1;
        s.L[9 * j + c] = a.pos[i];
        s.L[9 * j + 3 + c] = a.a[i];
        s.L[9 * j + 6 + c] = rect ? a.b[i] : 0.f;
        s.color[i] = a.color[i];
    }
    __syncthreads();
    for (int j = threadIdx.x; j < a.K; j += LS_THREADS) {
        const float* u = s.L + 9 * j + 3;
        if ((rect_mask >> j) & 1) {
            const float* v = s.L + 9 * j + 6;
            const float c0 = u[1] * v[2] - u[2] * v[1], c1 = u[2] * v[0] - u[0] * v[2], c2 = u[0] * v[1] - u[1] * v[0];
            const float cn = sqrtf(c0 * c0 + c1 * c1 + c2 * c2), den = fmaxf(cn, LIGHT_EPS);
            s.dir[3 * j] = c0 / den; s.dir[3 * j + 1] = c1 / den; s.dir[3 * j + 2] = c2 / den;
            s.sc[j] = 4.0f * cn;
            s.co[j] = 0.f; s.live[j] = 0.f;
        } else {
            const float an = fmaxf(sqrtf(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]), LIGHT_EPS);
            s.dir[3 * j] = u[0] / an; s.dir[3 * j + 1] = u[1] / an; s.dir[3 * j + 2] = u[2] / an;
            const float ci = a.cone[2 * j], co = a.cone[2 * j + 1];
            s.sc[j] = fmaxf(ci - co, 1e-6f);
            s.co[j] = co; s.live[j] = ci - co >= 1e-6f ? 1.f : 0.f;
        }
    }
    __syncthreads();
}

// One ray of a shaped light at the Gaussian: l, w and the scalar weight of E = color * wgt, with its operands
struct ShapedTerm {
    LightDir d;
    float st[2];          // rect: (s, t)
    float r2c, ce_r, xr, x, wgt, ndr, ndi;
};

__device__ __forceinline__ void shaped_term(bool rect, const ShapedSmem& s, int j, int M, uint32_t h, int q,
                                            const GaussianOperands& o, const float* m, ShapedTerm& t) {
    const float* L = s.L + 9 * j;
    const float* dir = s.dir + 3 * j;
    float y[3];
    if (rect) rect_sample(L, L + 3, L + 6, M, h, q, t.st[0], t.st[1], y);
    else { y[0] = L[0]; y[1] = L[1]; y[2] = L[2]; t.st[0] = t.st[1] = 0.f; }
    t.d = light_dir(1, y, m[0], m[1], m[2]);
    t.r2c = fmaxf(t.d.r2, LIGHT_R2_MIN);
    const float dl = dir[0] * t.d.l[0] + dir[1] * t.d.l[1] + dir[2] * t.d.l[2];
    if (rect) {
        t.ce_r = -dl;
        t.xr = t.x = 0.f;
        t.wgt = s.sc[j] * fmaxf(t.ce_r, 0.f) / ((float)(M * M) * t.r2c);
    } else {
        t.ce_r = 0.f;
        t.xr = (-dl - s.co[j]) / s.sc[j];
        t.x = fminf(fmaxf(t.xr, 0.f), 1.f);
        t.wgt = t.x * t.x * (3.0f - 2.0f * t.x) / t.r2c;
    }
    t.ndr = o.n[0] * t.d.l[0] + o.n[1] * t.d.l[1] + o.n[2] * t.d.l[2];
    t.ndi = fmaxf(t.ndr, 0.f);
}

}  // namespace r3dg
