// Per-pixel point, directional, spot and rect lights (include/r3dg_b200.h, PIXEL LIGHTS; DESIGN.md §4.30): the
// LIGHTS and SHAPED LIGHTS shading terms at every valid pixel of the per-pixel shading's G-buffer, with each pixel's
// shadows traced from its own surface point (lights_trace.cu).  Compiled with -fmad=false, as lights.cu.
//
// Design notes
//  * a pixel is a row of lights.cu's kernels: mean = its point, raw normal, viewdir = campos_v - point and row index p
//    (the rect hash); the per-light loop bodies are lights.cu's, with the same helpers (lights_eval.cuh), sums in
//    light then sample order, so every forward output and the per-pixel gradients equal the row path's bit for bit.
//    The loop bodies are copies: as shared functions they changed the scheduling of lights.cu's four kernels.
//  * one thread per (view, pixel), CTAs striding over V H W; the grid depends on V H W only, and the light gradients
//    are reduced as lights.cu reduces them (warp butterfly, warps in order, CTA partials summed in block order by
//    lights.cu's reduce kernels), so every output is bitwise reproducible without float atomics.
//  * masked pixels write zeros and add zeros to the light gradients; a warp with no valid pixel skips its light work.
#include "kernels.h"
#include "lights_eval.cuh"

namespace r3dg {

#define PL_MAX_BLOCKS 2048               // the CTA count of a large call (the grid depends on V H W only)

static int pixel_light_blocks(long long pixels) {
    const long long b = (pixels + LS_THREADS - 1) / LS_THREADS;
    return (int)(b < PL_MAX_BLOCKS ? b : PL_MAX_BLOCKS);
}

// The LIGHTS fields of the call, for stage_lights
struct PointLightFields {
    int K;
    const float *vec, *color;
};

// The operands of pixel q of view v as a row: material, raw normal, view operands of campos_v - point, and the point m
__device__ __forceinline__ void load_pixel_row(const r3dg_pixel_light_args& a, size_t HW, int v, size_t q, GaussianOperands& o,
                                               float* m) {
    float vd[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const size_t k = (3 * (size_t)v + c) * HW + q;
        o.base[c] = a.base_color[k];
        o.n[c] = a.normal[k];
        m[c] = a.points[k];
        vd[c] = a.campos[3 * v + c] - m[c];
    }
    o.rough = a.roughness[(size_t)v * HW + q];
    roughness_operands(o);
    view_operands(o.n, vd, o.V, o.vnorm, o.Ns);
}

// ---- directional and point lights: lights_fwd_kernel's and lights_bwd_kernel's per-light code ----------------
__global__ void __launch_bounds__(LS_THREADS) pixel_lights_fwd_kernel(const r3dg_pixel_light_args a, const uint32_t point_mask) {
    __shared__ LightSmem s;
    stage_lights(PointLightFields{a.K, a.pos, a.color}, s);
    const size_t HW = (size_t)a.H * a.W, total = (size_t)a.V * HW;
    for (size_t vq = (size_t)blockIdx.x * LS_THREADS + threadIdx.x; vq < total; vq += (size_t)gridDim.x * LS_THREADS) {
        const int v = (int)(vq / HW);
        const size_t q = vq - (size_t)v * HW;
        float pbr[3] = {0.f, 0.f, 0.f}, spec[3] = {0.f, 0.f, 0.f}, diff[3] = {0.f, 0.f, 0.f};
        if (!a.mask || a.mask[vq]) {
            GaussianOperands o;
            float m[3];
            load_pixel_row(a, HW, v, q, o, m);
            const float* Tp = a.shadows + (size_t)v * a.K * HW + q;
            for (int j = 0; j < a.K; ++j) {
                const LightTerm t = light_term((point_mask >> j) & 1, s, j, o, m);
                const float T = Tp[(size_t)j * HW];
                GgxEval e;
                eval_ggx<false>(o.V, o.Ns, o, t.d.l[0], t.d.l[1], t.d.l[2], e);
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float tr = t.E[c] * T * t.ndi;
                    const float fd = o.base[c] / PI_F;
                    pbr[c] += (fd + e.fs) * tr; spec[c] += e.fs * tr; diff[c] += tr;
                }
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t k = (3 * (size_t)v + c) * HW + q;
            a.pbr[k] = pbr[c]; a.specular[k] = spec[c]; a.diffuse_light[k] = diff[c];
        }
    }
}

// partial: [gridDim.x][K][6] = (dL/dvec, dL/dcolor) summed over the CTA's pixels, lights_reduce_kernel's layout
__global__ void __launch_bounds__(LS_THREADS) pixel_lights_bwd_kernel(const r3dg_pixel_light_args a, const uint32_t point_mask,
                                                                      float* __restrict__ partial) {
    __shared__ LightSmem s;
    __shared__ float sAcc[LS_WARPS][R3DG_MAX_LIGHTS * 6];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < LS_WARPS * R3DG_MAX_LIGHTS * 6; i += LS_THREADS) (&sAcc[0][0])[i] = 0.f;
    stage_lights(PointLightFields{a.K, a.pos, a.color}, s);
    const size_t HW = (size_t)a.H * a.W, total = (size_t)a.V * HW;
    for (size_t base = (size_t)blockIdx.x * LS_THREADS; base < total; base += (size_t)gridDim.x * LS_THREADS) {
        const size_t vq_raw = base + threadIdx.x;
        const size_t vq = vq_raw < total ? vq_raw : total - 1;     // idle threads shade a copy, contribute zeros
        const bool valid = vq_raw < total && (!a.mask || a.mask[vq]);
        const int v = (int)(vq / HW);
        const size_t q = vq - (size_t)v * HW;
        float dbase_v[3] = {0.f, 0.f, 0.f}, drough_v = 0.f, dV[3] = {0.f, 0.f, 0.f};         // dV: no viewdir gradient here
        if (__any_sync(0xffffffffu, valid)) {
            GaussianOperands o;
            float m[3], gp[3], gs[3], gd[3];
            load_pixel_row(a, HW, v, q, o, m);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const size_t k = (3 * (size_t)v + c) * HW + q;
                gp[c] = valid ? a.dL_dpbr[k] : 0.f;
                gs[c] = valid && a.dL_dspecular ? a.dL_dspecular[k] : 0.f;
                gd[c] = valid && a.dL_ddiffuse_light ? a.dL_ddiffuse_light[k] : 0.f;
            }
            const float* Tp = a.shadows + (size_t)v * a.K * HW + q;
            for (int j = 0; j < a.K; ++j) {
                const int kind = (point_mask >> j) & 1;
                const LightTerm t = light_term(kind, s, j, o, m);
                const float T = Tp[(size_t)j * HW];
                GgxEval e;
                eval_ggx<true>(o.V, o.Ns, o, t.d.l[0], t.d.l[1], t.d.l[2], e);
                float dfs = 0.f, dndi = 0.f, dE[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float tr = t.E[c] * T * t.ndi;
                    const float fd = o.base[c] * INV_PI_F;
                    dbase_v[c] += gp[c] * tr * INV_PI_F;
                    dfs += (gp[c] + gs[c]) * tr;
                    const float dtr = gp[c] * (fd + e.fs) + gs[c] * e.fs + gd[c];
                    dE[c] = dtr * T * t.ndi;
                    dndi += dtr * t.E[c] * T;
                }
                float dLn[3], dl[3];
                ggx_backward<true>(o.V, o.Ns, o, e, dfs, drough_v, dV, dLn);
                LightDir ll;
                ll.l[0] = t.d.l[0]; ll.l[1] = t.d.l[1]; ll.l[2] = t.d.l[2];
                ll.rn = sqrtf(ll.l[0] * ll.l[0] + ll.l[1] * ll.l[1] + ll.l[2] * ll.l[2]);
                const float lden = fmaxf(ll.rn, LIGHT_EPS);
#pragma unroll
                for (int c = 0; c < 3; ++c) ll.l[c] = ll.l[c] / lden;
                normalize_backward(ll, dLn, dl);
                const float dn = t.ndr >= 0.f ? dndi : 0.f;
#pragma unroll
                for (int c = 0; c < 3; ++c) dl[c] += dn * o.n[c];
                float dw[3], dvc[6];
                normalize_backward(t.d, dl, dw);
                if (kind == 0) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) { dvc[c] = dw[c]; dvc[3 + c] = dE[c]; }
                } else {
                    float dr2 = 0.f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) { dvc[3 + c] = dE[c] / t.r2c; dr2 -= dE[c] * t.E[c] / t.r2c; }
                    if (!(t.d.r2 >= LIGHT_R2_MIN)) dr2 = 0.f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) dvc[c] = dw[c] + 2.0f * t.d.w[c] * dr2;
                }
#pragma unroll
                for (int k = 0; k < 6; ++k) {
                    const float x = warp_sum(valid ? dvc[k] : 0.f);
                    if (lane == 0) sAcc[warp][6 * j + k] += x;
                }
            }
        }
        if (vq_raw < total) {
            // the row path's per-Gaussian sum over its one view: 0 + x (so a -0 becomes +0 there too)
#pragma unroll
            for (int c = 0; c < 3; ++c) a.dL_dbase_color[(3 * (size_t)v + c) * HW + q] = valid ? 0.f + dbase_v[c] : 0.f;
            a.dL_droughness[vq] = valid ? 0.f + drough_v : 0.f;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 6 * a.K; i += LS_THREADS) {
        float x = sAcc[0][i];
#pragma unroll
        for (int w = 1; w < LS_WARPS; ++w) x += sAcc[w][i];
        partial[(size_t)blockIdx.x * 6 * a.K + i] = x;
    }
}

// ---- spot and rect lights: shaped_fwd_kernel's and shaped_bwd_kernel's per-sample code -------------------------
__global__ void __launch_bounds__(LS_THREADS) pixel_shaped_fwd_kernel(const r3dg_pixel_light_args a, const uint32_t rect_mask,
                                                                      const int R) {
    __shared__ ShapedSmem s;
    stage_shaped(a, rect_mask, s);
    const size_t HW = (size_t)a.H * a.W, total = (size_t)a.V * HW;
    for (size_t vq = (size_t)blockIdx.x * LS_THREADS + threadIdx.x; vq < total; vq += (size_t)gridDim.x * LS_THREADS) {
        const int v = (int)(vq / HW);
        const size_t q = vq - (size_t)v * HW;
        float pbr[3] = {0.f, 0.f, 0.f}, spec[3] = {0.f, 0.f, 0.f}, diff[3] = {0.f, 0.f, 0.f};
        if (!a.mask || a.mask[vq]) {
            GaussianOperands o;
            float m[3];
            load_pixel_row(a, HW, v, q, o, m);
            const float* Tp = a.shadows + (size_t)v * R * HW + q;
            int col = 0;
            for (int j = 0; j < a.K; ++j) {
                const bool rect = (rect_mask >> j) & 1;
                const int n = rect ? a.M * a.M : 1;
                const uint32_t h = rect_hash(a.seed, (uint32_t)q, (uint32_t)j);
                for (int qq = 0; qq < n; ++qq, ++col) {
                    ShapedTerm t;
                    shaped_term(rect, s, j, a.M, h, qq, o, m, t);
                    const float T = Tp[(size_t)col * HW];
                    GgxEval e;
                    eval_ggx<false>(o.V, o.Ns, o, t.d.l[0], t.d.l[1], t.d.l[2], e);
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float tr = s.color[3 * j + c] * t.wgt * T * t.ndi;
                        const float fd = o.base[c] / PI_F;
                        pbr[c] += (fd + e.fs) * tr; spec[c] += e.fs * tr; diff[c] += tr;
                    }
                }
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t k = (3 * (size_t)v + c) * HW + q;
            a.pbr[k] = pbr[c]; a.specular[k] = spec[c]; a.diffuse_light[k] = diff[c];
        }
    }
}

// partial: [gridDim.x][K][SL_SLOTS], shaped_reduce_kernel's layout
__global__ void __launch_bounds__(LS_THREADS) pixel_shaped_bwd_kernel(const r3dg_pixel_light_args a, const uint32_t rect_mask,
                                                                      const int R, float* __restrict__ partial) {
    __shared__ ShapedSmem s;
    __shared__ float sAcc[LS_WARPS][R3DG_MAX_LIGHTS * SL_SLOTS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < LS_WARPS * R3DG_MAX_LIGHTS * SL_SLOTS; i += LS_THREADS) (&sAcc[0][0])[i] = 0.f;
    stage_shaped(a, rect_mask, s);
    const size_t HW = (size_t)a.H * a.W, total = (size_t)a.V * HW;
    for (size_t base = (size_t)blockIdx.x * LS_THREADS; base < total; base += (size_t)gridDim.x * LS_THREADS) {
        const size_t vq_raw = base + threadIdx.x;
        const size_t vq = vq_raw < total ? vq_raw : total - 1;     // idle threads shade a copy, contribute zeros
        const bool valid = vq_raw < total && (!a.mask || a.mask[vq]);
        const int v = (int)(vq / HW);
        const size_t q = vq - (size_t)v * HW;
        float dbase_v[3] = {0.f, 0.f, 0.f}, drough_v = 0.f, dV[3] = {0.f, 0.f, 0.f};         // dV: no viewdir gradient here
        if (__any_sync(0xffffffffu, valid)) {
            GaussianOperands o;
            float m[3], gp[3], gs[3], gd[3];
            load_pixel_row(a, HW, v, q, o, m);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const size_t k = (3 * (size_t)v + c) * HW + q;
                gp[c] = valid ? a.dL_dpbr[k] : 0.f;
                gs[c] = valid && a.dL_dspecular ? a.dL_dspecular[k] : 0.f;
                gd[c] = valid && a.dL_ddiffuse_light ? a.dL_ddiffuse_light[k] : 0.f;
            }
            const float* Tp = a.shadows + (size_t)v * R * HW + q;
            int col = 0;
            for (int j = 0; j < a.K; ++j) {
                const bool rect = (rect_mask >> j) & 1;
                const int n = rect ? a.M * a.M : 1;
                const uint32_t h = rect_hash(a.seed, (uint32_t)q, (uint32_t)j);
                const float* dir = s.dir + 3 * j;
                float acc[SL_SLOTS];
#pragma unroll
                for (int k = 0; k < SL_SLOTS; ++k) acc[k] = 0.f;
                for (int qq = 0; qq < n; ++qq, ++col) {
                    ShapedTerm t;
                    shaped_term(rect, s, j, a.M, h, qq, o, m, t);
                    const float T = Tp[(size_t)col * HW];
                    GgxEval e;
                    eval_ggx<true>(o.V, o.Ns, o, t.d.l[0], t.d.l[1], t.d.l[2], e);
                    float dfs = 0.f, dndi = 0.f, dwgt = 0.f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float E = s.color[3 * j + c] * t.wgt;
                        const float tr = E * T * t.ndi;
                        const float fd = o.base[c] * INV_PI_F;
                        dbase_v[c] += gp[c] * tr * INV_PI_F;
                        dfs += (gp[c] + gs[c]) * tr;
                        const float dtr = gp[c] * (fd + e.fs) + gs[c] * e.fs + gd[c];
                        const float dE = dtr * T * t.ndi;
                        dndi += dtr * E * T;
                        acc[9 + c] += dE * t.wgt;
                        dwgt += dE * s.color[3 * j + c];
                    }
                    float dLn[3], dl[3];
                    ggx_backward<true>(o.V, o.Ns, o, e, dfs, drough_v, dV, dLn);
                    LightDir ll;
                    ll.l[0] = t.d.l[0]; ll.l[1] = t.d.l[1]; ll.l[2] = t.d.l[2];
                    ll.rn = sqrtf(ll.l[0] * ll.l[0] + ll.l[1] * ll.l[1] + ll.l[2] * ll.l[2]);
                    const float lden = fmaxf(ll.rn, LIGHT_EPS);
#pragma unroll
                    for (int c = 0; c < 3; ++c) ll.l[c] = ll.l[c] / lden;
                    normalize_backward(ll, dLn, dl);
                    const float dn = t.ndr >= 0.f ? dndi : 0.f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) dl[c] += dn * o.n[c];
                    float dr2 = -dwgt * t.wgt / t.r2c;
                    if (rect) {
                        const float k = (float)(a.M * a.M) * t.r2c;
                        const float ce = fmaxf(t.ce_r, 0.f);
                        acc[15] += dwgt * ce / k;
                        const float dce = t.ce_r >= 0.f ? dwgt * s.sc[j] / k : 0.f;
#pragma unroll
                        for (int c = 0; c < 3; ++c) { acc[12 + c] -= dce * t.d.l[c]; dl[c] -= dce * dir[c]; }
                    } else {
                        const float dx = dwgt / t.r2c * 6.0f * t.x * (1.0f - t.x);
                        const float dxr = (t.xr >= 0.f && t.xr <= 1.f) ? dx : 0.f;
                        const float dnum = dxr / s.sc[j];
                        const float dden = s.live[j] != 0.f ? -dxr * t.xr / s.sc[j] : 0.f;
                        acc[6] += dden; acc[7] -= dden + dnum;
#pragma unroll
                        for (int c = 0; c < 3; ++c) { acc[3 + c] -= dnum * t.d.l[c]; dl[c] -= dnum * dir[c]; }
                    }
                    if (!(t.d.r2 >= LIGHT_R2_MIN)) dr2 = 0.f;
                    float dw[3];
                    normalize_backward(t.d, dl, dw);
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float dy = dw[c] + 2.0f * t.d.w[c] * dr2;
                        acc[c] += dy;
                        if (rect) { acc[3 + c] += t.st[0] * dy; acc[6 + c] += t.st[1] * dy; }
                    }
                }
#pragma unroll
                for (int k = 0; k < SL_SLOTS; ++k) {
                    const float x = warp_sum(valid ? acc[k] : 0.f);
                    if (lane == 0) sAcc[warp][SL_SLOTS * j + k] += x;
                }
            }
        }
        if (vq_raw < total) {
#pragma unroll
            for (int c = 0; c < 3; ++c) a.dL_dbase_color[(3 * (size_t)v + c) * HW + q] = valid ? 0.f + dbase_v[c] : 0.f;
            a.dL_droughness[vq] = valid ? 0.f + drough_v : 0.f;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < SL_SLOTS * a.K; i += LS_THREADS) {
        float x = sAcc[0][i];
#pragma unroll
        for (int w = 1; w < LS_WARPS; ++w) x += sAcc[w][i];
        partial[(size_t)blockIdx.x * SL_SLOTS * a.K + i] = x;
    }
}

}  // namespace r3dg

// ---- C ABI --------------------------------------------------------------------------------------
using namespace r3dg;
extern "C" {

size_t r3dg_shade_pixel_lights_work_bytes(int V, int H, int W, int K) {
    if (V < 1 || H < 1 || W < 1 || K < 1) return 0;
    return (size_t)pixel_light_blocks((long long)V * H * W) * SL_SLOTS * K * sizeof(float);
}

// the checks of both directions: 0 and the light set, or the call's R3DG_ERR_* code
static int shade_pixel_lights_args(const r3dg_pixel_light_args* a, PixelLightSet& ls) {
    const int err = pixel_light_set(a, true, ls);
    if (err != 0) return err;
    if (!a->base_color || !a->roughness || !a->normal || !a->campos || (a->K > 0 && !a->shadows)) return R3DG_ERR_BAD_ARG;
    return 0;
}

int r3dg_shade_pixel_lights_forward(const r3dg_pixel_light_args* a, r3dg_stream_t stream_) {
    PixelLightSet ls;
    const int err = shade_pixel_lights_args(a, ls);
    if (err != 0) return err;
    if (!a->pbr || !a->diffuse_light || !a->specular) return R3DG_ERR_BAD_ARG;
    const cudaStream_t stream = (cudaStream_t)stream_;
    const long long pixels = (long long)a->V * a->H * a->W;
    if (a->K == 0) {
        const size_t n = (size_t)pixels * 3 * sizeof(float);
        R3DG_CUDA_TRY(cudaMemsetAsync(a->pbr, 0, n, stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->diffuse_light, 0, n, stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->specular, 0, n, stream));
        return 0;
    }
    const int blocks = pixel_light_blocks(pixels);
    if (ls.shaped) pixel_shaped_fwd_kernel<<<blocks, LS_THREADS, 0, stream>>>(*a, ls.rect_mask, ls.R);
    else pixel_lights_fwd_kernel<<<blocks, LS_THREADS, 0, stream>>>(*a, ls.point_mask);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int r3dg_shade_pixel_lights_backward(const r3dg_pixel_light_args* a, r3dg_stream_t stream_) {
    PixelLightSet ls;
    const int err = shade_pixel_lights_args(a, ls);
    if (err != 0) return err;
    if (!a->dL_dpbr || !a->dL_dbase_color || !a->dL_droughness) return R3DG_ERR_BAD_ARG;
    if (a->K > 0 && (!a->dL_dpos || !a->dL_dcolor || (ls.shaped && (!a->dL_da || !a->dL_db || !a->dL_dcone))))
        return R3DG_ERR_BAD_ARG;
    const size_t need = r3dg_shade_pixel_lights_work_bytes(a->V, a->H, a->W, a->K);
    if (need > 0 && (!a->work || a->work_bytes < need)) return R3DG_ERR_BAD_ARG;
    const cudaStream_t stream = (cudaStream_t)stream_;
    const long long pixels = (long long)a->V * a->H * a->W;
    if (a->K == 0) {
        R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dbase_color, 0, (size_t)pixels * 3 * sizeof(float), stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_droughness, 0, (size_t)pixels * sizeof(float), stream));
        return 0;
    }
    const int blocks = pixel_light_blocks(pixels);
    float* partial = (float*)a->work;
    if (ls.shaped) {
        pixel_shaped_bwd_kernel<<<blocks, LS_THREADS, 0, stream>>>(*a, ls.rect_mask, ls.R, partial);
        R3DG_CUDA_TRY(cudaGetLastError());
        r3dg_shaped_light_args r{};                      // the fields shaped_reduce_kernel reads and writes
        r.K = a->K; r.a = a->a; r.b = a->b;
        r.dL_dpos = a->dL_dpos; r.dL_da = a->dL_da; r.dL_db = a->dL_db; r.dL_dcolor = a->dL_dcolor; r.dL_dcone = a->dL_dcone;
        return launch_shaped_reduce(r, ls.rect_mask, blocks, partial, stream);
    }
    pixel_lights_bwd_kernel<<<blocks, LS_THREADS, 0, stream>>>(*a, ls.point_mask, partial);
    R3DG_CUDA_TRY(cudaGetLastError());
    return launch_lights_reduce(a->K, blocks, partial, a->dL_dpos, a->dL_dcolor, stream);
}

}  // extern "C"
